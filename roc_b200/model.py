"""Python mirror of the reference's Model / op-builder API (gnn.h:162-203) over the
C++ host (include/roc_host.h).  Same method names and call order as the model
script in gnn.cc:65-111:

    host = Host(device, rank, world)            # Runtime (one per process / GPU)
    host.graph_from_arrays(row_end, col_src)    # Graph(ctx, runtime, config)
    m = Model(host)
    x = m.create_node_tensor(602); y = m.create_node_tensor(41); mk = m.create_node_tensor(1, is_int=True)
    t = m.dropout(x, 0.5); t = m.linear(t, 64); t = m.indegree_norm(t); t = m.scatter_gather(t) ...
    m.softmax_cross_entropy(t, y, mk)
    m.adam(lr, weight_decay); m.init()
    m.train_mode(); m.zero_gradients(); m.forward(); m.backward(); m.update()
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import PerfMetrics, check, lib


class Host:
    """Runtime + Graph of one process: owns the GPU, the stream, the partition's CSR."""

    def __init__(self, device=0, my_part=0, num_parts=1):
        _lib.require_device()
        self.device, self.my_part, self.num_parts = device, my_part, num_parts
        self.h = C.c_void_p(lib.roc_host_create(device, my_part, num_parts))
        self._keep = []

    # --- NCCL bootstrap: rank 0 makes the id, the launcher (torch.distributed) broadcasts it
    @staticmethod
    def nccl_unique_id():
        buf = (C.c_ubyte * 128)()
        check(lib.roc_host_nccl_unique_id(buf), "roc_host_nccl_unique_id")
        return bytes(buf)

    def nccl_init(self, uid):
        buf = (C.c_ubyte * 128).from_buffer_copy(uid)
        check(lib.roc_host_nccl_init(self.h, buf), "roc_host_nccl_init")

    def graph_from_lux(self, prefix):
        check(lib.roc_host_graph_from_lux(self.h, prefix.encode()))

    def graph_from_arrays(self, row_end, col_src):
        row_end = np.ascontiguousarray(row_end, dtype=np.uint64)
        col_src = np.ascontiguousarray(col_src, dtype=np.uint32)
        check(lib.roc_host_graph_from_arrays(self.h, row_end.shape[0], int(row_end[-1]), row_end.ctypes.data,
                                             col_src.ctypes.data))

    def graph_info(self):
        out = (C.c_uint64 * 6)()
        check(lib.roc_host_graph_info(self.h, out))
        k = ["numNodes", "numEdges", "rowLeft", "rowRight", "colLeft", "colRight"]
        return dict(zip(k, [int(v) for v in out]))

    def plan_info(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib.roc_sg_plan_info(lib.roc_host_graph_plan(self.h), C.byref(a), C.byref(b), C.byref(c)))
        return {"chunks": a.value, "carries": b.value, "heavy_rows": c.value}

    def synchronize(self):
        check(lib.roc_host_synchronize(self.h))

    @property
    def stream(self):
        return lib.roc_host_stream(self.h)

    def close(self):
        if self.h:
            lib.roc_host_destroy(self.h)
            self.h = None


class Model:
    def __init__(self, host, seed=None):
        self.host = host
        self.h = host.h
        self._bf16 = set()               # handles of the bf16 node tensors
        if seed is not None:
            lib.roc_host_srand(seed)     # std::srand(config.seed), gnn.cc:56

    # ---- builders (gnn.h:165-179)
    def create_node_tensor(self, hidden, is_int=False, dtype="float32"):
        """dtype "float32" (every tensor) or "bfloat16": a leaf feature tensor held in bf16 (rounded to nearest even,
        half the memory), which only linear and dropout may read; init() refuses any other op on it.  It has no
        gradient.  set_tensor takes fp32 rows or a torch.bfloat16 tensor, get_tensor returns fp32 (raw=True: the
        bits as uint16)."""
        if dtype in ("bfloat16", "bf16"):
            assert not is_int
            t = lib.roc_host_create_node_tensor_bf16(self.h, hidden)
            self._bf16.add(t)
            return t
        assert dtype in ("float32", np.float32), dtype
        return lib.roc_host_create_node_tensor(self.h, hidden, int(is_int))

    def is_bf16(self, t):
        return t in self._bf16

    def dropout(self, t, rate, seed=0):
        return lib.roc_host_dropout(self.h, t, rate, seed)

    def linear(self, t, out_dim, activation=_lib.AC_MODE_NONE):
        return lib.roc_host_linear(self.h, t, out_dim, activation)

    def indegree_norm(self, t):
        return lib.roc_host_indegree_norm(self.h, t)

    def create_edge_tensor(self, hidden=1):
        """One fp32 value per edge of this partition, in CSR order (Model::create_edge_tensor); hidden must be 1."""
        return lib.roc_host_create_edge_tensor(self.h, int(hidden))

    def set_edge_grad(self, edges, on=True):
        """Compute the edge tensor's gradient in backward (off by default): the sum over the weighted scatter_gathers
        that read it.  Call before init() when the weighted op's input has no gradient of its own."""
        check(lib.roc_host_set_edge_grad(self.h, edges, int(bool(on))))

    def scatter_gather(self, t, aggr=_lib.AGGR_SUM, weights=None, dropout=0.0, seed=0):
        """aggr: AGGR_SUM (the reference's op), AGGR_AVG (sum -> indegree_norm -> indegree_norm), AGGR_MAX / AGGR_MIN
        (per feature over the in-neighbours; one partition only).  weights: an edge tensor (create_edge_tensor) for
        the edge-weighted sum over each row's in-edges, whose backward is exact on any graph (one partition only).
        dropout: edge dropout of the sum in train mode (one partition only): each in-edge kept with probability
        1 - dropout and scaled by 1 / (1 - dropout), the mask drawn anew every step from `seed` and the op's position
        (include/roc_b200.h, roc_sg_forward_dropout_planned).  Degrees stay the full graph's: dropout on the normalised
        adjacency entries as in PyG's APPNP, not DropEdge's renormalisation.  A rate outside [0, 1), or dropout with
        weights or another aggregator than AGGR_SUM, raises ValueError."""
        _check_rate(dropout, "dropout")
        if dropout != 0 and (weights is not None or aggr != _lib.AGGR_SUM):
            raise ValueError("edge dropout goes with the unweighted sum aggregation only")
        if dropout != 0:
            return lib.roc_host_scatter_gather_dropout(self.h, t, float(dropout), int(seed))
        if weights is not None:
            assert aggr == _lib.AGGR_SUM, "edge weights go with the sum"
            return lib.roc_host_scatter_gather_weighted(self.h, t, weights)
        if aggr == _lib.AGGR_SUM:
            return lib.roc_host_scatter_gather(self.h, t)
        return lib.roc_host_scatter_gather_aggr(self.h, t, int(aggr))

    def attention_gather(self, t, scores, heads=1, negative_slope=0.2, dropout=0.0, seed=0):
        """GAT aggregation of t (H = heads * F columns) weighted by a per-head softmax over each row's in-edges of
        LeakyReLU(s_dst[v] + s_src[u]); scores has 2 * heads columns [s_dst | s_src].  One partition only.
        dropout: attention dropout in train mode, each head's weight of each (destination, source) pair kept with
        probability 1 - dropout and scaled by 1 / (1 - dropout), drawn anew every step from `seed` (include/roc_b200.h,
        roc_sg_attn_forward_dropout_planned).  A rate outside [0, 1) raises ValueError."""
        _check_rate(dropout, "dropout")
        if dropout == 0:
            return lib.roc_host_attention_gather(self.h, t, scores, int(heads), float(negative_slope))
        return lib.roc_host_attention_gather_dropout(self.h, t, scores, int(heads), float(negative_slope),
                                                     float(dropout), int(seed))

    def dynamic_attention_gather(self, xl, xr, heads=1, negative_slope=0.2):
        """GATv2's dynamic attention (Brody et al., PyG GATv2Conv without bias): per destination v and head k over v's
        in-edges u, e = sum_f a[k][f] LeakyReLU(xl[u][kF+f] + xr[v][kF+f]), p = softmax_u(e), and
        out[v][kF:(k+1)F] = sum_u p xl[u][kF:(k+1)F].  xl and xr have H = heads * F columns (H <= 256, heads <= 8) and
        may be one tensor (PyG's share_weights).  Appends one parameter a of parameter_shape (heads, F), so get_parameter
        returns it as (F, heads), drawn uniform in +-sqrt(6 / (heads + F)) as PyG's glorot draws GATv2Conv.att.  A mode
        of attention_gather: op_info reports it as one.  One partition only."""
        return lib.roc_host_dynamic_attention_gather(self.h, xl, xr, int(heads), float(negative_slope))

    def softmax_gather(self, t, temperature=1.0, learn_temperature=False):
        """Softmax aggregation with one temperature t (PyG SoftmaxAggregation(t, learn=learn_temperature), GENConv's
        default aggregator): per destination v and column f over v's in-edges u, p = softmax_u(t * x[u][f]) and
        out[v][f] = sum_u p * x[u][f] (0 for a row with no in-edge).  t = 0 is the mean, a large t approaches the max and
        a negative t leans towards the min.  learn_temperature: t is a parameter of parameter_shape (1, 1), appended
        here and set to `temperature` without a random draw, trained by Adam with the model's weight decay; otherwise a
        constant.  A mode of attention_gather: op_info reports it as one.  fp32 input only (init() refuses a bf16 one);
        one partition only.  A temperature that is not finite raises ValueError."""
        if not math.isfinite(float(temperature)):
            raise ValueError("temperature must be finite")
        return lib.roc_host_softmax_gather(self.h, t, float(temperature), int(bool(learn_temperature)))

    def dot_attention_gather(self, q, k, v, heads=1, scale=None):
        """Dot-product attention, the graph transformer layer's (PyG TransformerConv's attention; UniMP, Shi et al.
        2021): per destination v and head k over v's in-edges u, s = scale * q[v]_k . k[u]_k, p = softmax_u(s) and
        out[v]_k = sum_u p * v[u]_k (0 for a row with no in-edge).  q, k and v have H = heads * F columns (H <= 256,
        heads <= 8), and any of them may be the same tensor, whose gradient then takes every part.  scale=None is
        1 / sqrt(F), computed in double and rounded once to fp32.  No parameter.  A mode of attention_gather: op_info
        reports it as one.  fp32 inputs only; one partition only.  heads outside [1, 8] and a scale that is 0 or not
        finite in fp32 raise ValueError."""
        if isinstance(heads, bool) or not isinstance(heads, (int, np.integer)) or not 1 <= heads <= 8:
            raise ValueError("heads must be an integer in [1, 8]")
        if scale is None:
            scale = fp32(1.0 / math.sqrt(max(self.tensor_shape(q)[1] // int(heads), 1)))
        if not math.isfinite(fp32(scale)) or fp32(scale) == 0.0:
            raise ValueError("scale must be finite and not 0 in fp32")
        return lib.roc_host_dot_attention_gather(self.h, q, k, v, int(heads), fp32(scale))

    def attention_scores(self, t, heads=1):
        """GAT's per-head scores of t (H = heads * F columns): [s_dst | s_src], 2 * heads columns, the scores attention_gather
        takes.  Head k's scores are the dot products of its own F columns with its a_dst and a_src.  Appends one parameter
        A of parameter_shape (F, 2 * heads), so get_parameter returns it as (2 * heads, F): rows 0 .. heads - 1 the a_dst,
        the rest the a_src, drawn as a Linear F -> 2 * heads draws its W.  One partition only."""
        return lib.roc_host_attention_scores(self.h, t, int(heads))

    def relu(self, t):
        return lib.roc_host_relu(self.h, t)

    def elu(self, t):
        """ELU with alpha = 1: x > 0 ? x : exp(x) - 1.  Never fused; linear() does not take it as an activation."""
        return lib.roc_host_elu(self.h, t)

    def sigmoid(self, t):
        return lib.roc_host_sigmoid(self.h, t)

    def add(self, a, b):
        return lib.roc_host_add(self.h, a, b)

    def scaled_add(self, a, b, alpha, beta):
        """fmaf(alpha, a, beta * b) with alpha and beta rounded to fp32 (Model::scaled_add), the initial residual of
        APPNP and GCNII; a and b are different tensors of one shape.  A non-finite coefficient raises ValueError.  With
        fusion on, init() folds it into the store of a sum scatter_gather whose indegree_norm feeds only it (as a)."""
        for name, v in (("alpha", alpha), ("beta", beta)):
            if not (math.isfinite(float(v)) and abs(float(v)) <= float(np.finfo(np.float32).max)):
                raise ValueError("%s must be finite in fp32" % name)
        return lib.roc_host_scaled_add(self.h, a, b, float(alpha), float(beta))

    def batch_norm(self, t, momentum=0.1, eps=1e-5):
        """torch.nn.BatchNorm1d over every local row: appends two parameters, gamma (ones) then beta (zeros), each of
        parameter_shape (H, 1).  A training forward uses the batch statistics and updates the running mean / variance
        (start 0 / 1); infer mode uses the running statistics.  A relu that alone reads the output is fused into it.
        One partition only; init() refuses fewer than 2 rows."""
        return lib.roc_host_batch_norm(self.h, t, float(momentum), float(eps))

    def layer_norm(self, t, eps=1e-5):
        """torch.nn.LayerNorm(H, eps) over the columns of each local row: appends two parameters, gamma (ones) then
        beta (zeros), each of parameter_shape (H, 1).  The same forward in train and infer mode (no running
        statistics).  A relu that alone reads the output is fused into it.  op_info reports it as a batch_norm, the
        normalisation kind.  A negative or non-finite eps raises ValueError.  One partition only."""
        if not (math.isfinite(float(eps)) and float(eps) >= 0.0 and abs(float(eps)) <= float(np.finfo(np.float32).max)):
            raise ValueError("eps must be finite and >= 0")
        return lib.roc_host_layer_norm(self.h, t, float(eps))

    def batch_norm_stats(self, t):
        """(running mean, running variance), fp32 [H] each, of the batch_norm whose output is t."""
        h = self.tensor_shape(t)[1]
        mean, var = np.empty(h, dtype=np.float32), np.empty(h, dtype=np.float32)
        check(lib.roc_host_get_batch_norm_stats(self.h, t, mean.ctypes.data, var.ctypes.data))
        return mean, var

    def set_batch_norm_stats(self, t, mean, var):
        h = self.tensor_shape(t)[1]
        mean, var = np.ascontiguousarray(mean, dtype=np.float32), np.ascontiguousarray(var, dtype=np.float32)
        assert mean.shape == (h,) and var.shape == (h,), (mean.shape, var.shape, h)
        check(lib.roc_host_set_batch_norm_stats(self.h, t, mean.ctypes.data, var.ctypes.data))

    def softmax_cross_entropy(self, logits, labels, mask):
        check(lib.roc_host_softmax_cross_entropy(self.h, logits, labels, mask))

    def sigmoid_cross_entropy(self, logits, labels, mask):
        """Multi-label loss: per class, binary cross-entropy on the logit (labels from set_multilabels).  Gradient
        sigmoid(z) - y on train rows; metrics in multilabel_metrics().  One partition only."""
        check(lib.roc_host_sigmoid_cross_entropy(self.h, logits, labels, mask))

    def adam(self, lr=0.01, weight_decay=0.05):
        check(lib.roc_host_adam(self.h, lr, weight_decay))

    @property
    def lr(self):
        return lib.roc_host_get_lr(self.h)

    @lr.setter
    def lr(self, v):
        check(lib.roc_host_set_lr(self.h, v))

    def set_fusion(self, on):
        check(lib.roc_host_set_fusion(self.h, int(on)))

    def set_exact_backward(self, on=True):
        """Train the sum (and mean), max / min and attention aggregations on their exact gradient over the graph's
        transpose, which is right on directed graphs and multigraphs (off by default: the gather over the same CSR,
        exact only on a symmetric graph).  Call before init().  One partition only."""
        check(lib.roc_host_set_exact_backward(self.h, int(bool(on))))

    def set_bf16_aggregation(self, on=True):
        """Store in bf16 each tensor that a Linear without activation writes (its output, or the indegree_norm fused
        into it) and that one sum scatter_gather alone reads; and each tensor that a Linear without activation or an
        unfused relu writes, that a max / min, weighted or attention aggregation reads as its features, and that
        nothing else reads but those and Linears taking it as X without a fused dropout.  The producer rounds as it
        stores (a relu's backward masks by the stored value), the aggregations read half-width rows and compute in
        fp32.  Gradients and every other tensor stay fp32; tensor_dtype() shows which tensors init() chose.  Call
        before init().  One partition only."""
        check(lib.roc_host_set_bf16_aggregation(self.h, int(bool(on))))

    def init(self):
        check(lib.roc_host_init(self.h))

    # ---- data
    def load_features(self, t, prefix):
        check(lib.roc_host_load_features(self.h, t, prefix.encode()))

    def load_labels(self, t, prefix):
        check(lib.roc_host_load_labels(self.h, t, prefix.encode()))

    def load_train_mask(self, t, prefix):
        check(lib.roc_host_load_train_mask(self.h, t, prefix.encode()))

    def tensor_shape(self, t):
        out = (C.c_int64 * 3)()
        check(lib.roc_host_tensor_shape(self.h, t, out))
        return int(out[0]), int(out[1]), int(out[2])

    def tensor_ptr(self, t, grad=False):
        return lib.roc_host_tensor_ptr(self.h, t, int(grad))

    def tensor_dtype(self, t):
        """How the tensor's data is stored: "float32", "bfloat16" or "int32" (gradients are always fp32)."""
        return _lib.HOST_DTYPES[lib.roc_host_tensor_dtype(self.h, t)]

    def set_tensor(self, t, arr, grad=False):
        rows, hidden, _ = self.tensor_shape(t)
        if t in self._bf16 or (not grad and self.tensor_dtype(t) == "bfloat16"):
            if grad:
                raise _lib.RocError("set_tensor(grad=True): a bf16 leaf tensor has no gradient")
            if str(getattr(arr, "dtype", "")) == "torch.bfloat16":
                import torch   # only a torch tensor can carry bf16 rows
                bits = np.ascontiguousarray(arr.detach().contiguous().cpu().view(torch.int16).numpy())   # copied as is
                assert bits.size == rows * hidden, (bits.shape, rows, hidden)
                check(lib.roc_host_set_tensor_bf16(self.h, t, bits.ctypes.data))
                return
            arr = np.ascontiguousarray(arr, dtype=np.float32)   # fp32 rows, rounded on the device
        arr = np.ascontiguousarray(arr)
        assert arr.itemsize == 4 and arr.size == rows * hidden, (arr.shape, rows, hidden)
        check(lib.roc_host_set_tensor(self.h, t, arr.ctypes.data, int(grad)))

    def set_tensor_from_host_ptr(self, t, ptr, grad=False):
        """ptr: address of a dense [rows][hidden] 4-byte host buffer (e.g. pinned torch memory)."""
        check(lib.roc_host_set_tensor(self.h, t, C.c_void_p(ptr), int(grad)))

    def get_tensor(self, t, grad=False, dtype=np.float32, raw=False):
        """the tensor's rows as fp32 (a bf16 tensor widened exactly); raw=True on a bf16 tensor: its bits (uint16).
        grad=True on a bf16 tensor an op produces (set_bf16_aggregation) gives its fp32 gradient."""
        rows, hidden, _ = self.tensor_shape(t)
        if t in self._bf16 or (not grad and self.tensor_dtype(t) == "bfloat16"):
            if grad:
                raise _lib.RocError("get_tensor(grad=True): a bf16 leaf tensor has no gradient")
            if raw:
                out = np.empty((rows, hidden), dtype=np.uint16)
                check(lib.roc_host_get_tensor_bf16(self.h, t, out.ctypes.data))
                return out
        out = np.empty((rows, hidden), dtype=dtype)
        check(lib.roc_host_get_tensor(self.h, t, out.ctypes.data, int(grad)))
        return out

    def get_aggr_index(self, t):
        """The source ids a max / min scatter_gather output t was taken from, [rows][hidden] uint32 (after forward)."""
        rows, hidden, _ = self.tensor_shape(t)
        out = np.empty((rows, hidden), dtype=np.uint32)
        check(lib.roc_host_get_aggr_index(self.h, t, out.ctypes.data))
        return out

    def set_labels(self, t, class_idx):
        a = np.ascontiguousarray(class_idx, dtype=np.int32)
        check(lib.roc_host_set_labels(self.h, t, a.ctypes.data))

    def set_multilabels(self, t, labels):
        """labels: a [rows][C] 0/1 or bool array for the label tensor t (C = its width), packed here
        (pack_multilabels) for sigmoid_cross_entropy."""
        rows, hidden, _ = self.tensor_shape(t)
        labels = np.asarray(labels)
        assert labels.shape == (rows, hidden), (labels.shape, rows, hidden)
        bits = pack_multilabels(labels)
        check(lib.roc_host_set_multilabels(self.h, t, bits.ctypes.data))

    def num_parameters(self):
        return lib.roc_host_num_parameters(self.h)

    def parameter_shape(self, p):
        out = (C.c_int64 * 2)()
        check(lib.roc_host_parameter_shape(self.h, p, out))
        return int(out[0]), int(out[1])   # inDim, outDim

    def get_parameter(self, p, which="w"):
        i, o = self.parameter_shape(p)
        out = np.empty((o, i), dtype=np.float32)   # W_mem[o*inDim + i]
        check(lib.roc_host_get_parameter(self.h, p, out.ctypes.data, {"w": 0, "grad": 1, "m": 2, "v": 3}[which]))
        return out

    def set_parameter(self, p, w):
        i, o = self.parameter_shape(p)
        w = np.ascontiguousarray(w, dtype=np.float32)
        assert w.shape == (o, i)
        check(lib.roc_host_set_parameter(self.h, p, w.ctypes.data))

    def op_info(self):
        """Per layer, in creation order, what init() decided: the op kind and its fusion fields (roc_host_op_info),
        tensors as handles or -1."""
        out = []
        for layer in range(lib.roc_host_num_ops(self.h)):
            info = _lib.HostOpInfo()
            check(lib.roc_host_op_info(self.h, layer, C.byref(info)), "roc_host_op_info")
            out.append(info.as_dict())
        return out

    # ---- train loop (gnn.cc:99-111)
    def train_mode(self):
        check(lib.roc_host_train_mode(self.h))

    def infer_mode(self):
        check(lib.roc_host_infer_mode(self.h))

    def zero_gradients(self):
        check(lib.roc_host_zero_gradients(self.h))

    def forward(self):
        check(lib.roc_host_forward(self.h))

    def backward(self):
        check(lib.roc_host_backward(self.h))

    def update(self):
        check(lib.roc_host_update(self.h))

    def train_epoch(self):
        check(lib.roc_host_train_epoch(self.h))

    def profile_sg(self, on=True):
        check(lib.roc_host_profile_sg(self.h, int(on)))

    def profile_sg_read(self, max_entries=4096):
        hs = (C.c_int * max_entries)()
        ms = (C.c_float * max_entries)()
        n = lib.roc_host_profile_sg_read(self.h, max_entries, hs, ms)
        return [(int(hs[i]), float(ms[i])) for i in range(n)]

    def metrics(self):
        pm = PerfMetrics()
        check(lib.roc_host_metrics(self.h, C.byref(pm)))
        return pm.as_dict()

    def multilabel_metrics(self):
        """The last sigmoid_cross_entropy pass's metrics: loss, rows, exact, tp, fp, fn (each [train, val, test]) and
        micro_f1 = 2tp / (2tp + fp + fn) per split (NaN where that denominator is 0)."""
        mm = _lib.MultilabelMetrics()
        check(lib.roc_host_multilabel_metrics(self.h, C.byref(mm)), "roc_host_multilabel_metrics")
        d = mm.as_dict()
        d["micro_f1"] = [_micro_f1(tp, fp, fn) for tp, fp, fn in zip(d["tp"], d["fp"], d["fn"])]
        return d


def _micro_f1(tp, fp, fn):
    den = 2 * tp + fp + fn
    return 2.0 * tp / den if den else float("nan")


def pack_multilabels(labels):
    """[rows][C] 0/1 or bool labels -> uint32 [rows][ceil(C / 32)]: bit c % 32 of word c // 32 is label c (the layout
    of roc_sigmoid_xent_bwd and Model.set_multilabels)."""
    y = np.asarray(labels)
    assert y.ndim == 2, "labels must be [rows][C]"
    rows, c = y.shape
    w = (c + 31) // 32
    padded = np.zeros((rows, w * 32), dtype=np.uint8)
    padded[:, :c] = y != 0
    bytes_ = np.packbits(padded.reshape(rows, w * 4, 8), axis=2, bitorder="little").reshape(rows, w * 4)
    return np.ascontiguousarray(bytes_).view("<u4").astype(np.uint32).reshape(rows, w)


def _input_tensor(model, hidden, features):
    """the builders' input features: fp32, or bf16 with features="bfloat16" (the plain call for fp32, so that any object
    with the builder methods can stand in for a Model)"""
    if features == "float32":
        return model.create_node_tensor(hidden)
    return model.create_node_tensor(hidden, dtype=features)


def _aggregation(model, aggregation):
    """aggregation="bfloat16": Model.set_bf16_aggregation; "float32" (the default) leaves the model as it is."""
    if aggregation not in ("float32", "bfloat16"):
        raise ValueError("aggregation must be \"float32\" or \"bfloat16\"")
    if aggregation == "bfloat16":
        model.set_bf16_aggregation(True)


def _loss(model, loss, logits, label, mask):
    """The builders' head: loss="softmax" (the default) is softmax_cross_entropy with one class per row (set_labels);
    "sigmoid" is the multi-label sigmoid_cross_entropy (set_multilabels)."""
    if loss == "softmax":
        model.softmax_cross_entropy(logits, label, mask)
    elif loss == "sigmoid":
        model.sigmoid_cross_entropy(logits, label, mask)
    else:
        raise ValueError("loss must be \"softmax\" or \"sigmoid\"")


def _check_norm(norm):
    if norm not in (None, "batch", "layer_norm"):
        raise ValueError("norm must be None, \"batch\" or \"layer_norm\"")


def _check_rate(rate, name):
    if not 0.0 <= float(rate) < 1.0:
        raise ValueError("%s must be in [0, 1)" % name)


def _sum_gather(model, t, edge_dropout):
    """The sum scatter_gather of a builder, with edge dropout when edge_dropout > 0 (else the plain call)."""
    if edge_dropout:
        return model.scatter_gather(t, dropout=float(edge_dropout))
    return model.scatter_gather(t)


def _hidden_norm(model, norm, t, bns):
    """norm="batch": batch_norm on a hidden layer's output, right before its relu; norm="layer_norm": layer_norm in
    the same place; None leaves t as it is."""
    if norm is None:
        return t
    t = model.layer_norm(t) if norm == "layer_norm" else model.batch_norm(t)
    bns.append(t)
    return t


def build_gcn(model, layers, dropout_rate, lr=0.01, weight_decay=0.05, exact_backward=False, features="float32",
              aggregation="float32", loss="softmax", norm=None, edge_dropout=0.0):
    """The model script of gnn.cc:65-98 for `-layers a-b-...-c`.  Returns the handles.  exact_backward: train on the
    exact gradient over the graph's transpose (Model.set_exact_backward), for directed graphs; the same keyword on
    build_sage_mean, build_sage_pool and build_gat.  features="bfloat16" keeps the input features in bf16
    (Model.create_node_tensor); the same keyword on every builder.  aggregation="bfloat16" stores the fused
    linear -> indegree_norm output each scatter_gather reads in bf16 (Model.set_bf16_aggregation); the same keyword
    on every builder.  loss="sigmoid" ends the model in the multi-label sigmoid_cross_entropy instead of the softmax
    (labels then go in with Model.set_multilabels); the same keyword on every builder.  norm="batch" puts a
    batch_norm (Model.batch_norm) on every hidden layer's output right before its relu (here after the second
    indegree_norm, and before the residual add), never on the last layer; norm="layer_norm" puts a layer_norm
    (Model.layer_norm, torch.nn.LayerNorm over each row's features) in the same place.  The same keyword on every
    builder, which then returns the norm outputs as `bns`.  edge_dropout > 0 drops each layer's in-edges at that rate in
    train mode (Model.scatter_gather(dropout=)), a fresh mask per layer and step, with the degrees of the full graph
    (DropEdge's regulariser on the normalised adjacency, without its renormalisation); a rate outside [0, 1) raises
    ValueError, and 0 builds the model without it."""
    _check_norm(norm)
    _check_rate(edge_dropout, "edge_dropout")
    L = len(layers)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    t = x
    relu_outs, bns = [], []
    for i in range(1, L):
        t = model.dropout(t, dropout_rate)
        skip = t
        t = model.linear(t, layers[i], _lib.AC_MODE_NONE)
        t = model.indegree_norm(t)
        t = _sum_gather(model, t, edge_dropout)
        t = model.indegree_norm(t)
        if i != L - 1:
            t = model.relu(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
        if L > 3:   # residual branch, gnn.cc:86-90
            skip = model.linear(skip, layers[i], _lib.AC_MODE_NONE)
            t = model.add(t, skip)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    _aggregation(model, aggregation)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "bns": bns}


def build_sage_mean(model, layers, dropout_rate, lr=0.01, weight_decay=0.05, exact_backward=False,
                    features="float32", aggregation="float32", loss="softmax", norm=None):
    """GraphSAGE with the mean aggregator (BASELINE.json configs[2]) composed from the reference's own ops
    (gnn.h:165-179; AGGR_AVG is declared at gnn.h:75-80 but the reference's ScatterGather only sums):

        D    = dropout(t)
        nb   = indegree_norm(indegree_norm(scatter_gather(linear(D, d_i))))    # D^-1 A (D W_nb): the mean over
                                                                               # N(v) + v (self loops are in A)
        t    = add(nb, linear(D, d_i))                                         # + the root / self weight
        t    = relu(t)                                                         # all but the last layer

    x / sqrt(deg) / sqrt(deg) is the mean to within one fp32 rounding.  Same wiring as the reference's residual
    GCN layer (gnn.cc:79-90) with both norms after the aggregation.  aggregation="bfloat16" stores linear(D, d_i),
    which only the scatter_gather reads, in bf16 (Model.set_bf16_aggregation).  norm="batch" / "layer_norm": batch_norm / layer_norm on t before
    each hidden relu (see build_gcn)."""
    _check_norm(norm)
    L = len(layers)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    t = x
    relu_outs, bns = [], []
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        nb = model.linear(d, layers[i], _lib.AC_MODE_NONE)
        nb = model.scatter_gather(nb)
        nb = model.indegree_norm(nb)
        nb = model.indegree_norm(nb)
        root = model.linear(d, layers[i], _lib.AC_MODE_NONE)
        t = model.add(nb, root)
        if i != L - 1:
            t = model.relu(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    _aggregation(model, aggregation)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "bns": bns}


def build_sage_pool(model, layers, dropout_rate, aggr=_lib.AGGR_MAX, lr=0.01, weight_decay=0.05, exact_backward=False,
                    features="float32", aggregation="float32", loss="softmax", norm=None):
    """GraphSAGE with the pooling aggregator (Hamilton et al., 2017) composed from the reference's ops plus the max
    (or min) ScatterGather.  The reference's Linear has no bias, so neither has this.  Per layer:

        d  = dropout(t)
        p  = relu(linear(d, d_i))                      # the pooling network
        nb = scatter_gather(p, aggr)                   # per feature, max (min) over N(v) + v (self loops are in A)
        t  = add(linear(nb, d_i), linear(d, d_i))      # neighbour weight + root / self weight
        t  = relu(t)                                   # all but the last layer

    Single partition; init refuses a graph with a duplicate edge in a row.  aggregation="bfloat16" stores p, the relu
    output the scatter_gather reads, in bf16 (Model.set_bf16_aggregation).  norm="batch" / "layer_norm": batch_norm / layer_norm on t before each
    hidden layer's last relu (see build_gcn; the pooling network's relu is not a hidden layer's output).  Returns the
    handles, with `pools` (the scatter_gather outputs, for get_aggr_index) and `pool_ins` (their inputs)."""
    _check_norm(norm)
    L = len(layers)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    t = x
    relu_outs, pools, pool_ins, bns = [], [], [], []
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        p = model.relu(model.linear(d, layers[i], _lib.AC_MODE_NONE))
        nb = model.scatter_gather(p, aggr)
        pool_ins.append(p)
        pools.append(nb)
        t = model.add(model.linear(nb, layers[i], _lib.AC_MODE_NONE), model.linear(d, layers[i], _lib.AC_MODE_NONE))
        if i != L - 1:
            t = model.relu(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    _aggregation(model, aggregation)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "pools": pools,
            "pool_ins": pool_ins, "bns": bns}


def build_gat(model, layers, dropout_rate, heads=1, negative_slope=0.2, lr=0.01, weight_decay=0.05,
              exact_backward=False, features="float32", aggregation="float32", loss="softmax", norm=None,
              scores="dense", activation="relu", attn_dropout=0.0):
    """GAT (Velickovic et al., 2018) built from the reference's ops plus attention_gather.  `heads` (an int, or one
    value per hidden layer) applies to the hidden layers; the last layer has one head.  layers[i] is the width of
    layer i's output, heads_i * F_i.  Per layer:

        d  = dropout(t)
        wh = linear(d, layers[i])                       # heads_i * F_i columns
        sc = linear(wh, 2 * heads_i)                    # scores="dense": [s_dst | s_src] per head
        sc = attention_scores(wh, heads_i)              # scores="per_head": the same, head k from its own F columns
        t  = attention_gather(wh, sc, heads_i, slope)   # per head, softmax over N(v) + v (self loops are in A),
                                                        # attn_dropout > 0: with that attention dropout
        t  = relu(t)                                    # all but the last layer; activation="elu": elu(t)

    scores="per_head" gives each head its own a_dst and a_src (Model.attention_scores), as the paper and PyG's GATConv
    do; the default "dense" projects all heads' features for every head's scores, which is the same function only
    with one head.  activation="elu" uses the paper's ELU in place of ReLU.  attn_dropout: dropout of the normalised
    attention coefficients at that rate on every layer (Model.attention_gather's dropout; the paper uses 0.6 beside
    dropout_rate = 0.6).  With scores="per_head", activation="elu" and attn_dropout, the model is the paper's GAT
    without bias, with any number of heads.

    Where this differs from the paper: there is no bias (the reference's Linear has none; norm="batch" gives a
    per-feature shift).  Single partition.  aggregation="bfloat16" stores wh, which the attention_gather and the score
    op read, in bf16 (Model.set_bf16_aggregation).  norm="batch" / "layer_norm": batch_norm / layer_norm on t before each hidden activation (see
    build_gcn).  Returns the handles, with `attn` (the attention_gather outputs), `attn_ins` (their feature inputs),
    `scores` and `relu_outs` (the hidden activations' outputs, ELU or ReLU)."""
    _check_norm(norm)
    if scores not in ("dense", "per_head"):
        raise ValueError("scores must be \"dense\" or \"per_head\"")
    if activation not in ("relu", "elu"):
        raise ValueError("activation must be \"relu\" or \"elu\"")
    _check_rate(attn_dropout, "attn_dropout")
    L = len(layers)
    hs = list(heads) if isinstance(heads, (list, tuple)) else [int(heads)] * (L - 2)
    assert len(hs) == L - 2, "one head count per hidden layer"
    hs.append(1)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    act = model.elu if activation == "elu" else model.relu
    t = x
    relu_outs, attn, attn_ins, score_outs, bns = [], [], [], [], []
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        wh = model.linear(d, layers[i], _lib.AC_MODE_NONE)
        if scores == "per_head":
            sc = model.attention_scores(wh, hs[i - 1])
        else:
            sc = model.linear(wh, 2 * hs[i - 1], _lib.AC_MODE_NONE)
        if attn_dropout:
            t = model.attention_gather(wh, sc, hs[i - 1], negative_slope, attn_dropout)
        else:
            t = model.attention_gather(wh, sc, hs[i - 1], negative_slope)
        attn_ins.append(wh)
        score_outs.append(sc)
        attn.append(t)
        if i != L - 1:
            t = act(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    _aggregation(model, aggregation)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "attn": attn,
            "attn_ins": attn_ins, "scores": score_outs, "bns": bns}


def build_gatv2(model, layers, dropout_rate, heads=1, negative_slope=0.2, share_weights=False, lr=0.01,
                weight_decay=0.05, exact_backward=False, features="float32", loss="softmax", norm=None,
                activation="relu"):
    """GATv2 (Brody et al., "How Attentive are Graph Attention Networks?"; PyG GATv2Conv without bias) built on
    dynamic_attention_gather.  `heads` (an int, or one value per hidden layer) applies to the hidden layers; the last
    layer has one head.  layers[i] is the width of layer i's output, heads_i * F_i.  Per layer:

        d  = dropout(t)
        xl = linear(d, layers[i])                          # the source / value rows
        xr = linear(d, layers[i])                          # the target rows; share_weights: xr = xl
        t  = dynamic_attention_gather(xl, xr, heads_i, slope)
        t  = relu(t)                                       # all but the last layer; activation="elu": elu(t)

    norm="batch" / "layer_norm": batch_norm / layer_norm on t before each hidden activation (see build_gcn).  exact_backward: the attention's
    source pass over the transposed graph (Model.set_exact_backward), exact on directed graphs and multigraphs.
    Single partition; the attention reads fp32 rows (features="bfloat16" stores only the input features in bf16).
    Returns the handles, with `attn` (the attention outputs), `attn_ins` (their (xl, xr) pairs) and `relu_outs`."""
    _check_norm(norm)
    if activation not in ("relu", "elu"):
        raise ValueError("activation must be \"relu\" or \"elu\"")
    L = len(layers)
    hs = list(heads) if isinstance(heads, (list, tuple)) else [heads] * (L - 2)
    if len(hs) != L - 2 or any(isinstance(h, bool) or not isinstance(h, (int, np.integer)) or not 1 <= h <= 8
                               for h in hs):
        raise ValueError("heads must be an integer in [1, 8], or one per hidden layer")
    if any(layers[i] % hs[i - 1] for i in range(1, L - 1)):
        raise ValueError("each hidden width must be a multiple of its heads")
    hs = [int(h) for h in hs] + [1]
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    act = model.elu if activation == "elu" else model.relu
    t = x
    relu_outs, attn, attn_ins, bns = [], [], [], []
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        xl = model.linear(d, layers[i], _lib.AC_MODE_NONE)
        xr = xl if share_weights else model.linear(d, layers[i], _lib.AC_MODE_NONE)
        t = model.dynamic_attention_gather(xl, xr, hs[i - 1], negative_slope)
        attn_ins.append((xl, xr))
        attn.append(t)
        if i != L - 1:
            t = act(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "attn": attn,
            "attn_ins": attn_ins, "bns": bns}


def build_graph_transformer(model, layers, dropout_rate, heads=1, root_weight=True, lr=0.01, weight_decay=0.05,
                            exact_backward=False, features="float32", loss="softmax", norm=None, activation="relu"):
    """The graph transformer (UniMP, Shi et al., "Masked Label Prediction", 2021; PyG TransformerConv without bias,
    edge features, beta or attention dropout) built on dot_attention_gather and stacked as build_gat stacks GAT.
    `heads` (an int, or one value per hidden layer) applies to the hidden layers; the last layer has one head.
    layers[i] is the width of layer i's output, heads_i * F_i.  Per layer:

        d       = dropout(t)
        q, k, v = linear(d, layers[i]) x 3                  # PyG's lin_query, lin_key, lin_value
        t       = dot_attention_gather(q, k, v, heads_i)    # scale 1 / sqrt(F_i)
        t       = add(t, linear(d, layers[i]))              # root_weight: PyG's lin_skip
        t       = act(norm(t))                              # all but the last layer

    activation: "relu" or "elu".  norm="batch" / "layer_norm": batch_norm / layer_norm before each hidden activation
    (see build_gcn).  exact_backward: the attention's source pass over the transposed graph
    (Model.set_exact_backward), exact on directed graphs and multigraphs.  Single partition; the attention reads fp32
    rows (features="bfloat16" stores only the input features in bf16).  Bad heads, widths, norm or activation raise
    ValueError.  Returns the handles, with `attn` (the attention outputs), `attn_ins` (their (q, k, v) triples),
    `relu_outs` (the hidden activations' outputs) and `bns`."""
    _check_norm(norm)
    if activation not in ("relu", "elu"):
        raise ValueError("activation must be \"relu\" or \"elu\"")
    L = len(layers)
    hs = list(heads) if isinstance(heads, (list, tuple)) else [heads] * (L - 2)
    if len(hs) != L - 2 or any(isinstance(h, bool) or not isinstance(h, (int, np.integer)) or not 1 <= h <= 8
                               for h in hs):
        raise ValueError("heads must be an integer in [1, 8], or one per hidden layer")
    if any(layers[i] % hs[i - 1] for i in range(1, L - 1)):
        raise ValueError("each hidden width must be a multiple of its heads")
    if any(w > 256 for w in layers[1:]):
        raise ValueError("the attention widths must be at most 256")
    hs = [int(h) for h in hs] + [1]
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    act = model.elu if activation == "elu" else model.relu
    t = x
    relu_outs, attn, attn_ins, bns = [], [], [], []
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        q, k, v = (model.linear(d, layers[i], _lib.AC_MODE_NONE) for _ in range(3))
        t = model.dot_attention_gather(q, k, v, hs[i - 1], fp32(1.0 / math.sqrt(layers[i] // hs[i - 1])))
        attn_ins.append((q, k, v))
        attn.append(t)
        if root_weight:
            t = model.add(t, model.linear(d, layers[i], _lib.AC_MODE_NONE))
        if i != L - 1:
            t = act(_hidden_norm(model, norm, t, bns))
            relu_outs.append(t)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "relu_outs": relu_outs, "attn": attn,
            "attn_ins": attn_ins, "bns": bns}


def build_deepergcn(model, layers, dropout_rate, depth, temperature=1.0, learn_temperature=True, norm="batch",
                    expansion=2, lr=0.01, weight_decay=0.05, exact_backward=False, features="float32", loss="softmax"):
    """DeeperGCN (Li et al., "DeeperGCN: All You Need to Train Deeper GCNs", 2020) as PyG's
    examples/ogbn_proteins_deepgcn.py builds it: DeepGCNLayer(block="res+") over GENConv(aggr="softmax", learn_t=True),
    without edge features.  layers = [in, hidden, out]:

        x = linear(x, hidden)                                   # node encoder
        x = genconv_1(x)                                        # layer 1: the conv alone
        for l in 2 .. depth:
            h = dropout(relu(norm(x)))                          # res+: norm, relu, dropout, conv, then the residual
            x = add(x, genconv_l(h))
        logits = linear(dropout(relu(norm(x))), out)

        genconv_l(h):  a = softmax_gather(relu(h), temperature, learn_temperature)
                       s = add(a, h)
                       z = relu(norm(linear(s, expansion * hidden)))
                       return linear(z, hidden)

    norm="layer_norm" is layer_norm, as PyG's example uses; norm="batch" is batch_norm; either fuses the relu after it;
    None leaves it out.  With norm="layer_norm" the model is PyG's except in two ways: there is no bias (the Linear has
    none), and GENConv's eps = 1e-7 added to each message is left out (the softmax weights sum to 1, so its only effect
    is to add eps to each aggregated value of a row that has an in-edge).  Each layer learns its own t when
    learn_temperature, else every t is the constant `temperature`.  exact_backward: the aggregation's backward over the
    transposed graph (Model.set_exact_backward), exact on directed graphs and multigraphs.  Single partition; the
    aggregation reads fp32 rows (features="bfloat16" stores only the input features in bf16).  Bad layers, depth,
    expansion, rates, norm or temperature raise ValueError.  Returns the handles, with `aggs` (the softmax_gather
    outputs), `temperatures` (each layer's t parameter index, or None) and `bns` (the norm outputs)."""
    if len(layers) != 3 or any(isinstance(w, bool) or not isinstance(w, (int, np.integer)) or w < 1 for w in layers):
        raise ValueError("layers must be [in, hidden, out], three positive integers")
    if isinstance(depth, bool) or not isinstance(depth, (int, np.integer)) or depth < 1:
        raise ValueError("depth must be an integer >= 1")
    if isinstance(expansion, bool) or not isinstance(expansion, (int, np.integer)) or expansion < 1:
        raise ValueError("expansion must be an integer >= 1")
    _check_rate(dropout_rate, "dropout_rate")
    _check_norm(norm)
    if not math.isfinite(float(temperature)):
        raise ValueError("temperature must be finite")
    hidden = int(layers[1])
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    aggs, temps, bns = [], [], []

    def norm_relu(t):
        return model.relu(_hidden_norm(model, norm, t, bns))

    def genconv(h):
        a = model.softmax_gather(model.relu(h), float(temperature), bool(learn_temperature))
        aggs.append(a)
        temps.append(model.num_parameters() - 1 if learn_temperature else None)
        z = norm_relu(model.linear(model.add(a, h), int(expansion) * hidden, _lib.AC_MODE_NONE))
        return model.linear(z, hidden, _lib.AC_MODE_NONE)

    t = genconv(model.linear(x, hidden, _lib.AC_MODE_NONE))
    for _ in range(2, int(depth) + 1):
        t = model.add(t, genconv(model.dropout(norm_relu(t), dropout_rate)))
    logits = model.linear(model.dropout(norm_relu(t), dropout_rate), layers[-1], _lib.AC_MODE_NONE)
    _loss(model, loss, logits, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": logits, "aggs": aggs, "temperatures": temps,
            "bns": bns}


def build_gcn_weighted(model, layers, dropout_rate, edge_weights, edge_grad=False, lr=0.01, weight_decay=0.05,
                       features="float32", aggregation="float32", loss="softmax", norm=None):
    """GCN with edge weights (e.g. datasets.gcn_edge_weights, which folds in the symmetric normalisation).  Per layer

        t = relu(scatter_gather(linear(dropout(t), layers[i]), weights=e))     # no relu on the last layer

    with one edge tensor e shared by every layer.  edge_weights: one fp32 value per edge in CSR order, loaded after
    init().  edge_grad: compute e's gradient in backward (the sum of the layers' contributions).  Single partition.
    aggregation="bfloat16" stores each linear output the scatter_gather reads in bf16 (Model.set_bf16_aggregation).
    norm="batch" / "layer_norm": batch_norm / layer_norm on t before each hidden relu (see build_gcn).  Returns the handles, with `edges` and the
    aggregations' inputs `sg_ins` and outputs `sg_outs`."""
    _check_norm(norm)
    L = len(layers)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    e = model.create_edge_tensor(1)
    t = x
    sg_ins, sg_outs, bns = [], [], []
    for i in range(1, L):
        t = model.linear(model.dropout(t, dropout_rate), layers[i], _lib.AC_MODE_NONE)
        sg_ins.append(t)
        t = model.scatter_gather(t, weights=e)
        sg_outs.append(t)
        if i != L - 1:
            t = model.relu(_hidden_norm(model, norm, t, bns))
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    model.set_edge_grad(e, edge_grad)
    _aggregation(model, aggregation)
    model.init()
    model.set_tensor(e, np.asarray(edge_weights, dtype=np.float32))
    return {"input": x, "label": label, "mask": mask, "logits": t, "edges": e, "sg_ins": sg_ins, "sg_outs": sg_outs,
            "bns": bns}


def _check_count(v, name):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
        raise ValueError("%s must be an integer >= 1" % name)


def _check_alpha(alpha):
    if not (isinstance(alpha, (int, float, np.floating)) and 0.0 <= float(alpha) <= 1.0):
        raise ValueError("alpha must be in [0, 1]")


def fp32(x):
    """x (computed in double) rounded once to fp32, as the builders pass their coefficients to scaled_add."""
    return float(np.float32(x))


def build_appnp(model, layers, dropout_rate, K=10, alpha=0.1, lr=0.01, weight_decay=0.05, exact_backward=False,
                features="float32", loss="softmax", edge_dropout=0.0):
    """APPNP (Klicpera et al., 2019), PyG's APPNP after an MLP:

        h = MLP(x)                     # per layer: dropout -> linear -> relu, no relu on the last layer
        z = h
        z = scaled_add(indegree_norm(scatter_gather(indegree_norm(z))), h, 1 - alpha, alpha)     # K times
        loss(z)

    i.e. z' = (1 - alpha) D^-1/2 A D^-1/2 z + alpha h with the self loops already in A.  The coefficients are computed
    in double and rounded to fp32 once (fp32()).  With fusion on, each hop's scaled_add is fused into its
    scatter_gather's store, and so is the next hop's first indegree_norm (Model.init); one partition for the fusion.
    edge_dropout > 0 is the paper's (and PyG APPNP(dropout=)'s) dropout of the propagation matrix: every hop's
    scatter_gather drops its in-edges at that rate in train mode (Model.scatter_gather(dropout=)), each hop and step
    drawing its own mask, with the degrees of the full graph; the fusions still apply.  0 builds the model without it.
    Bad K, alpha or edge_dropout raises ValueError.  Returns the handles, with `h` (the MLP output), `hops` (each
    hop's z) and `coefficients` (the fp32 pair (1 - alpha, alpha)).  With fusion on, a hop's z before the last is never
    written (its scatter_gather stores the next hop's normalised z instead), so only the last, the logits, can be read
    after a forward; set_fusion(False) writes every hop's z."""
    _check_count(K, "K")
    _check_alpha(alpha)
    _check_rate(dropout_rate, "dropout_rate")
    _check_rate(edge_dropout, "edge_dropout")
    c = (fp32(1.0 - float(alpha)), fp32(float(alpha)))
    L = len(layers)
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    t = x
    for i in range(1, L):
        t = model.linear(model.dropout(t, dropout_rate), layers[i], _lib.AC_MODE_NONE)
        if i != L - 1:
            t = model.relu(t)
    h = z = t
    hops = []
    for _ in range(int(K)):
        z = model.indegree_norm(_sum_gather(model, model.indegree_norm(z), edge_dropout))
        z = model.scaled_add(z, h, c[0], c[1])
        hops.append(z)
    _loss(model, loss, z, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": z, "h": h, "hops": hops, "coefficients": c}


def gcnii_beta(theta, layer):
    """GCNII's identity-mapping strength of layer `layer` (1-based): log(theta / layer + 1), in double."""
    return math.log(float(theta) / layer + 1.0)


def build_gcnii(model, layers, dropout_rate, depth, alpha=0.1, theta=0.5, lr=0.01, weight_decay=0.05,
                exact_backward=False, features="float32", loss="softmax"):
    """GCNII (Chen et al., 2020), PyG's gcn2_cora example with shared weights; layers = [in, hidden, out]:

        x0 = relu(linear(dropout(x), hidden))
        h  = x0
        for l in 1 .. depth:
            p = scaled_add(indegree_norm(scatter_gather(indegree_norm(dropout(h)))), x0, 1 - alpha, alpha)
            h = relu(scaled_add(p, linear(p, hidden), 1 - beta_l, beta_l))       # beta_l = log(theta / l + 1)
        logits = linear(dropout(h), out)

    The coefficients are computed in double and rounded to fp32 once (fp32(), gcnii_beta()).  With fusion on, each
    hop's first scaled_add is fused into its scatter_gather's store.  One weight decay for every weight (PyG's example
    uses two).  Bad layers, depth, alpha or theta raise ValueError.  Returns the handles, with `x0`, `hops` (each
    layer's p), `relu_outs` (each layer's h) and `coefficients` (the fp32 (1 - alpha, alpha) and, per layer, the fp32
    (1 - beta_l, beta_l))."""
    if len(layers) != 3:
        raise ValueError("layers must be [in, hidden, out]")
    _check_count(depth, "depth")
    _check_alpha(alpha)
    if not (isinstance(theta, (int, float, np.floating)) and math.isfinite(float(theta)) and float(theta) > 0.0):
        raise ValueError("theta must be finite and > 0")
    _check_rate(dropout_rate, "dropout_rate")
    ca = (fp32(1.0 - float(alpha)), fp32(float(alpha)))
    cb = [(fp32(1.0 - gcnii_beta(theta, l)), fp32(gcnii_beta(theta, l))) for l in range(1, int(depth) + 1)]
    x = _input_tensor(model, layers[0], features)
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    x0 = h = model.relu(model.linear(model.dropout(x, dropout_rate), layers[1], _lib.AC_MODE_NONE))
    hops, relu_outs = [], []
    for l in range(int(depth)):
        z = model.indegree_norm(model.scatter_gather(model.indegree_norm(model.dropout(h, dropout_rate))))
        p = model.scaled_add(z, x0, ca[0], ca[1])
        hops.append(p)
        h = model.relu(model.scaled_add(p, model.linear(p, layers[1], _lib.AC_MODE_NONE), cb[l][0], cb[l][1]))
        relu_outs.append(h)
    t = model.linear(model.dropout(h, dropout_rate), layers[2], _lib.AC_MODE_NONE)
    _loss(model, loss, t, label, mask)
    model.adam(lr, weight_decay)
    if exact_backward:
        model.set_exact_backward(True)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t, "x0": x0, "hops": hops, "relu_outs": relu_outs,
            "coefficients": {"alpha": ca, "beta": cb}}
