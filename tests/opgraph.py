"""An op-graph recorder over roc_b200.model.Model and an fp64 interpreter of what it recorded.

Recorder(model) offers every builder method of the Model with the same signatures.  Each call goes to the product,
and the recorder appends one IR node per layer the product creates (scatter_gather(t, AGGR_AVG) appends three: the sum
and two norms), numbered by layer index as Model::layers is.  A node is a dict:

    kind    one of roc_b200._lib.HOST_OPS: "linear", "indegree_norm", "scatter_gather", "scatter_gather_max",
            "scatter_gather_min", "scatter_gather_weighted", "attention_gather", "attention_scores", "relu", "elu",
            "sigmoid", "add", "scaled_add", "dropout", "batch_norm", "softmax_cross_entropy" or "sigmoid_cross_entropy";
            or "layer_norm", which op_info reports as "batch_norm" (the normalisation kind)
    ins     input tensor ids (tensor handles; the inner tensors of AGGR_AVG get ids of their own, from INNER on)
    out     output tensor id (None for a loss)
    layer   the layer index
    attrs   out_dim, activation, param (linear); rate, seed, key (dropout); aggr, and dropout, seed, key for a sum with
            edge dropout (scatter_gather); mode (attention_gather: "gat", "dynamic", "softmax" or "dot"), then per mode
            heads, slope, dropout, seed, key (gat: ins [t, scores]); heads, slope, param (dynamic: ins [xl, xr], the
            parameter a); temperature, learn, param (softmax: ins [x], param the learned t or None); heads, scale
            (dot: ins [q, k, v]); heads, param (attention_scores); edges (weighted); alpha, beta (scaled_add, the fp32
            coefficients as doubles); gamma, beta (parameter indices), momentum, eps (batch_norm); gamma, beta, eps
            (layer_norm).  Every fp32 attribute (slope, temperature, scale, eps) is held as the fp32 value, as a double.

A dropout's, an attention_gather's and a dropped sum's Philox key is (seed << 32) | layer, as Model::dropout computes
it.  Parameters are numbered in the product's order: a Linear's W, attention_scores' A, a dynamic gather's a, a
learned temperature, a norm's gamma then beta.  The recorder also keeps the bf16 leaves
(create_node_tensor(dtype="bfloat16")) and whether set_bf16_aggregation is on.

witness() runs the recorded graph in torch fp64 with autograd over edge lists (index_add): no code shared with the
product.  The op semantics are the ones include/roc_b200.h and include/roc_gnn.h state; the newer aggregations take
their per-edge math from the feature witnesses (gatv2_witness, softmax_aggr_witness, transformer_witness and
edge_dropout_witness's keep bits), which are test code too."""
import numpy as np
import torch

import attn_dropout_oracle as ado
import edge_dropout_witness as edw
from gatv2_witness import dynamic_attend
from oracle import oracle
from roc_b200 import _lib
from softmax_aggr_witness import softmax_aggr
from transformer_witness import dot_attend
from witness_gat import attend, edge_lists, train_loss

INNER = 1 << 20      # ids of tensors the caller holds no handle for
LOSSES = ("softmax_cross_entropy", "sigmoid_cross_entropy")


class Recorder:
    """model: a roc_b200.model.Model, or None to write an IR by hand (tensor ids are then handed out here)."""

    def __init__(self, model=None):
        self.m = model
        self._next = 0
        self.nodes = []
        self.width = {}           # tensor id -> hidden width
        self.leaves = []          # float node tensors the script created, in order
        self.bf16 = set()         # the leaves held in bf16
        self.edges = []           # edge tensors
        self.edge_grad = {}       # edge tensor -> set_edge_grad's last value
        self.exact = False
        self.bf16_aggregation = False
        self.params = 0
        self._inner = INNER

    def _call(self, name, *args):
        if self.m is not None:
            return getattr(self.m, name)(*args)
        self._next += 1
        return self._next - 1

    def _node(self, kind, ins, out, width=None, **attrs):
        n = dict(kind=kind, ins=list(ins), out=out, layer=len(self.nodes), attrs=attrs)
        self.nodes.append(n)
        if out is not None:
            self.width[out] = width if width is not None else self.width[ins[0]]
        return out

    # ---- builders (roc_b200.model.Model)
    def create_node_tensor(self, hidden, is_int=False, dtype="float32"):
        bf16 = dtype in ("bfloat16", "bf16")
        t = self._call("create_node_tensor", hidden, is_int, dtype) if bf16 else \
            self._call("create_node_tensor", hidden, is_int)
        self.width[t] = hidden
        if not is_int:
            self.leaves.append(t)
        if bf16:
            self.bf16.add(t)
        return t

    def create_edge_tensor(self, hidden=1):
        e = self._call("create_edge_tensor", hidden)
        self.edges.append(e)
        self.edge_grad[e] = False
        return e

    def set_edge_grad(self, edges, on=True):
        self._call("set_edge_grad", edges, on)
        self.edge_grad[edges] = bool(on)

    def set_exact_backward(self, on=True):
        self._call("set_exact_backward", on)
        self.exact = bool(on)

    def set_bf16_aggregation(self, on=True):
        self._call("set_bf16_aggregation", on)
        self.bf16_aggregation = bool(on)

    def _key(self, seed):
        # Model::dropout / Model::attention_gather: opIndex = the layer index; the Philox key is (seed << 32) | opIndex
        return ((seed & 0xFFFFFFFF) << 32) | len(self.nodes)

    def dropout(self, t, rate, seed=0):
        key = self._key(seed)
        return self._node("dropout", [t], self._call("dropout", t, rate, seed), rate=float(rate), seed=seed, key=key)

    def linear(self, t, out_dim, activation=_lib.AC_MODE_NONE):
        self.params += 1
        return self._node("linear", [t], self._call("linear", t, out_dim, activation), width=out_dim, out_dim=out_dim,
                          activation=activation, param=self.params - 1)

    def indegree_norm(self, t):
        return self._node("indegree_norm", [t], self._call("indegree_norm", t))

    def scatter_gather(self, t, aggr=_lib.AGGR_SUM, weights=None, dropout=0.0, seed=0):
        if dropout:                        # Model::scatter_gather with edge dropout: one sum, keyed by its layer
            key = self._key(seed)
            return self._node("scatter_gather", [t], self._call("scatter_gather", t, aggr, weights, dropout, seed),
                              aggr=aggr, dropout=float(dropout), seed=seed, key=key)
        out = self._call("scatter_gather", t, aggr, weights)
        if weights is not None:
            return self._node("scatter_gather_weighted", [t, weights], out, edges=weights)
        if aggr == _lib.AGGR_AVG:          # Model::scatter_gather: indegree_norm(indegree_norm(scatter_gather(t)))
            a, b = self._inner, self._inner + 1
            self._inner += 2
            self._node("scatter_gather", [t], a, width=self.width[t], aggr=_lib.AGGR_SUM)
            self._node("indegree_norm", [a], b)
            return self._node("indegree_norm", [b], out)
        kind = {_lib.AGGR_SUM: "scatter_gather", _lib.AGGR_MAX: "scatter_gather_max",
                _lib.AGGR_MIN: "scatter_gather_min"}[aggr]
        return self._node(kind, [t], out, aggr=aggr)

    def attention_gather(self, t, scores, heads=1, negative_slope=0.2, dropout=0.0, seed=0):
        key = self._key(seed)
        # the rate-0 call takes the four arguments Model.attention_gather has always taken
        args = (t, scores, heads, negative_slope) + ((dropout, seed) if dropout or seed else ())
        return self._node("attention_gather", [t, scores], self._call("attention_gather", *args), width=self.width[t],
                          mode="gat", heads=int(heads), slope=float(np.float32(negative_slope)),
                          dropout=float(dropout), seed=seed, key=key)

    def dynamic_attention_gather(self, xl, xr, heads=1, negative_slope=0.2):
        self.params += 1
        return self._node("attention_gather", [xl, xr],
                          self._call("dynamic_attention_gather", xl, xr, heads, negative_slope), mode="dynamic",
                          heads=int(heads), slope=float(np.float32(negative_slope)), param=self.params - 1)

    def softmax_gather(self, t, temperature=1.0, learn_temperature=False):
        if learn_temperature:
            self.params += 1
        return self._node("attention_gather", [t], self._call("softmax_gather", t, temperature, learn_temperature),
                          mode="softmax", temperature=float(np.float32(temperature)), learn=bool(learn_temperature),
                          param=self.params - 1 if learn_temperature else None)

    def dot_attention_gather(self, q, k, v, heads=1, scale=None):
        if scale is None:                  # Model.dot_attention_gather's default, from this recorder's widths
            scale = float(np.float32(1.0 / np.sqrt(max(self.width[q] // int(heads), 1))))
        return self._node("attention_gather", [q, k, v], self._call("dot_attention_gather", q, k, v, heads, scale),
                          mode="dot", heads=int(heads), scale=float(np.float32(scale)))

    def attention_scores(self, t, heads=1):
        self.params += 1
        return self._node("attention_scores", [t], self._call("attention_scores", t, heads), width=2 * int(heads),
                          heads=int(heads), param=self.params - 1)

    def relu(self, t):
        return self._node("relu", [t], self._call("relu", t))

    def elu(self, t):
        return self._node("elu", [t], self._call("elu", t))

    def sigmoid(self, t):
        return self._node("sigmoid", [t], self._call("sigmoid", t))

    def add(self, a, b):
        return self._node("add", [a, b], self._call("add", a, b))

    def scaled_add(self, a, b, alpha, beta):
        return self._node("scaled_add", [a, b], self._call("scaled_add", a, b, alpha, beta),
                          alpha=float(np.float32(alpha)), beta=float(np.float32(beta)))

    def batch_norm(self, t, momentum=0.1, eps=1e-5):
        self.params += 2
        return self._node("batch_norm", [t], self._call("batch_norm", t, momentum, eps), gamma=self.params - 2,
                          beta=self.params - 1, momentum=float(momentum), eps=float(np.float32(eps)))

    def layer_norm(self, t, eps=1e-5):
        self.params += 2
        return self._node("layer_norm", [t], self._call("layer_norm", t, eps), gamma=self.params - 2,
                          beta=self.params - 1, eps=float(np.float32(eps)))

    def softmax_cross_entropy(self, logits, labels, mask):
        self._call("softmax_cross_entropy", logits, labels, mask)
        return self._node("softmax_cross_entropy", [logits, labels, mask], None)

    def sigmoid_cross_entropy(self, logits, labels, mask):
        self._call("sigmoid_cross_entropy", logits, labels, mask)
        return self._node("sigmoid_cross_entropy", [logits, labels, mask], None)

    def init(self):
        if self.m is not None:
            self.m.init()
            self.check_against_product()

    def num_parameters(self):
        return self.params if self.m is None else self.m.num_parameters()

    def __getattr__(self, name):          # adam, set_fusion, set_tensor, forward, ...: straight to the product
        if self.m is None:                # a hand-written IR: nothing to run
            return lambda *args, **kw: None
        return getattr(self.m, name)

    def check_against_product(self):
        """The product's layer list matches the recorded one, kind by kind (a layer_norm reports as batch_norm, the
        normalisation kind)."""
        got = [i["kind"] for i in self.m.op_info()]
        want = ["batch_norm" if n["kind"] == "layer_norm" else n["kind"] for n in self.nodes]
        assert got == want, (got, want)
        assert self.m.num_parameters() == self.params, (self.m.num_parameters(), self.params)

    # ---- what the IR implies
    def loss_node(self):
        losses = [n for n in self.nodes if n["kind"] in LOSSES]
        assert len(losses) == 1, "one loss"
        return losses[0]


def bce_train_loss(logits, labels, mask):
    """The sigmoid loss in fp64: binary cross-entropy summed over the train rows and every class.
    labels: [N][C] 0/1."""
    train = torch.from_numpy(np.asarray(mask) == _lib.MASK_TRAIN)
    y = torch.from_numpy(np.asarray(labels, dtype=np.float64))
    return torch.nn.functional.binary_cross_entropy_with_logits(logits[train], y[train], reduction="sum")


def _relu_with_mask(pre, product_mask, what):
    """ReLU whose mask is the product's where fp32 and fp64 disagree at a pre-activation within rounding of 0.
    product_mask: a bool array or tensor (moved to pre's device).  The result saves a bool mask for autograd, not a
    float one, so that tests/scale_witness.py can use it at full size."""
    if product_mask is None:
        return torch.relu(pre)
    p = pre.detach()
    pm = torch.as_tensor(product_mask).to(p.device, torch.bool)
    diff = (p > 0) != pm
    if diff.any():
        assert p[diff].abs().max() <= 1e-4 * p.abs().max(), "%s: relu masks differ away from zero" % what
    return torch.where(pm, pre, 0.0)


def _extreme_sources(row_end, col, x, is_max, product_args, what):
    """[N][H] sources of the first extreme in CSR order, or the product's choice where the candidates tie to 1e-5."""
    n, h = row_end.shape[0], x.shape[1]
    out = np.zeros((n, h), dtype=np.int64)
    s = 0
    for v in range(n):
        e = int(row_end[v])
        if e > s:
            vals = x[col[s:e]]
            k = np.argmax(vals, axis=0) if is_max else np.argmin(vals, axis=0)
            out[v] = col[s:e][k]
        s = e
    if product_args is not None:
        pa = product_args.astype(np.int64)
        diff = pa != out
        if diff.any():
            cols = np.nonzero(diff)[1]
            a, b = x[pa[diff], cols], x[out[diff], cols]
            assert np.abs(a - b).max() <= 1e-5 * np.abs(x).max(), "%s: max / min choice differs away from a tie" % what
        out = pa
    return out


def witness(ir, graph, feats, labels, mask, weights, edge_values=None, step=1, relu_masks=None, aggr_args=None,
            training=True, run_stats=None, rounded=None):
    """The recorded graph (a Recorder) in torch fp64 with autograd, for one training step.

    graph: (row_end, col).  feats: {leaf id: [N][H] array} (one array: the first leaf); a bf16 leaf is read as its
    bf16 rounding.  labels: [N] class indices (softmax loss) or [N][C] 0/1 (sigmoid loss).  mask: [N] MASK_*.
    weights: W_mem[o][i] per parameter (a batch_norm's gamma / beta as (1, H)).  edge_values: {edge tensor: [E]
    weights}.  step: the product's train-step counter during this step's forward (Model::forward increments it before
    the first op, so the first step is 1).  relu_masks / aggr_args: {layer: the product's relu output > 0 /
    get_aggr_index}, taken where fp32 and fp64 tie.  rounded: {tensor: the product's values of a tensor it stores in
    bf16 (set_bf16_aggregation)}, each checked to be a rounding of the fp64 value and taken in the forward with the
    gradient passed straight through.

    training=False is the infer-mode model: dropout, attention dropout and edge dropout are copies, batch_norm uses
    run_stats {bn output: (running mean, running variance)}, and nothing is differentiated.

    Returns dict(logits, dW (zeros for a parameter off the loss's path), edge_grad {edge tensor: dL/dw}, pre {layer: the
    ReLU pre-activation}, stats {bn output: its batch (mean, biased variance)})."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    relu_masks, aggr_args, rounded = relu_masks or {}, aggr_args or {}, rounded or {}
    if not isinstance(feats, dict):
        feats = {ir.leaves[0]: feats}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(training) for w in weights]
    ew = {e: torch.from_numpy(np.asarray(v, dtype=np.float64)).requires_grad_(training)
          for e, v in (edge_values or {}).items()}
    val = {t: torch.from_numpy(np.asarray(a, dtype=np.float64)) for t, a in feats.items()}
    for t in ir.bf16 & set(val):                 # the fp32 rows as the product stores them: rounded to nearest even
        val[t] = val[t].float().bfloat16().double()
    pre, stats, loss, logits = {}, {}, None, None
    for node in ir.nodes:
        k, a, ins, what = node["kind"], node["attrs"], node["ins"], "layer %d (%s)" % (node["layer"], node["kind"])
        x = val[ins[0]] if ins[0] in val else None
        if k == "linear":
            y = x @ ws[a["param"]].T
            if a["activation"] == _lib.AC_MODE_RELU:
                pre[node["layer"]] = y.detach().numpy()
                y = _relu_with_mask(y, relu_masks.get(node["layer"]), what)
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            rows = x[src]
            if training and a.get("dropout", 0.0) > 0:
                keep = edw.edge_keep(row_end, col, a["dropout"], a["key"], step)
                rows = rows * torch.from_numpy(keep.astype(np.float64) * edw.drop_scale(a["dropout"])).unsqueeze(1)
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, rows)
        elif k in ("scatter_gather_max", "scatter_gather_min"):
            s = _extreme_sources(row_end, col, x.detach().numpy(), k.endswith("max"), aggr_args.get(node["layer"]),
                                 what)
            y = x.gather(0, torch.from_numpy(s))
        elif k == "scatter_gather_weighted":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, ew[a["edges"]][:, None] * x[src])
        elif k == "attention_gather" and a["mode"] == "dynamic":
            y = dynamic_attend(x, val[ins[1]], ws[a["param"]].T, dst, src, n, a["heads"], a["slope"])[0]
        elif k == "attention_gather" and a["mode"] == "softmax":
            t = ws[a["param"]][0, 0] if a["learn"] else torch.tensor(a["temperature"], dtype=torch.float64)
            y = softmax_aggr(x, t, dst, src, n)[0]
        elif k == "attention_gather" and a["mode"] == "dot":
            y = dot_attend(x, val[ins[1]], val[ins[2]], dst, src, n, a["heads"], a["scale"])[0]
        elif k == "attention_gather":
            drop = None
            if training and a.get("dropout", 0.0) > 0:
                drop = ado.multipliers(ado.edge_keep(row_end, col, a["dropout"], a["key"], step), a["heads"],
                                       a["dropout"])
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"], drop)
        elif k == "attention_scores":
            hd, w = a["heads"], ws[a["param"]]
            xv = x.reshape(n, hd, -1)
            y = torch.cat([(xv * w[:hd]).sum(2), (xv * w[hd:]).sum(2)], 1)
        elif k == "relu":
            pre[node["layer"]] = x.detach().numpy()
            y = _relu_with_mask(x, relu_masks.get(node["layer"]), what)
        elif k == "elu":
            y = torch.nn.functional.elu(x)
        elif k == "sigmoid":
            y = torch.sigmoid(x)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "scaled_add":
            y = a["alpha"] * x + a["beta"] * val[ins[1]]
        elif k == "batch_norm":
            gam, bet = ws[a["gamma"]][0], ws[a["beta"]][0]
            if training:
                mean = x.detach().mean(0)
                stats[node["out"]] = (mean.numpy(), ((x.detach() - mean) ** 2).mean(0).numpy())
                y = torch.nn.functional.batch_norm(x, None, None, gam, bet, training=True, eps=a["eps"])
            else:
                rm, rv = (torch.from_numpy(np.asarray(v, dtype=np.float64)) for v in run_stats[node["out"]])
                y = torch.nn.functional.batch_norm(x, rm, rv, gam, bet, training=False, eps=a["eps"])
        elif k == "layer_norm":
            y = torch.nn.functional.layer_norm(x, (x.shape[1],), ws[a["gamma"]][0], ws[a["beta"]][0], a["eps"])
        elif k == "dropout":
            if a["rate"] > 0 and training:
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
                y = x * torch.from_numpy(keep.astype(np.float64) * scale)
            else:
                y = x
        elif k in LOSSES:
            logits = x
            if training:
                f = train_loss if k == "softmax_cross_entropy" else bce_train_loss
                loss = f(x, np.asarray(labels), np.asarray(mask))
            continue
        else:
            raise AssertionError("unknown op " + k)
        if node["out"] in rounded:
            r, p = torch.from_numpy(np.asarray(rounded[node["out"]], dtype=np.float64)), y.detach()
            assert ((r - p).abs() <= 2.0 ** -8 * 1.001 * p.abs() + 1e-5 * p.abs().max()).all(), \
                "%s: the product's bf16 value is not a rounding of the fp64 one" % what
            y = y + (r - p)
        val[node["out"]] = y
    if loss is not None and loss.requires_grad:      # else no parameter reaches the loss
        loss.backward()
    return dict(logits=logits.detach().numpy(),
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws],
                edge_grad={e: (t.grad.numpy() if t.grad is not None else np.zeros(t.shape)) for e, t in ew.items()},
                pre=pre, stats=stats)
