"""An op-graph recorder over roc_b200.model.Model and an fp64 interpreter of what it recorded.

Recorder(model) offers the Model's builder methods with the same signatures.  Each call goes to the product, and the
recorder appends one IR node per layer the product creates (scatter_gather(t, AGGR_AVG) appends three: the sum and two
norms), numbered by layer index as Model::layers is.  A node is a dict:

    kind    "linear", "indegree_norm", "scatter_gather", "scatter_gather_max", "scatter_gather_min",
            "scatter_gather_weighted", "attention_gather", "relu", "sigmoid", "add", "dropout" or
            "softmax_cross_entropy" (roc_b200._lib.HOST_OPS)
    ins     input tensor ids (tensor handles; the inner tensors of AGGR_AVG get ids of their own, from INNER on)
    out     output tensor id (None for the loss)
    layer   the layer index
    attrs   out_dim, activation, param (linear); rate, seed, key (dropout); heads, slope (attention); edges (weighted)

witness() runs the recorded graph in torch fp64 with autograd over edge lists (index_add): no code shared with the
product.  The op semantics are the ones include/roc_b200.h and include/roc_gnn.h state."""
import numpy as np
import torch

from oracle import oracle
from roc_b200 import _lib
from witness_gat import attend, edge_lists, train_loss

INNER = 1 << 20      # ids of tensors the caller holds no handle for


class Recorder:
    """model: a roc_b200.model.Model, or None to write an IR by hand (tensor ids are then handed out here)."""

    def __init__(self, model=None):
        self.m = model
        self._next = 0
        self.nodes = []
        self.width = {}           # tensor id -> hidden width
        self.leaves = []          # float node tensors the script created, in order
        self.edges = []           # edge tensors
        self.edge_grad = {}       # edge tensor -> set_edge_grad's last value
        self.exact = False
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
    def create_node_tensor(self, hidden, is_int=False):
        t = self._call("create_node_tensor", hidden, is_int)
        self.width[t] = hidden
        if not is_int:
            self.leaves.append(t)
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

    def dropout(self, t, rate, seed=0):
        layer = len(self.nodes)
        # Model::dropout: opIndex = the layer index; the Philox key is (seed << 32) | opIndex
        return self._node("dropout", [t], self._call("dropout", t, rate, seed), rate=float(rate), seed=seed,
                          key=((seed & 0xFFFFFFFF) << 32) | layer)

    def linear(self, t, out_dim, activation=_lib.AC_MODE_NONE):
        self.params += 1
        return self._node("linear", [t], self._call("linear", t, out_dim, activation), width=out_dim, out_dim=out_dim,
                          activation=activation, param=self.params - 1)

    def indegree_norm(self, t):
        return self._node("indegree_norm", [t], self._call("indegree_norm", t))

    def scatter_gather(self, t, aggr=_lib.AGGR_SUM, weights=None):
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

    def attention_gather(self, t, scores, heads=1, negative_slope=0.2):
        return self._node("attention_gather", [t, scores], self._call("attention_gather", t, scores, heads, negative_slope),
                          width=self.width[t], heads=int(heads), slope=float(np.float32(negative_slope)))

    def relu(self, t):
        return self._node("relu", [t], self._call("relu", t))

    def sigmoid(self, t):
        return self._node("sigmoid", [t], self._call("sigmoid", t))

    def add(self, a, b):
        return self._node("add", [a, b], self._call("add", a, b))

    def softmax_cross_entropy(self, logits, labels, mask):
        self._call("softmax_cross_entropy", logits, labels, mask)
        return self._node("softmax_cross_entropy", [logits, labels, mask], None)

    def init(self):
        if self.m is not None:
            self.m.init()
            self.check_against_product()

    def __getattr__(self, name):          # adam, set_fusion, set_tensor, forward, ...: straight to the product
        if self.m is None:                # a hand-written IR: nothing to run
            return lambda *args, **kw: None
        return getattr(self.m, name)

    def check_against_product(self):
        """The product's layer list matches the recorded one, kind by kind."""
        got = [i["kind"] for i in self.m.op_info()]
        assert got == [n["kind"] for n in self.nodes], (got, [n["kind"] for n in self.nodes])

    # ---- what the IR implies
    def loss_node(self):
        losses = [n for n in self.nodes if n["kind"] == "softmax_cross_entropy"]
        assert len(losses) == 1, "one loss"
        return losses[0]


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


def witness(ir, graph, feats, labels, mask, weights, edge_values=None, step=1, relu_masks=None, aggr_args=None):
    """The recorded graph (a Recorder) in torch fp64 with autograd, for one training step.

    graph: (row_end, col).  feats: {leaf id: [N][H] array} (one array: the first leaf).  labels: [N] class indices.
    mask: [N] MASK_*.  weights: W_mem[o][i] per parameter.  edge_values: {edge tensor: [E] weights}.  step: the
    product's train-step counter during this step's forward (Model::forward increments it before the first op, so the
    first step is 1).  relu_masks / aggr_args: {layer: the product's relu output > 0 / get_aggr_index}, taken where
    fp32 and fp64 tie.

    Returns dict(logits, dW (zeros for a Linear off the loss's path), edge_grad {edge tensor: dL/dw}, pre {layer: the
    ReLU pre-activation})."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    relu_masks, aggr_args = relu_masks or {}, aggr_args or {}
    if not isinstance(feats, dict):
        feats = {ir.leaves[0]: feats}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    ew = {e: torch.from_numpy(np.asarray(v, dtype=np.float64)).requires_grad_(True)
          for e, v in (edge_values or {}).items()}
    val = {t: torch.from_numpy(np.asarray(a, dtype=np.float64)) for t, a in feats.items()}
    pre, loss = {}, None
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
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, x[src])
        elif k in ("scatter_gather_max", "scatter_gather_min"):
            s = _extreme_sources(row_end, col, x.detach().numpy(), k.endswith("max"), aggr_args.get(node["layer"]),
                                 what)
            y = x.gather(0, torch.from_numpy(s))
        elif k == "scatter_gather_weighted":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, ew[a["edges"]][:, None] * x[src])
        elif k == "attention_gather":
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"])
        elif k == "relu":
            pre[node["layer"]] = x.detach().numpy()
            y = _relu_with_mask(x, relu_masks.get(node["layer"]), what)
        elif k == "sigmoid":
            y = torch.sigmoid(x)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "dropout":
            if a["rate"] > 0:
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
                y = x * torch.from_numpy(keep.astype(np.float64) * scale)
            else:
                y = x
        elif k == "softmax_cross_entropy":
            loss = train_loss(x, np.asarray(labels), np.asarray(mask))
            logits = x
            continue
        else:
            raise AssertionError("unknown op " + k)
        val[node["out"]] = y
    if loss.requires_grad:               # else no parameter reaches the loss
        loss.backward()
    return dict(logits=logits.detach().numpy(),
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws],
                edge_grad={e: (t.grad.numpy() if t.grad is not None else np.zeros(t.shape)) for e, t in ew.items()},
                pre=pre)
