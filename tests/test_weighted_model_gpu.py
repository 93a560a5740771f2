"""The weighted GCN (build_gcn_weighted: dropout -> linear -> scatter_gather(., weights=e) -> relu, one edge tensor
shared by every layer) against a torch fp64 autograd witness on a small directed, weighted graph with duplicate edges:
logits, every dW and the edge tensor's gradient, over several Adam steps.  Then the edge gradient's opt-in, and the
refusals of the Model layer."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, rel_close
from roc_b200 import datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gcn_weighted
from witness_weighted import gcn_weighted_witness

pytestmark = pytest.mark.gpu
WSUM, EDOT = 8, 9


def directed_case(layers, n=300, e=2500, seed=5):
    rng = np.random.RandomState(seed)
    dst = np.sort(rng.randint(0, n, size=e))
    src = rng.randint(0, n, size=e)
    src[1::4] = src[0::4][:src[1::4].shape[0]]              # duplicate edges where dst repeats
    dst[:150] = 7                                           # a heavy row
    dst = np.sort(dst)
    order = np.lexsort((src, dst))
    row_end = np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64)
    col = src[order].astype(np.uint32)
    w = datasets.gcn_edge_weights(row_end, col, rng.uniform(0.2, 3.0, size=e))
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=seed)
    return row_end, col, w, feats.numpy(), labels.numpy(), mask.numpy()


def build(case, layers, edge_grad, dropout=0.0):
    row_end, col, w, feats, labels, mask = case
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    hd = build_gcn_weighted(m, list(layers), dropout, w, edge_grad=edge_grad)
    m.set_tensor(hd["input"], feats)
    m.set_labels(hd["label"], labels)
    m.set_tensor(hd["mask"], mask.astype(np.int32))
    return host, m, hd


@pytest.mark.parametrize("layers", [(12, 16, 5), (12, 32, 16, 5)])
def test_weighted_gcn_against_torch_fp64_witness(layers):
    """Each of three Adam steps: logits, dW and the shared edge tensor's gradient (the sum over the layers, never
    including the previous step's) match the witness evaluated at that step's weights."""
    case = directed_case(layers)
    row_end, col, w, feats, labels, mask = case
    host, m, hd = build(case, layers, edge_grad=True)
    assert m.tensor_shape(hd["edges"]) == (col.shape[0], 1, 1)
    for step in range(3):
        w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
        m.train_mode(); m.zero_gradients(); m.forward()
        logits = m.get_tensor(hd["logits"])
        m.backward()
        dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        dedge = m.get_tensor(hd["edges"], grad=True)[:, 0]
        m.update()
        wl, wdw, wde = gcn_weighted_witness(row_end, col, feats, labels, mask, layers, w0, w)
        what = "step %d" % step
        rel_close(logits, wl, what=what + " logits vs torch fp64")
        for p, (a, b) in enumerate(zip(dw, wdw)):
            rel_close(a, b, rtol=2e-4, atol_scale=2e-5, what=what + " dW[%d] vs torch autograd" % p)
        rel_close(dedge, wde, rtol=2e-4, atol_scale=2e-5, what=what + " edge gradient vs torch autograd")
    np.testing.assert_array_equal(m.get_tensor(hd["edges"])[:, 0], w)     # no optimizer touches the edge tensor
    host.close()


def test_edge_grad_off_leaves_the_gradient_and_launches_no_edge_dot():
    layers = (12, 16, 5)
    case = directed_case(layers)
    host, m, hd = build(case, layers, edge_grad=False)
    e = hd["edges"]
    sentinel = np.full((case[1].shape[0],), -7.25, dtype=np.float32)
    m.set_tensor(e, sentinel, grad=True)
    m.train_mode(); m.zero_gradients(); m.forward(); m.backward()
    host.synchronize()
    # the first layer's aggregation runs backward last: its last ScatterGather call is the input gradient's
    reds = [l["red"] for l in K.sg_launches()]
    assert EDOT not in reds and WSUM in reds and K.sg_launches()[0]["kind"] == "permute"
    np.testing.assert_array_equal(m.get_tensor(e, grad=True)[:, 0], sentinel)
    # switched on (the aggregations' inputs have gradients of their own, so this may follow init): the last call is
    # the edge dot, and the sentinel is overwritten
    m.set_edge_grad(e, True)
    m.train_mode(); m.zero_gradients(); m.forward(); m.backward()
    host.synchronize()
    assert [l["red"] for l in K.sg_launches() if l["kind"] == "main"] == [EDOT]
    assert not (m.get_tensor(e, grad=True)[:, 0] == sentinel).any()
    host.close()


def run_prog(lines):
    prog = "\n".join(["import sys; sys.path.insert(0, %r)" % ROOT, "import numpy as np",
                      "from roc_b200.model import Host, Model, build_gcn_weighted"] + lines)
    return subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                          env=dict(os.environ))


def test_weighted_scatter_gather_refuses_more_than_one_partition():
    p = run_prog(["host = Host(0, 0, 2)",
                  "host.graph_from_arrays(np.array([2, 4, 6, 8], dtype=np.uint64), "
                  "np.array([0, 1, 0, 1, 2, 3, 2, 3], dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "x = m.create_node_tensor(4)",
                  "m.scatter_gather(x, weights=m.create_edge_tensor(1))",
                  "print('built')"])
    assert p.returncode != 0 and "built" not in p.stdout
    assert "one partition only" in p.stderr, p.stderr[-2000:]


def test_edge_tensor_refuses_more_than_one_value_per_edge():
    p = run_prog(["host = Host(0, 0, 1)",
                  "host.graph_from_arrays(np.array([2, 4], dtype=np.uint64), np.array([0, 1, 0, 1], dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "m.create_edge_tensor(2)",
                  "print('built')"])
    assert p.returncode != 0 and "built" not in p.stdout
    assert "numHidden == 1" in p.stderr, p.stderr[-2000:]
