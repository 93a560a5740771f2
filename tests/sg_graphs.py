"""The graphs the ScatterGather GPU tests run on, and their upload to the device."""
import numpy as np
import torch

from roc_b200 import datasets


def to_dev(row_end, col):
    return (torch.from_numpy(np.asarray(row_end).astype(np.int64)).to("cuda"),
            torch.from_numpy(np.asarray(col).astype(np.int32)).to("cuda"))


def graph(kind):
    if kind == "uniform":
        re, col = datasets.uniform_graph(1000, 4500, seed=1)
    elif kind == "rmat":
        re, col = datasets.rmat_graph(12, 40000, seed=3)           # hubs with degree >> 64
    elif kind == "dense":
        re, col = datasets.powerlaw_graph(600, 60000, seed=4)      # mean degree ~150: every row heavy
    elif kind == "ragged":
        # empty rows, a 1-edge graph tail, one 5000-edge row
        deg = np.zeros(400, dtype=np.int64)
        deg[3] = 5000; deg[10:200:7] = 1; deg[250] = 63; deg[251] = 64; deg[252] = 65; deg[399] = 2
        re = torch.from_numpy(np.cumsum(deg))
        col = torch.from_numpy(np.random.RandomState(9).randint(0, 400, size=int(deg.sum())).astype(np.int32))
    elif kind == "single":
        re, col = torch.tensor([1]), torch.tensor([0], dtype=torch.int32)
    else:
        raise KeyError(kind)
    return re.numpy().astype(np.uint64), col.numpy().astype(np.uint32)
