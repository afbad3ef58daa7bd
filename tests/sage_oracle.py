"""NumPy / fp64 reference of the max aggregation (pgcn_forward_max, pgcn_backward_max, op.PSpMMMax) and of the PSAGE
trainer (sage.py) — TEST INFRASTRUCTURE, the product never imports it.

max_aggregate takes each row's winner by numpy.argmax over the row's stored entries in CSR order: the first entry with
the largest value, NaN above every number. Z is copied from the winner, so it keeps its bits. intended_training routes
the gradient by gathering at the oracle's arg (the first winner); scatter_reduce("amax")'s autograd would split it over
tied entries instead.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pgat_oracle as po


def max_aggregate(rowptr, colidx, X):
    """(Z, arg): Z [rows, f] in X's dtype, arg [rows, f] int32 entry indices into colidx (-1 and Z = 0 for empty rows)."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    colidx = np.asarray(colidx, dtype=np.int64)
    rows = rowptr.shape[0] - 1
    f = X.shape[1]
    Z = np.zeros((rows, f), dtype=X.dtype)
    arg = np.full((rows, f), -1, dtype=np.int32)
    for i in range(rows):
        e0, e1 = rowptr[i], rowptr[i + 1]
        if e1 == e0:
            continue
        w = np.argmax(X[colidx[e0:e1]], axis=0)
        arg[i] = e0 + w
        Z[i] = X[colidx[e0 + w], np.arange(f)]
    return Z, arg


def max_backward(colidx, arg, gZ, ncols):
    """G [ncols, f] in fp64: gZ[i, c] summed into the column of the entry arg[i, c] names (arg < 0: nothing)."""
    colidx = np.asarray(colidx, dtype=np.int64)
    i, c = np.nonzero(arg >= 0)
    G = np.zeros((ncols, gZ.shape[1]))
    np.add.at(G, (colidx[arg[i, c]], c), gZ[i, c].astype(np.float64))
    return G


def init_params(nlayers, f, seed):
    """[(Wp, bp, Ws, Wn)] as sage.PSAGE draws them on the CPU after torch.manual_seed(seed): pool = Linear(f, f),
    self_lin and neigh_lin = Linear(f, f, bias=False), default initialisation. fp32 draws, returned as fp64 numpy."""
    torch.manual_seed(seed)
    out = []
    for _ in range(nlayers):
        pool = nn.Linear(f, f, bias=True)
        s = nn.Linear(f, f, bias=False)
        nb = nn.Linear(f, f, bias=False)
        out.append(tuple(t.detach().numpy().astype(np.float64) for t in (pool.weight, pool.bias, s.weight, nb.weight)))
    return out


def max_gather(rowptr, colidx, P):
    """The max aggregation of P (fp64 torch) as a differentiable gather at the oracle's arg."""
    _, arg = max_aggregate(rowptr, colidx, P.detach().numpy())
    valid = torch.from_numpy(arg >= 0)
    cols = torch.from_numpy(np.where(arg >= 0, np.asarray(colidx, dtype=np.int64)[np.maximum(arg, 0)], 0))
    return torch.where(valid, P.gather(0, cols), torch.zeros((), dtype=P.dtype))


def intended_forward(A, H, params):
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    C.sort_indices()
    X = torch.as_tensor(H, dtype=torch.float64)
    for p in params:
        Wp, bp, Ws, Wn = (torch.as_tensor(t, dtype=torch.float64) for t in p)
        P = F.relu(X @ Wp.T + bp)
        N = max_gather(C.indptr, C.indices, P)
        X = F.relu(X @ Ws.T + N @ Wn.T)
    return X


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3):
    """The loss curve sage.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    params = [tuple(torch.tensor(t, requires_grad=True) for t in p) for p in init_params(nlayers, f, seed)]
    return po.train(params, lambda ps: intended_forward(A, H, ps), n, f, k, epochs, lr)
