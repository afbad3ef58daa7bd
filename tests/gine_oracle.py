"""NumPy / fp64 reference of GINE's aggregation (pgcn_gine_*, op.PGINE) and of the PGINE trainer (gine.py) — TEST
INFRASTRUCTURE, the product never imports it.

For the entries e = (i, j) of a CSR, with pre = X[j] + E_e:
    Z[i]  = sum_row relu(pre)
    dE_e  = gZ[i] where pre > 0 or pre is NaN, else 0
    dX[j] = sum_col dE
`terms` computes these in fp64 and propagates a first-order bound of the kernels' fp32 error alongside: the rounded
add moves relu(pre) by at most u |pre| (relu is 1-Lipschitz, and round-to-nearest keeps the sign of a sum, so the mask
is the same in fp32 and fp64 and dE is exact), every sum of d terms d roundings of its sum|terms| (a split row's chunk
partials and their fixup add no more than that), and the reverse exchange's halo additions two more. The bound it
returns is twice that estimate.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from gatedgcn_oracle import entries, graph, _scatter
from oracle import pgat_oracle as po

EPS32 = 2.0 ** -24
BLOCK = 32       # features per block: bounds the [nnz, block] temporaries


def terms(rowptr, colidx, ncols, X, E, gZ=None):
    """Forward and, with gZ, backward of the CSR (rowptr over rows, colidx in [0, ncols)) on X [ncols, f], E [nnz, f]
    and gZ [rows, f]. Returns {name: (fp64 value, bound)}: "Z" ([rows, f]), and with gZ "dE" ([nnz, f], bound 0: the
    kernels give its bits) and "dX" ([ncols, f])."""
    rows, cols = entries(rowptr, colidx)
    nr, f, nnz = len(rowptr) - 1, X.shape[1], len(rows)
    R, Cm = _scatter(rows, nr, nnz), _scatter(cols, ncols, nnz)
    drow = np.diff(np.asarray(rowptr, np.int64))[:, None].astype(np.float64)
    dcol = np.bincount(cols, minlength=ncols)[:, None].astype(np.float64)
    names = ["Z"] + (["dE", "dX"] if gZ is not None else [])
    shapes = {"Z": nr, "dE": nnz, "dX": ncols}
    out = {k: (np.zeros((shapes[k], f)), np.zeros((shapes[k], f))) for k in names}
    u = EPS32
    for c0 in range(0, f, BLOCK):
        c = slice(c0, min(f, c0 + BLOCK))
        pre = X[cols, c].astype(np.float64) + E[:, c].astype(np.float64)
        msg = np.maximum(pre, 0.0)
        vals = {"Z": (R @ msg, R @ (u * np.abs(pre)) + drow * u * (R @ msg))}
        if gZ is not None:
            de = np.where(pre > 0, gZ[rows, c].astype(np.float64), 0.0)
            vals["dE"] = (de, 0.0 * de)
            vals["dX"] = (Cm @ de, (dcol + 2) * u * (Cm @ np.abs(de)))
        for k in names:
            out[k][0][:, c] = vals[k][0]
            out[k][1][:, c] = 2.0 * vals[k][1]
    return out


def fp32_reference(rowptr, colidx, ncols, X, E, gZ):
    """The kernels' formulas in fp32 with sums in entry order, relu and its mask by torch.relu's rules: where their
    results are NaN or +-inf, and dE's bits."""
    rows, cols = entries(rowptr, colidx)
    nr, f = len(rowptr) - 1, X.shape[1]
    with np.errstate(over="ignore", invalid="ignore"):
        pre = np.asarray(X, np.float32)[cols] + np.asarray(E, np.float32)
        msg = np.where(pre < 0, np.float32(0), pre)
        de = np.where(~(pre <= 0), np.asarray(gZ, np.float32)[rows], np.float32(0))

        def add(at, t, n):
            acc = np.zeros((n, f), np.float32)
            np.add.at(acc, at, t)
            return acc
        return {"Z": add(rows, msg, nr), "dE": de, "dX": add(cols, de, ncols)}


def torch_gine(rows, cols, m, X, E):
    """Z of the plain formula as a differentiable torch gather / relu / index_add (rows, cols int64 tensors)."""
    z = torch.zeros((m, X.shape[1]), dtype=X.dtype, device=X.device)
    return z.index_add(0, rows, torch.relu(X[cols] + E))


def init_params(nlayers, f, seed):
    """[layer] as gine.PGINE draws them on the CPU after torch.manual_seed(seed): per layer lin_edge Linear(1, f), then
    the MLP's Linear(f, f) twice, as (We, be, W0, b0, W2, b2). fp32 draws, returned as fp64 numpy."""
    torch.manual_seed(seed)
    layers = []
    for _ in range(nlayers):
        lins = [nn.Linear(1, f), nn.Linear(f, f), nn.Linear(f, f)]
        layers.append(tuple(t.detach().numpy().astype(np.float64) for lin in lins for t in (lin.weight, lin.bias)))
    return layers


def intended_forward(A, H, params, eps=0.0):
    """Logits of PGINE on the global graph A; H and params as numpy or fp64 tensors (params flat: each layer's six
    tensors)."""
    rows, cols, vals = graph(A)
    n = A.shape[0]
    t = [torch.as_tensor(x, dtype=torch.float64) for x in params]
    h = torch.as_tensor(H, dtype=torch.float64)
    e0 = vals[:, None]
    for l0 in range(0, len(t), 6):
        We, be, W0, b0, W2, b2 = t[l0:l0 + 6]
        Z = torch_gine(rows, cols, n, h, e0 @ We.T + be)
        x = (1 + eps) * h + Z
        h = h + F.relu(F.relu(x @ W0.T + b0) @ W2.T + b2)
    return h


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3):
    """The loss curve gine.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    flat = [torch.tensor(x, requires_grad=True) for p in init_params(nlayers, f, seed) for x in p]
    return po.train([tuple(flat)], lambda ps: intended_forward(A, H, ps[0]), n, f, k, epochs, lr)
