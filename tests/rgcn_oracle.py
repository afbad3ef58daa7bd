"""NumPy / fp64 reference of R-GCN's relational aggregation (pgcn_rgcn_*, op.PRGCN) and of the PRGCN trainer (rgcn.py)
— TEST INFRASTRUCTURE, the product never imports it.

For the entries e = (i, j) of a CSR with relations rel_e in [0, R) and weights w_e, the virtual row v_e = i R + rel_e:
    Z[v]  = sum_{e : v_e = v} w_e X[j]                  Z [rows, R, f]
    dX[j] = sum_{e in column j} w_e gZ[v_e]
with w_e = 1 (aggr "add", no w), the given w_e ("add"), 1 / c_e ("mean", c_e the entries of e's (row, relation) pair)
or w_e / c_e (both). `terms` computes these in fp64 with the exact weights, and a first-order bound of the kernels'
fp32 error alongside: the rounded product (when the kernels multiply at all), every sum of d terms d roundings of its
sum|terms| (a split row's chunk partials and their fixup add no more than that), the reverse exchange's halo additions
two more for dX, and the difference between the kernels' fp32 weights (the fp32 quotient 1 / c, and its fp32 product
with w) and the exact ones. The bound it returns is twice that estimate.
"""
import math

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from gatedgcn_oracle import entries, graph
from oracle import pgat_oracle as po

EPS32 = 2.0 ** -24
HASH_ROW, HASH_COL = 2654435761, 40503


def relation_hash(rows, cols, R):
    """rgcn.relation_hash restated: ((row * 2654435761 + col * 40503) mod 2^32 >> 16) mod R of global ids."""
    h = (np.asarray(rows, np.int64) * HASH_ROW + np.asarray(cols, np.int64) * HASH_COL) & 0xFFFFFFFF
    return (h >> 16) % R


def pair_counts(rowptr, rel, R):
    """c_e: the number of entries of every entry's (row, relation) pair."""
    rows, _ = entries(rowptr, np.zeros(len(rel), np.int64))
    v = rows * R + np.asarray(rel, np.int64)
    return np.bincount(v, minlength=(len(rowptr) - 1) * R)[v]


def kernel_weights(rowptr, rel, R, w=None, aggr="add"):
    """The fp32 weights the kernels take (op.rgcn_weights), or None for all ones."""
    if aggr == "add":
        return None if w is None else np.asarray(w, np.float32)
    mean = np.float32(1.0) / pair_counts(rowptr, rel, R).astype(np.float32)
    return mean if w is None else np.asarray(w, np.float32) * mean


def exact_weights(rowptr, rel, R, w=None, aggr="add"):
    """The intended weights in fp64."""
    one = np.ones(len(rel)) if w is None else np.asarray(w, np.float64)
    return one if aggr == "add" else one / pair_counts(rowptr, rel, R)


def terms(rowptr, colidx, ncols, rel, R, X, gZ=None, w=None, aggr="add"):
    """Forward and, with gZ ([rows, R, f]), backward of the CSR (rowptr over rows, colidx in [0, ncols)) on X
    [ncols, f]. Returns {name: (fp64 value, bound)}: "Z" ([rows, R, f]) and with gZ "dX" ([ncols, f])."""
    rows, cols = entries(rowptr, colidx)
    nr, f, nnz = len(rowptr) - 1, X.shape[1], len(rows)
    v = rows * R + np.asarray(rel, np.int64)
    w32 = kernel_weights(rowptr, rel, R, w, aggr)
    p = 0 if w32 is None else 1
    w32 = np.ones(nnz) if w32 is None else w32.astype(np.float64)
    we = exact_weights(rowptr, rel, R, w, aggr)
    shape = (nr * R, ncols)
    M = sp.csr_matrix((we, (v, cols)), shape=shape)
    Ma = sp.csr_matrix((np.abs(w32), (v, cols)), shape=shape)
    Md = sp.csr_matrix((np.abs(w32 - we), (v, cols)), shape=shape)
    dv = np.bincount(v, minlength=nr * R)[:, None].astype(np.float64)
    dc = np.bincount(cols, minlength=ncols)[:, None].astype(np.float64)
    X = np.asarray(X, np.float64)
    aX = np.abs(X)
    u = EPS32
    out = {"Z": (M @ X, 2.0 * ((dv + p) * u * (Ma @ aX) + Md @ aX))}
    if gZ is not None:
        g = np.asarray(gZ, np.float64).reshape(nr * R, f)
        ag = np.abs(g)
        out["dX"] = (M.T @ g, 2.0 * ((dc + p + 2) * u * (Ma.T @ ag) + Md.T @ ag))
    return {"Z": tuple(a.reshape(nr, R, f) for a in out["Z"]), **({"dX": out["dX"]} if gZ is not None else {})}


def fp32_reference(rowptr, colidx, ncols, rel, R, X, gZ, w=None, aggr="add"):
    """The kernels' formulas in fp32, sums in entry order: where their results are NaN or +-inf."""
    rows, cols = entries(rowptr, colidx)
    nr, f = len(rowptr) - 1, X.shape[1]
    v = rows * R + np.asarray(rel, np.int64)
    w32 = kernel_weights(rowptr, rel, R, w, aggr)
    X, g = np.asarray(X, np.float32), np.asarray(gZ, np.float32).reshape(nr * R, f)
    with np.errstate(over="ignore", invalid="ignore"):
        tz = X[cols] if w32 is None else w32[:, None] * X[cols]
        tx = g[v] if w32 is None else w32[:, None] * g[v]
        Z = np.zeros((nr * R, f), np.float32)
        np.add.at(Z, v, tz)
        dX = np.zeros((ncols, f), np.float32)
        np.add.at(dX, cols, tx)
    return {"Z": Z.reshape(nr, R, f), "dX": dX}


def torch_dense(rowptr, colidx, ncols, rel, R, X, w=None, aggr="add"):
    """Z [rows, R, f] of a dense per-relation matrix product, differentiable (X a torch tensor): A_r[i, j] sums the
    weights of row i's entries (i, j) with relation r."""
    rows, cols = entries(rowptr, colidx)
    nr = len(rowptr) - 1
    we = exact_weights(rowptr, rel, R, w, aggr)
    rel = np.asarray(rel, np.int64)
    out = []
    for r in range(R):
        s = rel == r
        A = np.zeros((nr, ncols))
        np.add.at(A, (rows[s], cols[s]), we[s])
        out.append(torch.from_numpy(A).to(X.dtype) @ X)
    return torch.stack(out, 1)


def init_params(nlayers, f, R, bases, seed):
    """[layer] as rgcn.PRGCN draws them on the CPU after torch.manual_seed(seed): weight [R, f, f] (with bases: basis
    [B, f, f], then comp [R, B]), then root [f, f], each glorot-uniform over its last two dimensions; bias zeros. fp32
    draws, returned as fp64 numpy tuples (weight, root, bias) or (basis, comp, root, bias)."""
    torch.manual_seed(seed)

    def glorot(*shape):
        a = math.sqrt(6.0 / (shape[-2] + shape[-1]))
        return torch.empty(*shape).uniform_(-a, a)
    layers = []
    for _ in range(nlayers):
        drawn = [glorot(R, f, f)] if bases is None else [glorot(bases, f, f), glorot(R, bases)]
        drawn += [glorot(f, f), torch.zeros(f)]
        layers.append(tuple(x.numpy().astype(np.float64) for x in drawn))
    return layers


def intended_forward(A, H, params, R, bases=None):
    """Logits of rgcn.PRGCN on the global graph A (relations from relation_hash, aggr "mean"); params flat: each
    layer's tensors as init_params orders them."""
    rows, cols, _ = graph(A)
    n = A.shape[0]
    r, c = rows.numpy(), cols.numpy()
    rel = torch.from_numpy(relation_hash(r, c, R))
    v = rows * R + rel
    cnt = torch.bincount(v, minlength=n * R).to(torch.float64)
    wt = (1.0 / cnt[v])[:, None]
    t = [torch.as_tensor(x, dtype=torch.float64) for x in params]
    h = torch.as_tensor(H, dtype=torch.float64)
    per = 3 if bases is None else 4
    nl = len(t) // per
    for li in range(nl):
        p = t[li * per:(li + 1) * per]
        if bases is None:
            W, root, bias = p
        else:
            basis, comp, root, bias = p
            W = (comp @ basis.reshape(bases, -1)).reshape(R, *basis.shape[1:])
        f_in = h.shape[1]
        Z = torch.zeros((n * R, f_in), dtype=torch.float64).index_add(0, v, wt * h[cols])
        h = Z.reshape(n, R * f_in) @ W.reshape(R * f_in, -1) + h @ root + bias
        if li + 1 < nl:
            h = F.relu(h)
    return h


def intended_training(A, nlayers, f, R, seed, bases=None, k=1, epochs=50, lr=1e-3):
    """The loss curve rgcn.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    flat = [torch.tensor(x, requires_grad=True) for p in init_params(nlayers, f, R, bases, seed) for x in p]
    return po.train([tuple(flat)], lambda ps: intended_forward(A, H, ps[0], R, bases), n, f, k, epochs, lr)
