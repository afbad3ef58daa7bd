"""NumPy / fp64 reference of the gated aggregation (pgcn_gated_*, op.PSpMMGated) and of the PGATED trainer (gated.py) —
TEST INFRASTRUCTURE, the product never imports it.

For the entries (i, j) of a CSR, with x = K[i] + Q[j] and eta = sigmoid(x):
    Z[i]  = sum_row eta V[j]          dK[i] = gZ[i] sum_row V[j] eta (1 - eta)
    dV[j] = sum_col eta gZ[i]         dQ[j] = V[j] sum_col gZ[i] eta (1 - eta)
`terms` computes these in fp64 with, by default, x rounded to fp32 as the kernels round it: sigmoid's condition number
|x| (1 - sigmoid(x)) would otherwise put the rounding of K + Q into the bound. It also returns each output's sum of
|terms|, the scale of the fp32 bound (d + c) 2^-24 sum|terms|.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pgat_oracle as po

BLOCK = 32       # features per block: bounds the [nnz, block] temporaries


def _entries(rowptr, idx):
    rowptr = np.asarray(rowptr, dtype=np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr)), np.asarray(idx, dtype=np.int64)


def _sigmoid(x):
    """(eta, eta (1 - eta)) in fp64, the latter as eta sigmoid(-x), accurate where eta is near 1."""
    with np.errstate(over="ignore"):
        eta = 1.0 / (1.0 + np.exp(-x))
        return eta, eta / (1.0 + np.exp(x))


def terms(rowptr, colidx, ncols, K, Q, V, gZ=None, round_x=True):
    """Forward and, with gZ, backward of the CSR (rowptr over rows, colidx in [0, ncols)) on K [rows, f], Q and V
    [ncols, f], gZ [rows, f], all fp64 results. Returns a dict of (value, sum|terms|) pairs: "Z", and with gZ "dK",
    "dQ", "dV" ([ncols, f] for dQ and dV)."""
    rows, cols = _entries(rowptr, colidx)
    nr, f = K.shape[0], K.shape[1]
    out = {name: (np.zeros((n, f)), np.zeros((n, f))) for name, n in
           (("Z", nr), ("dK", nr), ("dQ", ncols), ("dV", ncols))}
    for c0 in range(0, f, BLOCK):
        c = slice(c0, min(f, c0 + BLOCK))
        if round_x:
            x = (np.asarray(K[rows, c], np.float32) + np.asarray(Q[cols, c], np.float32)).astype(np.float64)
        else:
            x = K[rows, c].astype(np.float64) + Q[cols, c].astype(np.float64)
        eta, ds = _sigmoid(x)
        v = V[cols, c].astype(np.float64)
        parts = [("Z", rows, eta * v, None)]
        if gZ is not None:
            g = gZ[rows, c].astype(np.float64)
            parts += [("dK", rows, v * ds, gZ[:, c]), ("dV", cols, eta * g, None), ("dQ", cols, g * ds, V[:, c])]
        for name, at, t, scale in parts:
            val, mag = out[name]
            s, a = np.zeros((val.shape[0], t.shape[1])), np.zeros((val.shape[0], t.shape[1]))
            np.add.at(s, at, t)
            np.add.at(a, at, np.abs(t))
            if scale is not None:
                sc = scale.astype(np.float64)
                s, a = s * sc, a * np.abs(sc)
            val[:, c], mag[:, c] = s, a
    return out if gZ is not None else {"Z": out["Z"]}


def fp32_reference(rowptr, colidx, ncols, K, Q, V, gZ):
    """The same sums in fp32, the kernels' formulas in entry order: where their results are NaN or +-inf."""
    rows, cols = _entries(rowptr, colidx)
    nr, f = K.shape
    one = np.float32(1)
    with np.errstate(over="ignore", invalid="ignore"):
        x = K[rows] + Q[cols]
        e = np.exp(-x)
        eta = one / (one + e)
        ds = eta * np.where(np.isinf(e), one, e * eta)
        out = {}
        for name, at, t, n in (("Z", rows, eta * V[cols], nr), ("dK", rows, V[cols] * ds, nr),
                               ("dV", cols, eta * gZ[rows], ncols), ("dQ", cols, gZ[rows] * ds, ncols)):
            s = np.zeros((n, f), np.float32)
            np.add.at(s, at, t)
            out[name] = s
        out["dK"] = gZ * out["dK"]
        out["dQ"] = V * out["dQ"]
    return out


def torch_gated(rows, cols, K, Q, V):
    """out[i] = sum over the entries (i, j) of sigmoid(K[i] + Q[j]) V[j] as a differentiable torch gather / index_add_
    (rows, cols int64 tensors)."""
    msg = torch.sigmoid(K[rows] + Q[cols]) * V[cols]
    return torch.zeros((K.shape[0], V.shape[1]), dtype=V.dtype).index_add(0, rows, msg)


def init_params(nlayers, f, seed):
    """[(Wk, bk, Wq, bq, Wv, bv, Ws, b)] as gated.PGATED draws them on the CPU after torch.manual_seed(seed):
    lin_key, lin_query, lin_value = Linear(f, f), lin_skip = Linear(f, f, bias=False), bias zeros(f). fp32 draws,
    returned as fp64 numpy."""
    torch.manual_seed(seed)
    out = []
    for _ in range(nlayers):
        k, q, v = nn.Linear(f, f), nn.Linear(f, f), nn.Linear(f, f)
        s = nn.Linear(f, f, bias=False)
        out.append(tuple(t.detach().numpy().astype(np.float64) for t in (k.weight, k.bias, q.weight, q.bias, v.weight,
                                                                          v.bias, s.weight)) + (np.zeros(f),))
    return out


def intended_forward(A, H, params):
    """Logits of the intended model on the global graph A (its stored pattern, duplicates summed as the loader sums
    them); H and params as numpy or fp64 tensors."""
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    rows, cols = (torch.from_numpy(a) for a in _entries(C.indptr, C.indices))
    X = torch.as_tensor(H, dtype=torch.float64)
    for p in params:
        Wk, bk, Wq, bq, Wv, bv, Ws, b = (torch.as_tensor(t, dtype=torch.float64) for t in p)
        N = torch_gated(rows, cols, X @ Wk.T + bk, X @ Wq.T + bq, X @ Wv.T + bv)
        X = F.relu(N + X @ Ws.T + b)
    return X


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3):
    """The loss curve gated.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    params = [tuple(torch.tensor(t, requires_grad=True) for t in p) for p in init_params(nlayers, f, seed)]
    return po.train(params, lambda ps: intended_forward(A, H, ps), n, f, k, epochs, lr)
