"""NumPy / fp64 reference of GatedGCN's aggregation (pgcn_gatedgcn_*, op.PGatedGCN) and of the PGATEDGCN trainer
(gatedgcn.py) — TEST INFRASTRUCTURE, the product never imports it.

For the entries e = (i, j) of a CSR, with ehat = (Dx[i] + Ex[j]) + Ce_e and s = sigmoid(ehat):
    Z[i]   = num_i / (den_i + eps),  num_i = sum_row s Bx[j],  den_i = sum_row s
    U[i]   = gZ[i] / (den_i + eps)
    dCe_e  = gE_e + U[i] (Bx[j] - Z[i]) s (1 - s)
    dDx[i] = sum_row dCe,   dEx[j] = sum_col dCe,   dBx[j] = sum_col s U[i]
`terms` computes these in fp64 from ehat rounded to fp32 as the kernels round it (it is an output, exact in fp32, and
sigmoid's condition number would otherwise put its rounding into the bound), and propagates a first-order bound of the
kernels' fp32 error alongside: each gate and each s (1 - s) within CONST ulp (the gated aggregation's 4 and 12 ulp with
room), every other operation one rounding, every d-term sum d roundings of its sum|terms|, and the reverse exchange's
halo additions two more. The bound it returns is twice that estimate, for the second-order terms.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pgat_oracle as po

EPS32 = 2.0 ** -24
CONST = 16
BLOCK = 32       # features per block: bounds the [nnz, block] temporaries


def entries(rowptr, idx):
    rowptr = np.asarray(rowptr, dtype=np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr)), np.asarray(idx, dtype=np.int64)


def ehat32(rows, cols, Dx, Ex, Ce):
    """ehat in fp32, summed as the kernels sum it: (Dx[i] + Ex[j]) + Ce."""
    f32 = np.float32
    return (np.asarray(Dx, f32)[rows] + np.asarray(Ex, f32)[cols]) + np.asarray(Ce, f32)


def _sigmoid(x):
    """(s, s (1 - s)) in fp64, the latter as s sigmoid(-x), accurate where s is near 1."""
    with np.errstate(over="ignore"):
        s = 1.0 / (1.0 + np.exp(-x))
        return s, s / (1.0 + np.exp(x))


def _scatter(at, n, nnz):
    return sp.csr_matrix((np.ones(nnz), (at, np.arange(nnz))), shape=(n, nnz))


def terms(rowptr, colidx, ncols, Dx, Ex, Bx, Ce, gZ=None, gE=None, eps=1e-6, round_e=True):
    """Forward and, with gZ, backward of the CSR (rowptr over rows, colidx in [0, ncols)) on Dx [rows, f], Ex and Bx
    [ncols, f], Ce [nnz, f], gZ [rows, f] and gE [nnz, f] (None: zero). Returns {name: (fp64 value, bound)}: "Ehat"
    (bound 0: the kernels give its fp32 bits), "Z", "den", and with gZ "dCe", "dDx", "dEx", "dBx" ([ncols, f] for the
    last two). round_e=False evaluates ehat in fp64 too (the bounds then do not apply)."""
    rows, cols = entries(rowptr, colidx)
    nr, f, nnz = Dx.shape[0], Dx.shape[1], len(rows)
    R, Cm = _scatter(rows, nr, nnz), _scatter(cols, ncols, nnz)
    drow = np.diff(np.asarray(rowptr, np.int64))[:, None].astype(np.float64)
    dcol = np.bincount(cols, minlength=ncols)[:, None].astype(np.float64)
    names = ["Ehat", "Z", "den"] + (["dCe", "dDx", "dEx", "dBx"] if gZ is not None else [])
    shapes = {"Ehat": nnz, "Z": nr, "den": nr, "dCe": nnz, "dDx": nr, "dEx": ncols, "dBx": ncols}
    out = {k: (np.zeros((shapes[k], f)), np.zeros((shapes[k], f))) for k in names}
    u, G = EPS32, CONST * EPS32
    for c0 in range(0, f, BLOCK):
        c = slice(c0, min(f, c0 + BLOCK))
        if round_e:
            e = ehat32(rows, cols, Dx[:, c], Ex[:, c], Ce[:, c]).astype(np.float64)
        else:
            e = (Dx[rows, c].astype(np.float64) + Ex[cols, c].astype(np.float64)) + Ce[:, c].astype(np.float64)
        s, ds = _sigmoid(e)
        b = Bx[cols, c].astype(np.float64)
        den = R @ s
        num = R @ (s * b)
        eden = (drow + CONST) * u * den
        enum = (drow + CONST) * u * (R @ np.abs(s * b))
        q = den + eps
        eq = eden + u * q
        Z = num / q
        eZ = enum / q + np.abs(Z) * eq / q + u * np.abs(Z)
        vals = {"Ehat": (e, 0.0 * e), "Z": (Z, eZ), "den": (den, eden + u * den)}
        if gZ is not None:
            U = gZ[:, c].astype(np.float64) / q
            eU = np.abs(U) * (eq / q + u)
            g = np.zeros_like(e) if gE is None else gE[:, c].astype(np.float64)
            diff = b - Z[rows]
            ediff = eZ[rows] + u * np.abs(diff)
            dsig = U[rows] * diff
            edsig = np.abs(U[rows]) * ediff + np.abs(diff) * eU[rows] + u * np.abs(dsig)
            dce = g + dsig * ds
            edce = ds * edsig + np.abs(dsig) * G * ds + u * np.abs(dce)
            su = s * U[rows]
            esu = G * np.abs(su) + s * eU[rows] + u * np.abs(su)
            vals["dCe"] = (dce, edce)
            vals["dDx"] = (R @ dce, R @ edce + drow * u * (R @ np.abs(dce)))
            vals["dEx"] = (Cm @ dce, Cm @ edce + (dcol + 2) * u * (Cm @ np.abs(dce)))
            vals["dBx"] = (Cm @ su, Cm @ esu + (dcol + 2) * u * (Cm @ np.abs(su)))
        for k in names:
            out[k][0][:, c] = vals[k][0]
            out[k][1][:, c] = 2.0 * vals[k][1]
    return out


def fp32_reference(rowptr, colidx, ncols, Dx, Ex, Bx, Ce, gZ, gE=None, eps=1e-6):
    """The kernels' formulas in fp32 with sums in entry order: where their results are NaN or +-inf."""
    rows, cols = entries(rowptr, colidx)
    nr, f = Dx.shape
    one, e32 = np.float32(1), np.float32(eps)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        e = ehat32(rows, cols, Dx, Ex, Ce)
        x = np.exp(-e)
        s = one / (one + x)
        ds = s * np.where(np.isinf(x), one, x * s)
        b = Bx[cols]

        def add(at, t, n):
            acc = np.zeros((n, f), np.float32)
            np.add.at(acc, at, t)
            return acc
        num, den = add(rows, s * b, nr), add(rows, s, nr)
        Z = num / (den + e32)
        U = gZ / (den + e32)
        g = np.zeros_like(e) if gE is None else gE
        dce = g + (U[rows] * (b - Z[rows])) * ds
        return {"Ehat": e, "Z": Z, "den": den, "dCe": dce, "dDx": add(rows, dce, nr), "dEx": add(cols, dce, ncols),
                "dBx": add(cols, s * U[rows], ncols)}


def torch_gatedgcn(rows, cols, m, Dx, Ex, Bx, Ce, eps=1e-6):
    """(Z, Ehat) of the plain formula as a differentiable torch gather / index_add_ (rows, cols int64 tensors)."""
    e = (Dx[rows] + Ex[cols]) + Ce
    s = torch.sigmoid(e)
    z = torch.zeros((m, Bx.shape[1]), dtype=Bx.dtype, device=Bx.device)
    num = z.index_add(0, rows, s * Bx[cols])
    den = z.index_add(0, rows, s)
    return num / (den + eps), e


def init_params(nlayers, f, seed):
    """(encoder, [layer]) as gatedgcn.PGATEDGCN draws them on the CPU after torch.manual_seed(seed): the edge encoder
    Linear(1, f) as (W, b), then per layer Linear(f, f) A, B, D, E, C as (WA, bA, WB, bB, WD, bD, WE, bE, WC, bC). fp32
    draws, returned as fp64 numpy."""
    torch.manual_seed(seed)
    enc = nn.Linear(1, f)
    layers = []
    for _ in range(nlayers):
        lins = [nn.Linear(f, f) for _ in range(5)]          # A, B, D, E, C
        layers.append(tuple(t.detach().numpy().astype(np.float64) for lin in lins for t in (lin.weight, lin.bias)))
    return (enc.weight.detach().numpy().astype(np.float64), enc.bias.detach().numpy().astype(np.float64)), layers


def graph(A):
    """(rows, cols, vals) of A's stored pattern, duplicates summed in fp32 as the loader sums them, vals as fp64."""
    C = sp.csr_matrix(A).astype(np.float32)
    C.sum_duplicates()
    r, c = entries(C.indptr, C.indices)
    return torch.from_numpy(r), torch.from_numpy(c), torch.from_numpy(C.data.astype(np.float64))


def intended_forward(A, H, params):
    """Logits of PGATEDGCN on the global graph A; H and params as numpy or fp64 tensors (params flat: the encoder's
    W, b, then each layer's ten tensors)."""
    rows, cols, vals = graph(A)
    n = A.shape[0]
    t = [torch.as_tensor(x, dtype=torch.float64) for x in params]
    h = torch.as_tensor(H, dtype=torch.float64)
    e = vals[:, None] @ t[0].T + t[1]
    for l0 in range(2, len(t), 10):
        WA, bA, WB, bB, WD, bD, WE, bE, WC, bC = t[l0:l0 + 10]
        Z, eh = torch_gatedgcn(rows, cols, n, h @ WD.T + bD, h @ WE.T + bE, h @ WB.T + bB, e @ WC.T + bC)
        h, e = h + F.relu(h @ WA.T + bA + Z), e + F.relu(eh)
    return h


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3):
    """The loss curve gatedgcn.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    enc, layers = init_params(nlayers, f, seed)
    flat = [torch.tensor(x, requires_grad=True) for x in list(enc) + [x for p in layers for x in p]]
    return po.train([tuple(flat)], lambda ps: intended_forward(A, H, ps[0]), n, f, k, epochs, lr)
