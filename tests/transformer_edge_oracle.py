"""NumPy / fp64 reference of the graph transformer attention with edge features (pgcn_transformer_edge_*,
op.PTransformerEdgeAttention) and of PTRANSFORMER --edge-values (transformer.py) — TEST INFRASTRUCTURE, the product never
imports it.

For the entries e = (i, j) of a CSR, a head h of width C and the edge term E_e, with M the dropout factor:
    kk_e = k_j + E_e,  vv_e = v_j + E_e
    s_e = scale <q_i, kk_e>,  L_i = log sum_row exp(s_e),  p_e = exp(s_e - L_i),  P_e = M_e p_e
    Z_i = sum_row P_e vv_e
    D_i = <gZ_i, Z_i>,  ds_e = p_e (M_e <gZ_i, vv_e> - D_i)
    dQ_i = scale sum_row ds_e kk_e,  dE_e = P_e gZ_i + scale ds_e q_i,  dK_j = scale sum_col ds_e q_i,
    dV_j = sum_col P_e gZ_i
`attention` computes these in fp64 and, per output element, the fp32 bound of tests/transformer_oracle.attention with
the two roundings the kernels add: kk and vv are rounded to fp32 before they are used, so every product of the score
and of dp carries one more rounding (C + DOT + 1 in place of C + DOT), and so does every term of Z (C0 + 1). dQ sums
|kk| in place of |k|. dE_e takes the error of P and of ds and three more roundings (the product P gZ, scale ds and
the fused add).
"""
import numpy as np
import torch
import torch.nn as nn

import dropout_oracle as do
import gatedgcn_oracle as gco
import transformer_oracle as tro
from oracle import pgat_oracle as po

EPS = tro.EPS
DOT = tro.DOT


def attention(rowptr, colidx, ncols, Q, K, V, E, gZ, heads, scale, const, M=None, dcol=None):
    """{name: (fp64 value, fp32 bound)} for "Z", "L", "dQ" ([rows, f] / [rows, heads]), "dK", "dV" ([ncols, f]) and
    "dE" ([nnz, f]) of the CSR (rowptr over rows, colidx in [0, ncols)). Q, gZ [rows, f]; K, V [ncols, f]; E [nnz, f]
    in entry order; scale the fp32 scale as a float; M None or fp64 [nnz, heads]; dcol the column degrees the column
    sums run over (default: this CSR's), `const` the bound's constant."""
    rows, cols = tro.entries(rowptr, colidx)
    nr, f = Q.shape
    C = f // heads
    Q, K, V, E, gZ = (np.asarray(x, np.float64) for x in (Q, K, V, E, gZ))
    ent = np.arange(len(rows))
    KK, VV = K[cols] + E, V[cols] + E
    drow = np.bincount(rows, minlength=nr).astype(np.float64)
    dcol = np.bincount(cols, minlength=ncols).astype(np.float64) if dcol is None else np.asarray(dcol, np.float64)
    out = {"Z": np.zeros((nr, f)), "L": np.full((nr, heads), -np.inf), "dQ": np.zeros((nr, f)),
           "dK": np.zeros((ncols, f)), "dV": np.zeros((ncols, f)), "dE": np.zeros((len(rows), f))}
    tol = {name: np.zeros_like(v) for name, v in out.items()}
    for h in range(heads):
        sl = slice(h * C, (h + 1) * C)
        Mh = np.ones(len(rows)) if M is None else M[:, h]
        qk, aqk = tro._dot(Q, rows, KK, ent, sl)
        s, sig = scale * qk, (C + DOT + 1) * EPS * scale * aqk          # score and its error
        m = np.full(nr, -np.inf)
        np.maximum.at(m, rows, s)
        with np.errstate(invalid="ignore", divide="ignore"):
            e = np.exp(s - m[rows])
            l = np.bincount(rows, weights=e, minlength=nr)
            L = m + np.log(l)
        p = e / l[rows]
        w = Mh * p
        Z = tro._scatter(nr, rows, w, VV, ent, sl)
        magZ = tro._scatter(nr, rows, w, np.abs(VV), ent, sl)
        Em = np.zeros(nr)
        np.maximum.at(Em, rows, sig + 2 * np.abs(s - m[rows]) * EPS)
        ef = (10 * drow + const + 1) * EPS + 2 * Em                       # relative error of each weight, and of vv
        tZ = ef[:, None] * magZ
        with np.errstate(divide="ignore"):
            tL = (np.abs(m) + 2 * np.abs(np.log(l))) * EPS + ef
        # backward
        dp, adp = tro._dot(gZ, rows, VV, ent, sl)
        D = (gZ[:, sl] * Z).sum(1)
        dD = (C + DOT) * EPS * np.abs(gZ[:, sl] * Z).sum(1) + (np.abs(gZ[:, sl]) * tZ).sum(1)
        ds = p * (Mh * dp - D[rows])
        mds = p * (Mh * np.abs(dp) + np.abs(D[rows]))
        eb = sig + tL[rows] + (np.abs(s - L[rows]) + const) * EPS         # relative error of the backward's p
        eds = mds * eb + p * (Mh * (C + DOT + 1) * EPS * adp + dD[rows])
        out["Z"][:, sl], tol["Z"][:, sl] = Z, tZ
        has = drow > 0
        out["L"][has, h], tol["L"][has, h] = L[has], tL[has]
        out["dQ"][:, sl] = scale * tro._scatter(nr, rows, ds, KK, ent, sl)
        tol["dQ"][:, sl] = scale * tro._scatter(nr, rows, mds * (drow[rows] + const) * EPS + eds, np.abs(KK), ent, sl)
        out["dK"][:, sl] = scale * tro._scatter(ncols, cols, ds, Q, rows, sl)
        tol["dK"][:, sl] = scale * tro._scatter(ncols, cols, mds * (dcol[cols] + const) * EPS + eds, np.abs(Q), rows,
                                                sl)
        out["dV"][:, sl] = tro._scatter(ncols, cols, w, gZ, rows, sl)
        tol["dV"][:, sl] = tro._scatter(ncols, cols, w * (eb + (dcol[cols] + const) * EPS), np.abs(gZ), rows, sl)
        out["dE"][:, sl] = w[:, None] * gZ[rows, sl] + scale * ds[:, None] * Q[rows, sl]
        tol["dE"][:, sl] = ((w * (eb + 3 * EPS))[:, None] * np.abs(gZ[rows, sl])
                            + scale * (eds + 3 * EPS * mds)[:, None] * np.abs(Q[rows, sl]))
    return {name: (out[name], tol[name] + 1e-30) for name in out}


def torch_transformer_edge(rows, cols, n, Q, K, V, E, heads, scale, M=None):
    """out[i, h] = sum over the entries e = (i, j) of M alpha (V[j, h] + E_e[h]), alpha the per-row softmax of
    scale <Q[i, h], K[j, h] + E_e[h]>, as a differentiable torch gather / scatter (rows, cols int64 tensors; E [nnz, f];
    M None or [nnz, heads])."""
    f = Q.shape[1]
    C = f // heads
    KK, VV = K[cols] + E, V[cols] + E
    s = (Q[rows].view(-1, heads, C) * KK.view(-1, heads, C)).sum(2) * scale
    alpha = torch.stack([po.edge_softmax(rows, s[:, h], n) for h in range(heads)], 1)
    if M is not None:
        alpha = alpha * M
    msg = (alpha[:, :, None] * VV.view(-1, heads, C)).reshape(-1, f)
    return torch.zeros((n, f), dtype=V.dtype).index_add(0, rows, msg)


def init_params(nlayers, f, seed):
    """[(Wk, bk, Wq, bq, Wv, bv, We, Ws, bs)] as transformer.PTRANSFORMER(edge_values=True) draws them on the CPU after
    torch.manual_seed(seed): lin_key, lin_query, lin_value = Linear(f, f), lin_edge = Linear(1, f, bias=False),
    lin_skip = Linear(f, f). fp32 draws as fp64 numpy."""
    torch.manual_seed(seed)
    out = []
    for _ in range(nlayers):
        ls = [nn.Linear(f, f) for _ in range(3)] + [nn.Linear(1, f, bias=False), nn.Linear(f, f)]
        out.append(tuple(t.detach().numpy().astype(np.float64) for lin in ls for t in lin.parameters()))
    return out


def intended_forward(A, H, params, heads, p=0.0, seed=None, counter=None):
    """Logits of the intended model on the global graph A (its stored pattern, duplicates summed as the loader sums
    them, and their values as the edge input), with every layer's dropout mask at call counter `counter` when p > 0."""
    rows, cols, vals = gco.graph(A)
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for layer, prm in enumerate(params):
        Wk, bk, Wq, bq, Wv, bv, We, Ws, bs = (torch.as_tensor(t, dtype=torch.float64) for t in prm)
        f = Wk.shape[0]
        scale = float(np.float32(1.0 / np.sqrt(f / heads)))
        M = None
        if p > 0:
            M = do.weights(rows.numpy(), cols.numpy(), heads, p, ((seed or 0) * 2 ** 16 + layer) % 2 ** 64, counter)
        E = vals[:, None] @ We.T
        N = torch_transformer_edge(rows, cols, n, X @ Wq.T + bq, X @ Wk.T + bk, X @ Wv.T + bv, E, heads, scale, M)
        X = torch.relu(N + X @ Ws.T + bs)
    return X


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3, heads=1, p=0.0):
    """The loss curve transformer.run(edge_values=True) prints: inputs H[i, :] = i (pgat_oracle.inputs) and
    pgat_oracle.train's loop; epoch e draws its masks with counter e + 1."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    params = [tuple(torch.tensor(t, requires_grad=True) for t in prm) for prm in init_params(nlayers, f, seed)]
    epoch = iter(range(epochs))
    return po.train(params, lambda ps: intended_forward(A, H, ps, heads, p, seed, next(epoch) + 1), n, f, k, epochs, lr)
