"""NumPy / fp64 reference of GATv2 attention with edge features (pgcn_gatv2_edge_*, op.PGATv2EdgeAttention) and of
PGAT.py --v2 --edge-values (pgat.PGATv2(edge_values=True)) — TEST INFRASTRUCTURE, the product never imports it.

It extends tests/gatv2_oracle.py with the edge term and the dropout factor. For the entries e = (i, j) of a CSR, a head
h of width d (features c of the head), with M the dropout factor (tests/dropout_oracle.weights, 1 without dropout):
    t_e = (xr_i + xl_j) + E_e,  s_e = sum_c att_c LeakyReLU(t_ec),  L_i = log sum_row exp(s_e),  p_e = exp(s_e - L_i)
    Z_i = sum_row M_e p_e xl_j
    D_i = <gZ_i, Z_i>,  ds_e = p_e (M_e <gZ_i, xl_j> - D_i),  g_ec = ds_e att_c LeakyReLU'(t_ec)
    dE_e = g_e,  dXR_i = sum_row g_e,  datt_c = sum_e ds_e LeakyReLU(t_ec),  dXL_j = sum_col (M_e p_e gZ_i + g_e)
`attention` computes these in fp64 and, per output element, a first-order fp32 bound: the two roundings of t (each
relative to |xr| + |xl| + |E|, scaled by max(1, |slope|) through LeakyReLU) and the slope product enter the score
error beside the C + DOT roundings of a head's sum; the softmax, Z, D and ds follow tests/transformer_oracle.attention;
every gradient sum takes (terms + const) roundings of its magnitude sum. datt is summed per work item, per CTA of 8
items and over the CTAs, so its depth is the longest row plus the number of CTA partials.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

import dropout_oracle as do
import gatedgcn_oracle as gco
import gatv2_oracle as go
import transformer_oracle as tro
from oracle import pgat_oracle as po

EPS = tro.EPS
DOT = tro.DOT


def _terms(rows, cols, XL, XR, E, att, slope):
    """(t, LeakyReLU(t), LeakyReLU'(t), error of LeakyReLU(t)) per entry and feature, fp64."""
    t = (XR[rows] + XL[cols]) + E
    smax = max(1.0, abs(slope))
    lt = go.leaky(t, slope)
    err = 2 * EPS * smax * (np.abs(XR[rows]) + np.abs(XL[cols]) + np.abs(E)) + EPS * np.abs(lt)
    return t, lt, np.where(t > 0, 1.0, slope), err


def attention(rowptr, colidx, ncols, XL, XR, att, E, gZ, slope, const, M=None, dcol=None):
    """{name: (fp64 value, fp32 bound)} for "Z", "L", "dXR" ([rows, f] / [rows, heads]), "dXL" ([ncols, f]), "datt"
    ([heads, d]), "dE" ([nnz, f]), "P" and "ds" ([nnz, heads]) of the CSR (rowptr over rows, colidx in [0, ncols)).
    XR, gZ [rows, f]; XL [ncols, f]; E [nnz, f] in entry order; att [heads, d]; M None or fp64 [nnz, heads]; dcol the
    column degrees the column sums run over (default: this CSR's), `const` the bound's constant."""
    rows, cols = tro.entries(rowptr, colidx)
    nr, f = XR.shape
    heads, C = np.asarray(att).shape
    XL, XR, E, gZ = (np.asarray(x, np.float64) for x in (XL, XR, E, gZ))
    a = np.asarray(att, np.float64).reshape(-1)
    nnz = len(rows)
    t, lt, dl, elt = _terms(rows, cols, XL, XR, E, a, slope)
    drow = np.bincount(rows, minlength=nr).astype(np.float64)
    dcol = np.bincount(cols, minlength=ncols).astype(np.float64) if dcol is None else np.asarray(dcol, np.float64)
    datt_depth = (drow.max() if nr else 0) + (nr + nnz) / 256.0 + 40
    out = {"Z": np.zeros((nr, f)), "L": np.full((nr, heads), -np.inf), "dXR": np.zeros((nr, f)),
           "dXL": np.zeros((ncols, f)), "datt": np.zeros(f), "dE": np.zeros((nnz, f)), "P": np.zeros((nnz, heads)),
           "ds": np.zeros((nnz, heads))}
    tol = {name: np.zeros_like(v) for name, v in out.items()}
    ent = np.arange(nnz)
    for h in range(heads):
        sl = slice(h * C, (h + 1) * C)
        Mh = np.ones(nnz) if M is None else M[:, h]
        al = a[sl]
        s = (lt[:, sl] * al).sum(1)
        sig = (C + DOT + 1) * EPS * np.abs(lt[:, sl] * al).sum(1) + (elt[:, sl] * np.abs(al)).sum(1)
        m = np.full(nr, -np.inf)
        np.maximum.at(m, rows, s)
        with np.errstate(invalid="ignore", divide="ignore"):
            e = np.exp(s - m[rows])
            l = np.bincount(rows, weights=e, minlength=nr)
            L = m + np.log(l)
        p = e / l[rows]
        w = Mh * p
        Z = tro._scatter(nr, rows, w, XL, cols, sl)
        magZ = tro._scatter(nr, rows, w, np.abs(XL), cols, sl)
        Em = np.zeros(nr)
        np.maximum.at(Em, rows, sig + 2 * np.abs(s - m[rows]) * EPS)
        ef = (10 * drow + const) * EPS + 2 * Em                           # relative error of each weight
        tZ = ef[:, None] * magZ
        with np.errstate(divide="ignore"):
            tL = (np.abs(m) + 2 * np.abs(np.log(l))) * EPS + ef
        # backward
        dp, adp = tro._dot(gZ, rows, XL, cols, sl)
        D = (gZ[:, sl] * Z).sum(1)
        dD = (C + DOT) * EPS * np.abs(gZ[:, sl] * Z).sum(1) + (np.abs(gZ[:, sl]) * tZ).sum(1)
        ds = p * (Mh * dp - D[rows])
        mds = p * (Mh * np.abs(dp) + np.abs(D[rows]))
        eb = sig + tL[rows] + (np.abs(s - L[rows]) + const) * EPS         # relative error of the backward's p
        eds = mds * eb + p * (Mh * (C + DOT) * EPS * adp + dD[rows])
        g = ds[:, None] * al * dl[:, sl]
        ag = mds[:, None] * np.abs(al) * np.abs(dl[:, sl])
        eg = (eds + 3 * EPS * mds)[:, None] * np.abs(al) * np.abs(dl[:, sl])
        out["Z"][:, sl], tol["Z"][:, sl] = Z, tZ
        has = drow > 0
        out["L"][has, h], tol["L"][has, h] = L[has], tL[has]
        out["P"][:, h], tol["P"][:, h] = w, w * (eb + EPS)
        out["ds"][:, h], tol["ds"][:, h] = ds, eds
        out["dE"][:, sl], tol["dE"][:, sl] = g, eg
        one = np.ones(nnz)
        out["dXR"][:, sl] = tro._scatter(nr, rows, one, g, ent, slice(0, C))
        tol["dXR"][:, sl] = (tro._scatter(nr, rows, one, eg, ent, slice(0, C))
                             + (drow + const)[:, None] * EPS * tro._scatter(nr, rows, one, ag, ent, slice(0, C)))
        term = w[:, None] * gZ[rows, sl] + g
        aterm = w[:, None] * np.abs(gZ[rows, sl]) + ag
        eterm = (w * (eb + EPS))[:, None] * np.abs(gZ[rows, sl]) + eg + EPS * aterm
        out["dXL"][:, sl] = tro._scatter(ncols, cols, one, term, ent, slice(0, C))
        tol["dXL"][:, sl] = (tro._scatter(ncols, cols, one, eterm, ent, slice(0, C))
                             + (dcol + const)[:, None] * EPS * tro._scatter(ncols, cols, one, aterm, ent, slice(0, C)))
        out["datt"][sl] = (ds[:, None] * lt[:, sl]).sum(0)
        tol["datt"][sl] = ((eds[:, None] * np.abs(lt[:, sl]) + mds[:, None] * elt[:, sl]).sum(0)
                           + (datt_depth + const) * EPS * (mds[:, None] * np.abs(lt[:, sl])).sum(0))
    out["datt"], tol["datt"] = out["datt"].reshape(heads, C), tol["datt"].reshape(heads, C)
    return {name: (out[name], tol[name] + 1e-30) for name in out}


def fp32_reference(rowptr, colidx, XL, XR, att, E, gZ, slope, items, splits):
    """The kernels' formulas in fp32 without dropout: {name: value} of Z, L, dXR, dXL, datt and dE. The forward is
    tests/transformer_oracle.fp32_reference's online softmax over every work item in the kernels' order, on one
    "key" per entry (LeakyReLU(t_e)), att as every row's "query", scale 1 and XL[j] as the entry's value, since where a
    rescale meets +-inf decides NaN; the backward sums are order-free in their NaN / +-inf pattern."""
    f32 = np.float32
    rows, cols = tro.entries(rowptr, colidx)
    nr, f = XR.shape
    heads, C = np.asarray(att).shape
    a = np.asarray(att, f32).reshape(1, f)
    with np.errstate(all="ignore"):
        t = ((XR[rows] + XL[cols]).astype(f32) + E).astype(f32)
        lt = np.where(t > 0, t, t * f32(slope)).astype(f32)
        VV = XL[cols].astype(f32)
        out = tro.fp32_reference(rowptr, np.arange(len(rows)), len(rows), np.repeat(a, nr, 0), lt, VV, gZ, heads, 1.0,
                                 items, splits)
        hdot = lambda A, B: (A * B).reshape(len(A), heads, C).sum(2, dtype=f32)
        ex = lambda x: np.repeat(x, C, axis=1)
        s = hdot(np.repeat(a, len(rows), 0), lt)
        p = np.exp(s - out["L"][rows])
        D = hdot(gZ, out["Z"])
        ds = p * (hdot(gZ[rows], VV) - D[rows])
        da = ex(ds) * a
        g = np.where(t > 0, da, da * f32(slope)).astype(f32)
        res = {"Z": out["Z"], "L": out["L"], "dE": g}
        res["dXR"] = np.zeros((nr, f), f32)
        np.add.at(res["dXR"], rows, g)
        res["dXL"] = np.zeros((nr, f), f32)
        np.add.at(res["dXL"], cols, ex(p) * gZ[rows] + g)
        res["datt"] = (ex(ds) * lt).sum(0, dtype=f32).reshape(heads, C)
    return res


def torch_gatv2_edge(rows, cols, n, XL, XR, att, E, slope, M=None):
    """out[i, h] = sum over the entries e = (i, j) of M p_e XL[j, h], p the per-row softmax of
    sum_c att[h, c] LeakyReLU((XR[i] + XL[j]) + E_e), as a differentiable torch gather / scatter (rows, cols int64
    tensors; E [nnz, f]; M None or [nnz, heads])."""
    K, d = att.shape
    t = (XR[rows] + XL[cols]) + E
    s = (F.leaky_relu(t, slope).view(-1, K, d) * att[None]).sum(2)
    alpha = torch.stack([po.edge_softmax(rows, s[:, h], n) for h in range(K)], 1)
    if M is not None:
        alpha = alpha * M
    msg = (alpha[:, :, None] * XL[cols].view(-1, K, d)).reshape(-1, K * d)
    return torch.zeros((n, K * d), dtype=XL.dtype).index_add(0, rows, msg)


def init_params(nlayers, f, seed, heads):
    """[(W_l, W_r, att, W_e)] per layer, drawn as pgat.PGATv2(edge_values=True) draws them on the CPU after
    torch.manual_seed(seed): lin_l, lin_r (Linear(f, f, bias=False)) and att (heads, f / heads), then xavier_normal with
    the relu gain on each in that order, then lin_edge = Linear(1, f, bias=False). fp32 draws as fp64 numpy."""
    torch.manual_seed(seed)
    gain = nn.init.calculate_gain("relu")
    out = []
    for _ in range(nlayers):
        lin_l = nn.Linear(f, f, bias=False)
        lin_r = nn.Linear(f, f, bias=False)
        att = torch.empty(size=(heads, f // heads))
        for x in (lin_l.weight, lin_r.weight, att):
            nn.init.xavier_normal_(x, gain=gain)
        lin_edge = nn.Linear(1, f, bias=False)
        out.append(tuple(x.detach().numpy().astype(np.float64) for x in (lin_l.weight, lin_r.weight, att,
                                                                          lin_edge.weight)))
    return out


def intended_forward(A, H, params, slope, heads, p=0.0, seed=None, counter=None):
    """Logits of the intended model on the global graph A (its stored pattern, duplicates summed as the loader sums
    them, and their values as the edge input), with every layer's dropout mask at call counter `counter` when p > 0."""
    rows, cols, vals = gco.graph(A)
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for layer, prm in enumerate(params):
        Wl, Wr, att, We = (torch.as_tensor(x, dtype=torch.float64) for x in prm)
        M = None
        if p > 0:
            M = do.weights(rows.numpy(), cols.numpy(), heads, p, ((seed or 0) * 2 ** 16 + layer) % 2 ** 64, counter)
        X = torch_gatv2_edge(rows, cols, n, X @ Wl.T, X @ Wr.T, att, vals[:, None] @ We.T, slope, M)
    return X


def intended_training(A, nlayers, f, seed, slope, heads=1, k=1, epochs=50, lr=1e-3, p=0.0):
    """The loss curve PGAT.py --v2 --edge-values prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's
    loop; epoch e draws its masks with counter e + 1."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    params = [tuple(torch.tensor(x, requires_grad=True) for x in layer) for layer in init_params(nlayers, f, seed,
                                                                                                 heads)]
    epoch = iter(range(epochs))
    return po.train(params, lambda ps: intended_forward(A, H, ps, slope, heads, p, seed, next(epoch) + 1), n, f, k,
                    epochs, lr)
