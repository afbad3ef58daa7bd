"""NumPy / fp64 reference of the graph transformer attention (pgcn_transformer_*, op.PTransformerAttention) and of the
PTRANSFORMER trainer (transformer.py) — TEST INFRASTRUCTURE, the product never imports it.

For the entries e = (i, j) of a CSR and a head h of width C (features c of the head), with M the dropout factor
(tests/dropout_oracle.keep times float32(1 / (1 - p)), 1 without dropout):
    s_e = scale <q_i, k_j>,  m_i = max_e s_e,  l_i = sum_e exp(s_e - m_i),  L_i = m_i + log l_i,  p_e = exp(s_e - L_i)
    Z_i = sum_row M_e p_e v_j
    D_i = <gZ_i, Z_i>,  dp_e = <gZ_i, v_j>,  ds_e = p_e (M_e dp_e - D_i)
    dQ_i = scale sum_row ds_e k_j,  dK_j = scale sum_col ds_e q_i,  dV_j = sum_col M_e p_e gZ_i
`attention` computes these in fp64 and, per output element, the fp32 bound that tests/test_transformer_attention.py
derives, from the per-element magnitude sums (sum |w v|, sum |k| |ds|, ...) and the per-entry score errors.
`fp32_reference` restates the kernels' formulas in fp32, in their order (the online softmax per work item, the chunks
merged in order), to say where their results are NaN or +-inf.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

import dropout_oracle as do
from oracle import pgat_oracle as po

EPS = 2.0 ** -24
BLOCK = 32       # features per block: bounds the [nnz, block] temporaries
# roundings of a per-head dot product besides its C products: a butterfly over at most 32 lanes (5) and the scale (1)
DOT = 6


def entries(rowptr, idx):
    rowptr = np.asarray(rowptr, dtype=np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr)), np.asarray(idx, dtype=np.int64)


def _dot(A, ia, B, ib, sl):
    """(sum_c A[ia, c] B[ib, c], sum_c |A[ia, c] B[ib, c]|) over the features of slice sl, fp64, blockwise."""
    s = np.zeros(len(ia))
    a = np.zeros(len(ia))
    for c0 in range(sl.start, sl.stop, BLOCK):
        c = slice(c0, min(sl.stop, c0 + BLOCK))
        t = A[ia, c] * B[ib, c]
        s += t.sum(1)
        a += np.abs(t).sum(1)
    return s, a


def _scatter(n, at, w, X, ix, sl):
    """sum over entries of w_e X[ix_e, sl] into rows `at` ([n, C] fp64), blockwise."""
    out = np.zeros((n, sl.stop - sl.start))
    for c0 in range(sl.start, sl.stop, BLOCK):
        c = slice(c0, min(sl.stop, c0 + BLOCK))
        np.add.at(out[:, c0 - sl.start:c.stop - sl.start], at, w[:, None] * X[ix, c])
    return out


def attention(rowptr, colidx, ncols, Q, K, V, gZ, heads, scale, const, M=None, dcol=None):
    """{name: (fp64 value, fp32 bound)} for "Z", "L", "dQ" ([rows, f] / [rows, heads]) and "dK", "dV" ([ncols, f]) of the
    CSR (rowptr over rows, colidx in [0, ncols)). Q, gZ [rows, f]; K, V [ncols, f]; scale the fp32 scale as a float;
    M None or fp64 [nnz, heads]; dcol the column degrees the column sums run over (default: this CSR's), `const` the
    bound's constant."""
    rows, cols = entries(rowptr, colidx)
    nr, f = Q.shape
    C = f // heads
    Q, K, V, gZ = (np.asarray(x, np.float64) for x in (Q, K, V, gZ))
    drow = np.bincount(rows, minlength=nr).astype(np.float64)
    dcol = np.bincount(cols, minlength=ncols).astype(np.float64) if dcol is None else np.asarray(dcol, np.float64)
    out = {"Z": np.zeros((nr, f)), "L": np.full((nr, heads), -np.inf), "dQ": np.zeros((nr, f)),
           "dK": np.zeros((ncols, f)), "dV": np.zeros((ncols, f))}
    tol = {name: np.zeros_like(v) for name, v in out.items()}
    for h in range(heads):
        sl = slice(h * C, (h + 1) * C)
        Mh = np.ones(len(rows)) if M is None else M[:, h]
        qk, aqk = _dot(Q, rows, K, cols, sl)
        s, sig = scale * qk, (C + DOT) * EPS * scale * aqk              # score and its error
        m = np.full(nr, -np.inf)
        np.maximum.at(m, rows, s)
        with np.errstate(invalid="ignore", divide="ignore"):
            e = np.exp(s - m[rows])
            l = np.bincount(rows, weights=e, minlength=nr)
            L = m + np.log(l)
        p = e / l[rows]
        w = Mh * p
        Z = _scatter(nr, rows, w, V, cols, sl)
        magZ = _scatter(nr, rows, w, np.abs(V), cols, sl)
        E = np.zeros(nr)
        np.maximum.at(E, rows, sig + 2 * np.abs(s - m[rows]) * EPS)
        ef = (10 * drow + const) * EPS + 2 * E                            # relative error of each weight w / l
        tZ = ef[:, None] * magZ
        with np.errstate(divide="ignore"):
            tL = (np.abs(m) + 2 * np.abs(np.log(l))) * EPS + ef
        # backward
        dp, adp = _dot(gZ, rows, V, cols, sl)
        D = (gZ[:, sl] * Z).sum(1)
        dD = (C + DOT) * EPS * np.abs(gZ[:, sl] * Z).sum(1) + (np.abs(gZ[:, sl]) * tZ).sum(1)
        ds = p * (Mh * dp - D[rows])
        mds = p * (Mh * np.abs(dp) + np.abs(D[rows]))
        eb = sig + tL[rows] + (np.abs(s - L[rows]) + const) * EPS         # relative error of the backward's p
        eds = mds * eb + p * (Mh * (C + DOT) * EPS * adp + dD[rows])
        out["Z"][:, sl], tol["Z"][:, sl] = Z, tZ
        has = drow > 0
        out["L"][has, h], tol["L"][has, h] = L[has], tL[has]
        out["dQ"][:, sl] = scale * _scatter(nr, rows, ds, K, cols, sl)
        tol["dQ"][:, sl] = scale * (_scatter(nr, rows, mds * (drow[rows] + const) * EPS + eds, np.abs(K), cols, sl))
        out["dK"][:, sl] = scale * _scatter(ncols, cols, ds, Q, rows, sl)
        tol["dK"][:, sl] = scale * _scatter(ncols, cols, mds * (dcol[cols] + const) * EPS + eds, np.abs(Q), rows, sl)
        out["dV"][:, sl] = _scatter(ncols, cols, w, gZ, rows, sl)
        tol["dV"][:, sl] = _scatter(ncols, cols, w * (eb + (dcol[cols] + const) * EPS), np.abs(gZ), rows, sl)
    return {name: (out[name], tol[name] + 1e-30) for name in out}


def fp32_reference(rowptr, colidx, ncols, Q, K, V, gZ, heads, scale, items, splits):
    """The kernels' formulas in fp32 without dropout: {name: value} of Z, L, dQ, dK, dV. The forward runs the online
    softmax of every work item of (items, splits) (plan.gated_work_table) entry by entry and merges a split row's chunks
    in order, as the kernels do, since where a rescale meets +-inf decides NaN; the backward sums are order-free in
    their NaN / +-inf pattern."""
    f32 = np.float32
    nr, f = Q.shape
    C = f // heads
    sc = f32(scale)
    Q, K, V, gZ = (np.asarray(x, f32) for x in (Q, K, V, gZ))

    def hdot(A, B):                                   # [N, f] x [N, f] -> [N, heads]
        return (A * B).reshape(len(A), heads, C).sum(2, dtype=f32)

    def expand(x):                                    # [N, heads] -> [N, f]
        return np.repeat(x, C, axis=1)

    Z = np.zeros((nr, f), f32)
    L = np.full((nr, heads), -np.inf, f32)
    with np.errstate(all="ignore"):
        n_it = len(items)
        m = np.full((n_it, heads), -np.inf, f32)
        l = np.zeros((n_it, heads), f32)
        acc = np.zeros((n_it, f), f32)
        r, e0, e1 = items[:, 0], items[:, 1].astype(np.int64), items[:, 2].astype(np.int64)
        for t in range(int((e1 - e0).max()) if n_it else 0):
            act = np.flatnonzero(e0 + t < e1)
            j = np.asarray(colidx, np.int64)[e0[act] + t]
            s = hdot(Q[r[act]], K[j]) * sc
            mm, ll, aa = m[act], l[act], acc[act]
            up = s > mm
            cr = np.exp(mm - s)
            ll = np.where(up, ll * cr, ll)
            aa = np.where(expand(up), aa * expand(cr), aa)
            mm = np.where(up, s, mm)
            p = np.exp(s - mm)
            ll = ll + p
            aa = aa + expand(p) * V[j]
            m[act], l[act], acc[act] = mm, ll, aa

        def finish(rr, mm, ll, aa):
            Z[rr] = np.where(expand(ll) == 0, f32(0), aa / expand(ll))
            L[rr] = mm + np.log(ll)

        whole = items[:, 3] < 0
        finish(r[whole], m[whole], l[whole], acc[whole])
        for row, s0, n in splits:
            mm, ll, aa = m[s0:s0 + 1].copy(), l[s0:s0 + 1].copy(), acc[s0:s0 + 1].copy()
            for q in range(1, n):
                mc, lc, ac = m[s0 + q:s0 + q + 1], l[s0 + q:s0 + q + 1], acc[s0 + q:s0 + q + 1]
                up = mc > mm
                cr = np.exp(mm - mc)
                ll = np.where(up, ll * cr, ll)
                aa = np.where(expand(up), aa * expand(cr), aa)
                mm = np.where(up, mc, mm)
                b = np.exp(mc - mm)
                ll = lc * b + ll
                aa = ac * expand(b) + aa
            finish(np.array([row]), mm, ll, aa)
        rows, cols = entries(rowptr, colidx)
        s = hdot(Q[rows], K[cols]) * sc
        p = np.exp(s - L[rows])
        D = hdot(gZ, Z)
        ds = p * (hdot(gZ[rows], V[cols]) - D[rows])
        out = {"Z": Z, "L": L}
        for name, at, wt, X, ix, n, fac in (("dQ", rows, ds, K, cols, nr, sc), ("dK", cols, ds, Q, rows, ncols, sc),
                                            ("dV", cols, p, gZ, rows, ncols, None)):
            acc2 = np.zeros((n, f), f32)
            np.add.at(acc2, at, expand(wt) * X[ix])
            out[name] = acc2 * fac if fac is not None else acc2
    return out


def torch_transformer(rows, cols, n, Q, K, V, heads, scale, M=None):
    """out[i, h] = sum over the entries (i, j) of M alpha V[j, h], alpha the per-row softmax of scale <Q[i, h], K[j, h]>,
    as a differentiable torch gather / scatter (rows, cols int64 tensors; M None or [nnz, heads])."""
    f = Q.shape[1]
    C = f // heads
    s = (Q[rows].view(-1, heads, C) * K[cols].view(-1, heads, C)).sum(2) * scale
    alpha = torch.stack([po.edge_softmax(rows, s[:, h], n) for h in range(heads)], 1)
    if M is not None:
        alpha = alpha * M
    msg = (alpha[:, :, None] * V[cols].view(-1, heads, C)).reshape(-1, f)
    return torch.zeros((n, f), dtype=V.dtype).index_add(0, rows, msg)


def init_params(nlayers, f, seed):
    """[(Wk, bk, Wq, bq, Wv, bv, Ws, bs)] as transformer.PTRANSFORMER draws them on the CPU after
    torch.manual_seed(seed): lin_key, lin_query, lin_value, lin_skip = Linear(f, f). fp32 draws as fp64 numpy."""
    torch.manual_seed(seed)
    out = []
    for _ in range(nlayers):
        ls = [nn.Linear(f, f) for _ in range(4)]
        out.append(tuple(t.detach().numpy().astype(np.float64) for lin in ls for t in (lin.weight, lin.bias)))
    return out


def intended_forward(A, H, params, heads, p=0.0, seed=None, counter=None):
    """Logits of the intended model on the global graph A (its stored pattern, duplicates summed as the loader sums
    them), with every layer's dropout mask at call counter `counter` when p > 0."""
    Cm = sp.csr_matrix(A)
    Cm.sum_duplicates()
    r, c = entries(Cm.indptr, Cm.indices)
    rows, cols = torch.from_numpy(r), torch.from_numpy(c)
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for layer, prm in enumerate(params):
        Wk, bk, Wq, bq, Wv, bv, Ws, bs = (torch.as_tensor(t, dtype=torch.float64) for t in prm)
        f = Wk.shape[0]
        scale = float(np.float32(1.0 / np.sqrt(f / heads)))
        M = None
        if p > 0:
            M = do.weights(r, c, heads, p, ((seed or 0) * 2 ** 16 + layer) % 2 ** 64, counter)
        N = torch_transformer(rows, cols, n, X @ Wq.T + bq, X @ Wk.T + bk, X @ Wv.T + bv, heads, scale, M)
        X = torch.relu(N + X @ Ws.T + bs)
    return X


def intended_training(A, nlayers, f, seed, k=1, epochs=50, lr=1e-3, heads=1, p=0.0):
    """The loss curve transformer.run prints: inputs H[i, :] = i (pgat_oracle.inputs) and pgat_oracle.train's loop;
    epoch e draws its masks with counter e + 1."""
    n = A.shape[0]
    H, _ = po.inputs(n, f)
    params = [tuple(torch.tensor(t, requires_grad=True) for t in prm) for prm in init_params(nlayers, f, seed)]
    epoch = iter(range(epochs))
    return po.train(params, lambda ps: intended_forward(A, H, ps, heads, p, seed, next(epoch) + 1), n, f, k, epochs, lr)
