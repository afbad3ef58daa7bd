"""NumPy / fp64 reference of edge dropout (include/pgcn_dropout.h, op.EdgeDropout, PGAT.py --attn-dropout) — TEST
INFRASTRUCTURE.

  * philox4x32_10: Philox4x32-10 vectorised over counters, with the Random123 constants;
  * keep / apply: the mask rule, exact in fp32: entry (gi, gj), head h keeps iff word h & 3 of Philox(counter = (gi, gj,
    c, h >> 2), key) >= floor(p 2^32), and y = x * float32(1 / (1 - p)) or x * 0;
  * attention: fp64 single- and multi-head sparse attention with the mask between the softmax and the aggregation, from
    oracle/pgat_oracle.edge_softmax and tests/pgat_heads_oracle (neither is changed);
  * intended_training: PGAT.py's loss curve with --attn-dropout, layer l keyed seed * 2^16 + l, counter epoch + 1.
"""
import math

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn.functional as F

import pgat_heads_oracle as ho
from oracle import pgat_oracle as po

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32-valued [N, 4], key: (k0, k1). Returns uint32 [N, 4]."""
    c = [np.asarray(ctr, dtype=np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & LO, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & LO]
    return np.stack(c, 1).astype(np.uint32)


def constants(p):
    """(threshold, scale) of drop probability p: floor(p 2^32) and float32(1 / (1 - p))."""
    assert 0.0 <= p < 1.0
    return int(math.floor(p * 4294967296.0)), np.float32(1.0 / (1.0 - p))


def keep(gi, gj, heads, p, key, counter):
    """bool [N, heads]: which (entry, head) the mask keeps; gi, gj the entries' global row and column."""
    gi, gj = np.asarray(gi, dtype=np.uint64), np.asarray(gj, dtype=np.uint64)
    T, _ = constants(p)
    k0, k1 = key % 2 ** 32, (key >> 32) % 2 ** 32
    out = np.empty((gi.shape[0], heads), dtype=bool)
    for q in range((heads + 3) // 4):
        ctr = np.stack([gi, gj, np.full_like(gi, counter % 2 ** 32), np.full_like(gi, q)], 1)
        w = philox4x32_10(ctr, (k0, k1))
        for j in range(min(4, heads - 4 * q)):
            out[:, 4 * q + j] = w[:, j] >= T
    return out


def apply(x, gi, gj, p, key, counter):
    """The kernel's output for x (fp32 [N] or [N, K]), bit for bit."""
    x = np.asarray(x, dtype=np.float32)
    x2 = x.reshape(x.shape[0], -1)
    kp = keep(gi, gj, x2.shape[1], p, key, counter)
    _, scale = constants(p)
    with np.errstate(invalid="ignore", over="ignore"):
        y = np.where(kp, x2 * scale, x2 * np.float32(0))
    return y.astype(np.float32).reshape(x.shape)


def weights(gi, gj, heads, p, key, counter):
    """fp64 [N, heads] factor of the mask: float32(1 / (1 - p)) where kept, 0 where dropped."""
    _, scale = constants(p)
    return torch.from_numpy(keep(gi, gj, heads, p, key, counter) * np.float64(scale))


def attention(rows, cols, n, Z, el, er, slope, mask, heads=1):
    """(out, alpha): pgat_heads_oracle.attention with alpha_d = alpha * mask ([nnz, heads] fp64) aggregating Z."""
    d = Z.shape[1] // heads
    el = el.reshape(n, heads)
    er = er.reshape(n, heads)
    outs, alphas = [], []
    for h in range(heads):
        s = F.leaky_relu(el[rows, h] + er[cols, h], slope)
        a = po.edge_softmax(rows, s, n)
        ad = a * mask[:, h]
        outs.append(torch.zeros((n, d), dtype=Z.dtype).index_add(0, rows, ad[:, None] * Z[cols, h * d:(h + 1) * d]))
        alphas.append(a)
    return torch.cat(outs, 1), torch.stack(alphas, 1)


def intended_forward(A, H, params, slope, p, seed, counter, heads=1):
    """Logits of PGAT.py --attn-dropout p on the global graph A, every layer's mask at call counter `counter`."""
    C = sp.coo_matrix(A)
    rows, cols = torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64))
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for l, (W, a) in enumerate(params):
        W, a = torch.as_tensor(W, dtype=torch.float64), torch.as_tensor(a, dtype=torch.float64)
        Z = X @ W.T
        if heads == 1:
            f = W.shape[0]
            el, er = (Z @ a[:f]).squeeze(1), (Z @ a[f:]).squeeze(1)
        else:
            el, er = ho.scores(Z, a, heads)
        mask = weights(C.row, C.col, heads, p, (seed * 2 ** 16 + l) % 2 ** 64, counter)
        X, _ = attention(rows, cols, n, Z, el, er, slope, mask, heads)
    return X


def intended_training(A, nlayers, f, seed, slope, p, k=1, epochs=50, lr=1e-3, heads=1):
    """The loss curve PGAT.py -l nlayers -f f --seed seed --negative-slope slope --attn-dropout p [--heads heads] prints:
    epoch e draws its masks with counter e + 1."""
    n = A.shape[0]
    A = sp.csr_matrix(A)
    A.sum_duplicates()
    H, _ = po.inputs(n, f)
    params = [(torch.tensor(W, requires_grad=True), torch.tensor(a, requires_grad=True))
              for W, a in ho.init_params(nlayers, f, seed, heads)]
    epoch = iter(range(epochs))
    return po.train(params, lambda ps: intended_forward(A, H, ps, slope, p, seed, next(epoch) + 1, heads), n, f, k,
                    epochs, lr)
