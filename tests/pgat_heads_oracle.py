"""fp64 reference of multi-head sparse graph attention (op.PGATMultiHeadAttention, pgat.py --heads) — TEST
INFRASTRUCTURE. It extends oracle/pgat_oracle.py's intended semantics with a `heads` argument and leaves that module as
it is: heads=1 calls its functions unchanged.

With K heads of width d = f / K, head h aggregates its slice Z[:, h d:(h+1) d] with its own softmax alpha[:, h] of
LeakyReLU(el[row, h] + er[col, h]), and the heads are concatenated. Parameters per layer: W (f x f) and a (2d x K), drawn
as pgat.PGAT draws them (Linear then xavier_normal with the relu gain on W, then on a); el[:, h] = Z_h a[:d, h] and
er[:, h] = Z_h a[d:, h].
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from oracle import pgat_oracle as po


def init_params(nlayers, f, seed, heads=1):
    if heads == 1:
        return po.init_params(nlayers, f, seed)
    torch.manual_seed(seed)
    out = []
    gain = nn.init.calculate_gain("relu")
    for _ in range(nlayers):
        lin = nn.Linear(f, f, bias=False)
        a = torch.empty(size=(2 * (f // heads), heads))
        nn.init.xavier_normal_(lin.weight, gain=gain)
        nn.init.xavier_normal_(a, gain=gain)
        out.append((lin.weight.detach().numpy().astype(np.float64), a.detach().numpy().astype(np.float64)))
    return out


def attention(rows, cols, n, Z, el, er, slope, heads=1):
    """(out, alpha): el, er are [n, K] (heads > 1) and alpha is [nnz, K]; heads=1 is pgat_oracle.attention."""
    if heads == 1:
        return po.attention(rows, cols, n, Z, el, er, slope)
    d = Z.shape[1] // heads
    outs, alphas = [], []
    for h in range(heads):
        o, a = po.attention(rows, cols, n, Z[:, h * d:(h + 1) * d], el[:, h], er[:, h], slope)
        outs.append(o)
        alphas.append(a)
    return torch.cat(outs, 1), torch.stack(alphas, 1)


def scores(Z, a, heads):
    """(el, er) of one layer from Z = X W^T and its attention parameter a (2d x K)."""
    d = Z.shape[1] // heads
    Zh = Z.reshape(Z.shape[0], heads, d)
    return torch.einsum("nhd,dh->nh", Zh, a[:d]), torch.einsum("nhd,dh->nh", Zh, a[d:])


def intended_forward(A, H, params, slope, heads=1):
    if heads == 1:
        return po.intended_forward(A, H, params, slope)
    C = sp.coo_matrix(A)
    rows, cols = torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64))
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for W, a in params:
        W, a = torch.as_tensor(W, dtype=torch.float64), torch.as_tensor(a, dtype=torch.float64)
        Z = X @ W.T
        el, er = scores(Z, a, heads)
        X, _ = attention(rows, cols, n, Z, el, er, slope, heads)
    return X


def intended_training(A, nlayers, f, seed, slope, k=1, epochs=50, lr=1e-3, heads=1):
    if heads == 1:
        return po.intended_training(A, nlayers, f, seed, slope, k=k, epochs=epochs, lr=lr)
    n = A.shape[0]
    A = sp.csr_matrix(A)
    A.sum_duplicates()
    H, _ = po.inputs(n, f)
    params = [(torch.tensor(W, requires_grad=True), torch.tensor(a, requires_grad=True))
              for W, a in init_params(nlayers, f, seed, heads)]
    return po.train(params, lambda ps: intended_forward(A, H, ps, slope, heads), n, f, k, epochs, lr)
