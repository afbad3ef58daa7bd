"""fp64 reference of GATv2 attention (op.PGATv2Attention, pgat.py --v2) — TEST INFRASTRUCTURE.

Over the stored entries (rows[e], cols[e]) of an n-row matrix (duplicates kept as separate entries), with xl, xr [n, f],
att [K, d], d = f / K and t_e = xl[cols[e]] + xr[rows[e]]:
    s_eh      = sum_c att[h, c] * LeakyReLU(t_e[h d + c])
    alpha_.h  = softmax of s_.h over each row's entries
    Z[i, h d:(h+1) d] = sum_{e in row i} alpha_eh xl[cols[e], h d:(h+1) d]
backward() is the explicit formulas of the C-ABI header (dalpha, dscore, dxr, dxl, datt), in NumPy. The training loop
draws the layer as pgat.PGATv2 does: lin_l, lin_r (Linear(f, f, bias=False)) and att (K, d), each xavier_normal with the
relu gain, in that order, and runs the forward in torch float64 with autograd.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pgat_oracle as po


def leaky(t, slope):
    return np.where(t > 0, t, t * slope)


def forward(rows, cols, n, xl, xr, att, slope):
    """(Z [n, f], alpha [nnz, K], s [nnz, K]) in fp64."""
    xl, xr, att = (np.asarray(x, dtype=np.float64) for x in (xl, xr, att))
    K, d = att.shape
    t = xl[cols] + xr[rows]                                            # [nnz, f]
    s = (leaky(t, slope).reshape(-1, K, d) * att[None]).sum(2)        # [nnz, K]
    mx = np.full((n, K), -np.inf)
    np.maximum.at(mx, rows, s)
    ex = np.exp(s - mx[rows])
    den = np.zeros((n, K))
    np.add.at(den, rows, ex)
    alpha = ex / den[rows]
    Z = np.zeros((n, K * d))
    np.add.at(Z, rows, np.repeat(alpha, d, axis=1) * xl[cols])
    return Z, alpha, s


def backward(rows, cols, n, xl, xr, att, slope, alpha, gZ):
    """(dxl, dxr, datt, dalpha, dscore) of sum(Z * gZ), by the formulas of the header."""
    xl, xr, att, gZ = (np.asarray(x, dtype=np.float64) for x in (xl, xr, att, gZ))
    K, d = att.shape
    dalpha = (gZ[rows] * xl[cols]).reshape(-1, K, d).sum(2)
    c = np.zeros((n, K))
    np.add.at(c, rows, alpha * dalpha)
    dscore = alpha * (dalpha - c[rows])
    t = xl[cols] + xr[rows]
    dsc = np.repeat(dscore, d, axis=1)
    g = dsc * att.reshape(1, -1) * np.where(t > 0, 1.0, slope)
    dxr = np.zeros_like(xr)
    np.add.at(dxr, rows, g)
    dxl = np.zeros_like(xl)
    np.add.at(dxl, cols, np.repeat(alpha, d, axis=1) * gZ[rows] + g)
    datt = (dsc * leaky(t, slope)).sum(0).reshape(K, d)
    return dxl, dxr, datt, dalpha, dscore


def forward_torch(rows, cols, n, xl, xr, att, slope):
    """The forward in torch (any dtype, autograd): rows / cols int64 tensors."""
    K, d = att.shape
    t = xl[cols] + xr[rows]
    s = (F.leaky_relu(t, slope).reshape(-1, K, d) * att[None]).sum(2)
    mx = torch.full((n, K), -float("inf"), dtype=s.dtype).scatter_reduce(0, rows[:, None].expand(-1, K), s, "amax")
    ex = torch.exp(s - mx[rows].detach())
    den = torch.zeros((n, K), dtype=s.dtype).index_add(0, rows, ex)
    alpha = ex / den[rows]
    return torch.zeros((n, K * d), dtype=s.dtype).index_add(0, rows, alpha.repeat_interleave(d, 1) * xl[cols])


def init_params(nlayers, f, seed, heads):
    """[(W_l, W_r, att)] per layer, drawn as pgat.PGATv2 draws them."""
    torch.manual_seed(seed)
    gain = nn.init.calculate_gain("relu")
    out = []
    for _ in range(nlayers):
        lin_l = nn.Linear(f, f, bias=False)
        lin_r = nn.Linear(f, f, bias=False)
        att = torch.empty(size=(heads, f // heads))
        nn.init.xavier_normal_(lin_l.weight, gain=gain)
        nn.init.xavier_normal_(lin_r.weight, gain=gain)
        nn.init.xavier_normal_(att, gain=gain)
        out.append(tuple(x.detach().numpy().astype(np.float64) for x in (lin_l.weight, lin_r.weight, att)))
    return out


def intended_training(A, nlayers, f, seed, slope, heads, k=1, epochs=50, lr=1e-3):
    """The fp64 loss curve of PGAT.py --v2 (inputs, labels, loss and Adam as the PGAT loop)."""
    n = A.shape[0]
    A = sp.csr_matrix(A)
    A.sum_duplicates()
    C = A.tocoo()
    rows, cols = torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64))
    X0 = torch.as_tensor(po.inputs(n, f)[0], dtype=torch.float64)
    params = [tuple(torch.tensor(x, requires_grad=True) for x in layer) for layer in init_params(nlayers, f, seed, heads)]

    def logits(ps):
        X = X0
        for Wl, Wr, att in ps:
            X = forward_torch(rows, cols, n, X @ Wl.T, X @ Wr.T, att, slope)
        return X
    return po.train(params, logits, n, f, k, epochs, lr)
