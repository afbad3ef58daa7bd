"""fp64 oracle of the PGAT path (GPU/PGAT.py) — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Two semantics behind one switch (SURVEY.md §8a):

  literal   what the unmodified reference computes on each rank (GPU/PGAT.py:137-156, 204-218):
            G1 non-edges get score 0 and stay in the softmax; G2 the exchanged rows are discarded, every layer reads
            the rank's own full n-row input; G3 no LeakyReLU (score z1_i + z2_j); G4 the mask is A > 0 on values;
            G6 each rank's loss is the mean nll over all n rows, the printed loss their sum, gradients averaged.
            Pinned against the reference itself by tests/golden/pgat_*.npz (make_pgat_golden.py).
  intended  what pgcn_b200.op.PGATAttention and pgat.py compute: LeakyReLU(negative_slope) scores, a softmax over the
            stored entries of each row only (empty rows give 0), real halo exchange (one global graph), the loss
            sum_all nll / n with gradients averaged over k ranks. Written over the edge list (torch scatter ops in
            fp64), and checked against a dense -inf-masked formulation by the tests.

Parameters are fp64 copies of what the reference's / the CLI's seeded construction draws (init_params).
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn
import torch.nn.functional as F


def init_params(nlayers, f, seed):
    """[(W, a)] as GPU/PGAT.py:124-135 draws them on the CPU after torch.manual_seed(seed): nn.Linear(f, f, bias=False)
    then xavier_normal (relu gain) on W and on a (2f x 1). fp32 draws, returned as fp64 numpy."""
    torch.manual_seed(seed)
    out = []
    gain = nn.init.calculate_gain("relu")
    for _ in range(nlayers):
        lin = nn.Linear(f, f, bias=False)
        a = torch.empty(size=(2 * f, 1))
        nn.init.xavier_normal_(lin.weight, gain=gain)
        nn.init.xavier_normal_(a, gain=gain)
        out.append((lin.weight.detach().numpy().astype(np.float64), a.detach().numpy().astype(np.float64)))
    return out


def inputs(n, f):
    """H[i, :] = i and labels i % f (GPU/PGAT.py:186-192)."""
    return np.repeat(np.arange(n, dtype=np.float64)[:, None], f, axis=1), np.arange(n) % f


def train(params, logits, n, f, k, epochs, lr):
    """The loss curve the trainers print: sum_all nll / n against the labels of inputs(n, f), gradients averaged over
    k ranks, Adam(lr). params: per layer, a tuple of fp64 leaf tensors; logits(params) gives the n x f output."""
    labels = torch.from_numpy(inputs(n, f)[1])
    flat = [t for p in params for t in p]
    opt = torch.optim.Adam(flat, lr=lr)
    losses = []
    for _ in range(epochs):
        loss = F.nll_loss(F.log_softmax(logits(params), 1), labels, reduction="sum") / n
        opt.zero_grad()
        loss.backward()
        for t in flat:
            t.grad /= k
        opt.step()
        losses.append(float(loss))
    return losses


# ---- intended semantics --------------------------------------------------------------------------------------------

def edge_softmax(rows, scores, n):
    """alpha over the entries of each row (torch fp64, differentiable); rows with no entry have none."""
    mx = torch.full((n,), -float("inf"), dtype=scores.dtype).scatter_reduce(0, rows, scores, "amax")
    ex = torch.exp(scores - mx[rows].detach())
    den = torch.zeros(n, dtype=scores.dtype).index_add(0, rows, ex)
    return ex / den[rows]


def attention(rows, cols, n, Z, el, er, slope):
    """out = A(alpha) Z with alpha = edge_softmax(LeakyReLU(el[row] + er[col])) — the intended layer after the linear
    step, over the global edge list (rows, cols). Returns (out, alpha)."""
    s = F.leaky_relu(el[rows] + er[cols], slope)
    alpha = edge_softmax(rows, s, n)
    out = torch.zeros((n, Z.shape[1]), dtype=Z.dtype).index_add(0, rows, alpha[:, None] * Z[cols])
    return out, alpha


def intended_forward(A, H, params, slope):
    """Logits of the intended model on the global graph A (its stored pattern); H, params as numpy or fp64 tensors."""
    C = sp.coo_matrix(A)
    rows, cols = torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64))
    n = A.shape[0]
    X = torch.as_tensor(H, dtype=torch.float64)
    for W, a in params:
        W, a = torch.as_tensor(W, dtype=torch.float64), torch.as_tensor(a, dtype=torch.float64)
        f = W.shape[0]
        Z = X @ W.T
        X, _ = attention(rows, cols, n, Z, (Z @ a[:f]).squeeze(1), (Z @ a[f:]).squeeze(1), slope)
    return X


def intended_training(A, nlayers, f, seed, slope, k=1, epochs=50, lr=1e-3):
    """The loss curve pgat.run prints: sum_all nll / n, gradients averaged over k ranks, Adam(lr)."""
    n = A.shape[0]
    A = sp.csr_matrix(A)
    A.sum_duplicates()
    H, _ = inputs(n, f)
    params = [(torch.tensor(W, requires_grad=True), torch.tensor(a, requires_grad=True))
              for W, a in init_params(nlayers, f, seed)]
    return train(params, lambda ps: intended_forward(A, H, ps, slope), n, f, k, epochs, lr)


# ---- literal semantics (the reference's computation on one rank) --------------------------------------------------

def literal_rank_forward(A, partvec, rank, H, params):
    """Rank `rank`'s logits (n x f) as GPU/PGAT.py computes them: the dense n x n local matrix holds the rank's rows
    (:53-65), each layer takes the full previous output (G2), scores z1_i + z2_j (G3), zero on non-edges that stay in
    the softmax (G1), mask A > 0 on values (G4)."""
    A = sp.coo_matrix(A)
    n = A.shape[0]
    own = np.asarray(partvec)[A.row] == rank
    Aloc = torch.zeros((n, n), dtype=torch.float64)
    Aloc.index_put_((torch.from_numpy(A.row[own].astype(np.int64)), torch.from_numpy(A.col[own].astype(np.int64))),
                    torch.from_numpy(A.data[own].astype(np.float64)), accumulate=True)
    X = torch.as_tensor(H, dtype=torch.float64)
    for W, a in params:
        f = W.shape[0]
        Z = X @ W.T
        att = Z @ a[:f] + (Z @ a[f:]).T
        att = torch.where(Aloc > 0, att, torch.zeros_like(att))
        X = torch.softmax(att, 1) @ Z
    return X


def literal_rank_grads(A, partvec, rank, H, params, labels):
    """(logits, loss, [(dW, da)]) of one rank before gradient averaging: loss = mean nll over all n rows (G6)."""
    ps = [(torch.tensor(W, requires_grad=True), torch.tensor(a, requires_grad=True)) for W, a in params]
    logits = literal_rank_forward(A, partvec, rank, H, ps)
    loss = F.nll_loss(F.log_softmax(logits, 1), torch.as_tensor(labels))
    loss.backward()
    return logits.detach().numpy(), float(loss.detach()), [(W.grad.numpy(), a.grad.numpy()) for W, a in ps]


def literal_training(A, partvec, k, nlayers, f, seed, epochs=50, lr=1e-3):
    """The reference's printed loss curve: the sum over ranks of each rank's loss, gradients averaged over ranks."""
    n = A.shape[0]
    H, labels = inputs(n, f)
    labels = torch.from_numpy(labels)
    params = [(torch.tensor(W, requires_grad=True), torch.tensor(a, requires_grad=True))
              for W, a in init_params(nlayers, f, seed)]
    flat = [t for p in params for t in p]
    opt = torch.optim.Adam(flat, lr=lr)
    losses = []
    for _ in range(epochs):
        opt.zero_grad()
        total = 0.0
        for r in range(k):
            loss = F.nll_loss(F.log_softmax(literal_rank_forward(A, partvec, r, H, params), 1), labels)
            (loss / k).backward()
            total += float(loss)
        opt.step()
        losses.append(total)
    return losses
