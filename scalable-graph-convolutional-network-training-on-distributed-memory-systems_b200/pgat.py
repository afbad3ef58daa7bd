"""PGAT trainer CLI — the reference's graph-attention surface (GPU/PGAT.py:124-286) over the H100 operator.

    python PGAT.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--seed 0] [--negative-slope 1.0] [--heads K]

Kept from the reference: flags -a -p -b -s -l -f; rank/size from SLURM_PROCID / SLURM_NPROCS with torchrun's RANK /
WORLD_SIZE as a fallback (as pgcn.py); inputs H[i, :] = i (:186-188) and labels i % f (:192); L x PGAT layers with the
reference's parameters and initialisation (:124-135: Linear(f, f, bias=False) and a (2f x 1) attention vector, both
xavier_normal with the relu gain) averaged over ranks at start (:166-170); Adam lr 1e-3 (:200); 50 epochs (:204);
gradients all-reduced / world_size (:158-162); stdout `Epoch {:05d} | Loss {:.4f}` and `Elapsed time {:.4f}`.

Different by design (SURVEY.md §8a, the quirks G1-G6 of DESIGN.md §1): the softmax runs over each row's stored entries
only (the reference gives non-edges score 0 and keeps them in the softmax); halo rows really are exchanged in every
layer; the score goes through LeakyReLU(negative_slope), whose default here, 1.0, is the reference's raw score; the
flags are honoured (the reference overwrites them); every tensor is [m_local, f], each rank's loss is
sum_owned nll / n and the printed loss is its all-reduced sum, the global mean. `-b gloo` is refused: the H100 path has no
CPU fallback (the fp64 oracle lives under oracle/ and is test infrastructure).

--heads K (1, 2, 4 or 8, dividing f; default 1): K attention heads of width d = f / K per layer, concatenated, so every
layer stays f -> f. K = 1 is the single-head layer above, with the same parameter draws. K > 1: Linear(f, f, bias=False)
and a (2d x K) attention matrix, both xavier_normal with the relu gain in that order; el[:, h] = Z_h a[:d, h] and
er[:, h] = Z_h a[d:, h] for head h's slice Z_h of Z (op.PGATMultiHeadAttention).

--attn-dropout P (0 <= P < 1, default 0): attention dropout with probability P between the softmax and the aggregation
of every layer while training (op.EdgeDropout, the GAT paper's recipe uses 0.6). The mask is a function of the global
edge, so any partition trains the same model. Layer l draws with key seed * 2^16 + l (seed 0 when --seed is absent) and
call counter epoch + 1; nothing is drawn from torch's generator, so the parameters are those of a run without the flag.
Taken with --v2 only together with --edge-values (below).

--v2: GATv2 layers instead (dynamic attention, op.PGATv2Attention), with --heads K as above. Per layer lin_l and lin_r
(Linear(f, f, bias=False)) and att (K x d), drawn in that order, each xavier_normal with the relu gain; the layer is
PyG GATv2Conv(share_weights=False, concat=True, bias=False, add_self_loops=False) over the stored pattern.

--v2 --edge-values: GATv2Conv with edge_dim = 1, the edge input being each stored entry's fp32 value of A (the plan's
lp.vals, in the order of PgcnPlan.edge_pairs()) as [nnz, 1]. Each layer then also has lin_edge = Linear(1, f,
bias=False) with torch's default initialisation, drawn after lin_l, lin_r and att, and
    E = lin_edge(vals),  out = PGATv2EdgeAttention(A, lin_l(H), lin_r(H), att, E)    score of (XR[i] + XL[j]) + E_e
The edge input stays on the rank that owns its row. Without the flag the layers and their parameter draws are as above.
--attn-dropout P is taken with --v2 only together with --edge-values (the edge kernels draw the mask; the GATv2 kernels
without edges do not), with the keys and counters above. --edge-values without --v2 is refused.
"""
import sys

import torch
import torch.nn as nn

from .op import HEADS, EdgeDropout, PGATAttention, PGATMultiHeadAttention, PGATv2Attention, PGATv2EdgeAttention
from .pgcn import launch, parse_args, train


class PGAT(nn.Module):
    """GPU/PGAT.py:124-148 with the plan handle in place of the dense matrix and a sparse edge softmax. attn_dropout (an
    op.EdgeDropout or None) drops attention coefficients while the module is training; eval mode runs without it."""

    def __init__(self, A, in_features, out_features, negative_slope=0.2, heads=1, attn_dropout=None):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.A = A
        self.negative_slope = negative_slope
        self.heads = heads
        self.attn_dropout = attn_dropout
        self.linear = nn.Linear(in_features, out_features, bias=False)
        d = out_features // heads
        self.attention = nn.Parameter(torch.empty(size=(2 * out_features, 1) if heads == 1 else (2 * d, heads)))
        self.reset_parameters()

    def reset_parameters(self):
        gain = nn.init.calculate_gain("relu")
        nn.init.xavier_normal_(self.linear.weight, gain=gain)
        nn.init.xavier_normal_(self.attention, gain=gain)

    def forward(self, H):
        Z = self.linear(H)
        f = self.out_features
        drop = self.attn_dropout if self.training else None
        if self.heads > 1:
            d = f // self.heads
            Zh = Z.view(Z.shape[0], self.heads, d)
            el = torch.einsum("nhd,dh->nh", Zh, self.attention[:d])
            er = torch.einsum("nhd,dh->nh", Zh, self.attention[d:])
            return PGATMultiHeadAttention.apply(self.A, Z, el, er, self.negative_slope, drop)
        el = torch.matmul(Z, self.attention[:f, :]).squeeze(1)
        er = torch.matmul(Z, self.attention[f:, :]).squeeze(1)
        return PGATAttention.apply(self.A, Z, el, er, self.negative_slope, drop)


class PGATv2(nn.Module):
    """GATv2 layer f -> f with K heads: out = PGATv2Attention(A, lin_l(H), lin_r(H), att). edge_values: the values of A,
    through lin_edge = Linear(1, out_features, bias=False) (drawn after the other parameters), are the edge features of
    every entry, and out = PGATv2EdgeAttention(A, lin_l(H), lin_r(H), att, lin_edge(vals)). attn_dropout (an
    op.EdgeDropout or None) drops attention coefficients while the module is training; it needs edge_values."""

    def __init__(self, A, in_features, out_features, negative_slope=0.2, heads=1, edge_values=False,
                 attn_dropout=None):
        super().__init__()
        if attn_dropout is not None and not edge_values:
            raise ValueError("GATv2 attention dropout is drawn by the edge-feature kernels: it needs edge_values=True")
        self.A = A
        self.negative_slope = negative_slope
        self.attn_dropout = attn_dropout
        self.lin_l = nn.Linear(in_features, out_features, bias=False)
        self.lin_r = nn.Linear(in_features, out_features, bias=False)
        self.att = nn.Parameter(torch.empty(size=(heads, out_features // heads)))
        self.reset_parameters()
        self.lin_edge = nn.Linear(1, out_features, bias=False) if edge_values else None
        if edge_values:
            self.register_buffer("edge_input", torch.from_numpy(A.lp.vals.astype("float32")).reshape(-1, 1),
                                 persistent=False)

    def reset_parameters(self):
        gain = nn.init.calculate_gain("relu")
        nn.init.xavier_normal_(self.lin_l.weight, gain=gain)
        nn.init.xavier_normal_(self.lin_r.weight, gain=gain)
        nn.init.xavier_normal_(self.att, gain=gain)

    def forward(self, H):
        if self.lin_edge is None:
            return PGATv2Attention.apply(self.A, self.lin_l(H), self.lin_r(H), self.att, self.negative_slope)
        drop = self.attn_dropout if self.training else None
        return PGATv2EdgeAttention.apply(self.A, self.lin_l(H), self.lin_r(H), self.att,
                                         self.lin_edge(self.edge_input), self.negative_slope, drop)


def dropout_key(seed, layer):
    """The attention-dropout key of layer `layer` (0-based) under --seed `seed` (None: 0)."""
    return ((seed or 0) * 2 ** 16 + layer) % 2 ** 64


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        negative_slope=1.0, epochs=50, heads=1, v2=False, attn_dropout=0.0, edge_values=False):
    # the multi-head backward gets d_er from an aggregation of width 4 K (PGATMultiHeadAttention)
    f_max = nfeatures if heads == 1 or v2 else max(nfeatures, 4 * heads)
    index = iter(range(nlayers))          # train builds the layers in order

    def make(plan):
        drop = EdgeDropout(attn_dropout, dropout_key(seed, next(index)), plan.device) if attn_dropout > 0 else None
        if v2:
            return PGATv2(plan, nfeatures, nfeatures, negative_slope, heads, edge_values, drop)
        return PGAT(plan, nfeatures, nfeatures, negative_slope, heads, drop)
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PGAT", make, f_max, True,
                 transport=transport, out=out, seed=seed, epochs=epochs)


USAGE = ("usage: PGAT.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> "
         "[--seed N] [--negative-slope S] [--heads 1|2|4|8, dividing nfeatures] [--attn-dropout P, 0 <= P < 1] [--v2] "
         "[--edge-values, with --v2; --attn-dropout with --v2 needs it]")


def _heads(arg):
    try:
        return int(arg)
    except ValueError:
        return -1                         # refused with the usage text, as any other head count outside HEADS


def _valid(size, nlayers, nfeatures, kw):
    heads = kw.get("heads", 1)
    p = kw.get("attn_dropout", 0.0)
    return (heads in HEADS and nfeatures % heads == 0 and 0.0 <= p < 1.0
            and not ("attn_dropout" in kw and kw.get("v2") and not kw.get("edge_values"))
            and not (kw.get("edge_values") and not kw.get("v2")))


def main(argv):
    options = {"--negative-slope": ("negative_slope", float), "--heads": ("heads", _heads), "--v2": ("v2", None),
               "--attn-dropout": ("attn_dropout", float), "--edge-values": ("edge_values", None)}
    launch(run, *parse_args(argv, USAGE, options, _valid))


if __name__ == "__main__":
    main(sys.argv[1:])
