"""PTRANSFORMER trainer CLI — graph transformer layers (TransformerConv) over the H100 operator.

    python PTRANSFORMER.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--heads K] [--attn-dropout P] [--edge-values]
                           [--seed 0]

One layer is PyG's TransformerConv(f, f / K, heads=K, concat=True, beta=False, root_weight=True, bias=True) over the
stored pattern, followed by ReLU:

    q, k, v = lin_query(H), lin_key(H), lin_value(H)          Linear(f, f) with bias each
    N = PTransformerAttention(A, q, k, v, K)                  softmax over row i's entries of <q[i, h], k[j, h]> / sqrt(f / K)
    out = relu(N + lin_skip(H)),  lin_skip = Linear(f, f) with bias

with lin_key, lin_query, lin_value and lin_skip drawn in that order with torch's default initialisation. Everything
else is PSAGE.py's surface: flags -a -p -b -s -l -f; rank/size from SLURM_PROCID / SLURM_NPROCS with torchrun's RANK /
WORLD_SIZE as a fallback; inputs H[i, :] = i and labels i % f; L layers f -> f; parameters built on the CPU under
--seed, then moved to the device and averaged over ranks; Adam lr 1e-3; 50 epochs; gradients all-reduced / world_size;
stdout `Epoch {:05d} | Loss {:.4f}` (each rank's loss is sum_owned nll / n, the printed loss their all-reduced sum)
and `Elapsed time {:.4f}`. [k | v] is exchanged in every layer, so the plan is built with f_max = 2f. `-b gloo` is
refused: the H100 path has no CPU fallback.

--heads K (1, 2, 4 or 8, dividing f; default 1): K heads of width f / K, concatenated.

--attn-dropout P (0 <= P < 1, default 0): attention dropout with probability P on the softmax of every layer while
training, as PGAT.py's: the mask is a function of the global edge, so any partition trains the same model; layer l
draws with key seed * 2^16 + l (seed 0 when --seed is absent) and call counter epoch + 1; nothing is drawn from torch's
generator, so the parameters are those of a run without the flag.

--edge-values: TransformerConv with edge_dim = 1, the edge input being each stored entry's fp32 value of A (the plan's
lp.vals, in the order of PgcnPlan.edge_pairs()) as [nnz, 1]. Each layer then also has lin_edge = Linear(1, f,
bias=False), drawn between lin_value and lin_skip as PyG orders them, and
    E = lin_edge(vals),  N = PTransformerEdgeAttention(A, q, k, v, E, K)   keys k[j] + E_e, values v[j] + E_e
The edge input stays on the rank that owns its row. Without the flag the layers and their parameter draws are as above.
"""
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from .op import HEADS, EdgeDropout, PTransformerAttention, PTransformerEdgeAttention
from .pgat import dropout_key
from .pgcn import launch, parse_args, train


class PTRANSFORMER(nn.Module):
    """One TransformerConv layer with a ReLU on the plan handle A (a bound PgcnPlan with f_max >= 2 out_features).
    attn_dropout (an op.EdgeDropout or None) drops attention coefficients while the module is training. edge_values:
    the values of A, through lin_edge = Linear(1, out_features, bias=False), are the edge features of every entry."""

    def __init__(self, A, in_features, out_features, heads=1, attn_dropout=None, edge_values=False):
        super().__init__()
        self.A = A
        self.heads = heads
        self.attn_dropout = attn_dropout
        self.lin_key = nn.Linear(in_features, out_features)
        self.lin_query = nn.Linear(in_features, out_features)
        self.lin_value = nn.Linear(in_features, out_features)
        self.lin_edge = nn.Linear(1, out_features, bias=False) if edge_values else None
        self.lin_skip = nn.Linear(in_features, out_features)
        if edge_values:
            self.register_buffer("edge_input", torch.from_numpy(A.lp.vals.astype("float32")).reshape(-1, 1),
                                 persistent=False)

    def forward(self, H):
        drop = self.attn_dropout if self.training else None
        q, k, v = self.lin_query(H), self.lin_key(H), self.lin_value(H)
        if self.lin_edge is None:
            N = PTransformerAttention.apply(self.A, q, k, v, self.heads, None, drop)
        else:
            N = PTransformerEdgeAttention.apply(self.A, q, k, v, self.lin_edge(self.edge_input), self.heads, None,
                                                drop)
        return F.relu(N + self.lin_skip(H))


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        epochs=50, heads=1, attn_dropout=0.0, edge_values=False):
    index = iter(range(nlayers))          # train builds the layers in order

    def make(plan):
        drop = EdgeDropout(attn_dropout, dropout_key(seed, next(index)), plan.device) if attn_dropout > 0 else None
        return PTRANSFORMER(plan, nfeatures, nfeatures, heads, drop, edge_values)
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PTRANSFORMER", make, 2 * nfeatures,
                 False, transport=transport, out=out, seed=seed, epochs=epochs)


USAGE = ("usage: PTRANSFORMER.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> "
         "[--seed N] [--heads 1|2|4|8, dividing nfeatures] [--attn-dropout P, 0 <= P < 1] [--edge-values]")


def _heads(arg):
    try:
        return int(arg)
    except ValueError:
        return -1                         # refused with the usage text, as any other head count outside HEADS


def _valid(size, nlayers, nfeatures, kw):
    heads = kw.get("heads", 1)
    p = kw.get("attn_dropout", 0.0)
    return min(size, nlayers, nfeatures) >= 1 and heads in HEADS and nfeatures % heads == 0 and 0.0 <= p < 1.0


def main(argv):
    options = {"--heads": ("heads", _heads), "--attn-dropout": ("attn_dropout", float),
               "--edge-values": ("edge_values", None)}
    try:
        parsed = parse_args(argv, USAGE, options, _valid, unknown_flag_text=USAGE)
    except ValueError:
        print(USAGE, flush=True)
        sys.exit(2)
    if parsed[2][4] != "nccl":
        print(USAGE, flush=True)
        sys.exit(2)
    launch(run, *parsed)


if __name__ == "__main__":
    main(sys.argv[1:])
