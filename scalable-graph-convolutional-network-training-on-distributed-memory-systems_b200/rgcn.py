"""PRGCN trainer CLI — R-GCN layers over typed edges on the H100 operator.

    python PRGCN.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 --relations 4 [--bases 2] [--seed 0]

The network is a stack of R-GCN layers (Schlichtkrull et al., "Modeling Relational Data with Graph Convolutional
Networks"; PyG's RGCNConv(f, f, R, num_bases, aggr="mean")) with a ReLU between layers; the logits are the last
layer's output. Each layer computes

    Z = PRGCN(plan, h, rel, R)                   Z[i, r] = mean over the stored entries (i, j) with rel = r of h[j]
    out = h @ root + bias + Z.reshape(rows, R f) @ W.reshape(R f, f)

with W = weight, or W[r] = sum_b comp[r, b] basis[b] with --bases B. The relation of each stored entry comes from
relation_hash of its global (row, column), so every partition of the graph gives an entry the same type; a user with
real typed edges passes their own rel, in edge_pairs() order, to RGCNLayer. Parameters are drawn on the CPU under --seed
in this order, per layer: weight ([R, f, f]; with bases the basis [B, f, f], then comp [R, B]), then root [f, f], each
uniform in +-sqrt(6 / (fan_in + fan_out)) of its last two dimensions (PyG's glorot); the bias starts at zero and is
not drawn. Everything else is PGINE.py's surface: flags -a -p -b -s -l -f; rank/size from SLURM_PROCID / SLURM_NPROCS
with torchrun's RANK / WORLD_SIZE as a fallback; inputs H[i, :] = i and labels i % f; parameters moved to the device
and averaged over ranks; Adam lr 1e-3; 50 epochs; gradients all-reduced / world_size; stdout
`Epoch {:05d} | Loss {:.4f}` (each rank's loss is sum_owned nll / n, the printed loss their all-reduced sum) and
`Elapsed time {:.4f}`. h is exchanged in every layer, f floats per row whatever R is, so the plan is built with
f_max = f. `-b gloo` is refused: the H100 path has no CPU fallback.
"""
import math
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import op
from .pgcn import launch, parse_args, train

# relation_hash's constants: Knuth's multiplicative constant for the row, a small odd one for the column
HASH_ROW, HASH_COL = 2654435761, 40503


def relation_hash(pairs, R):
    """Synthetic relation types of the entries `pairs` (an int [nnz, 2] tensor of global (row, column), as
    PgcnPlan.edge_pairs() gives): rel = ((row * 2654435761 + col * 40503) mod 2^32 >> 16) mod R, an int64 tensor
    [nnz] on pairs' device. It depends on the global pair only, so every partition types an entry alike."""
    p = pairs.to(torch.int64)
    h = (p[:, 0] * HASH_ROW + p[:, 1] * HASH_COL) & 0xFFFFFFFF
    return (h >> 16) % int(R)


def _glorot(t):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


class RGCNLayer(nn.Module):
    """One R-GCN layer, PyG RGCNConv's semantics, on the plan handle A (a bound PgcnPlan with f_max >= f_in):
    forward(h) -> [rows, f_out], h [rows, f_in] in the plan's layout. rel: the relation of every local entry, an integer
    tensor [nnz_local] in edge_pairs() order with values in [0, R). num_bases: the basis decomposition
    W[r] = sum_b comp[r, b] basis[b] (None: one full weight per relation). aggr: "mean" (per relation, PyG's default)
    or "add". root_weight adds h @ root, bias a learned bias. The relational aggregation runs in libpgcn_rgcn.so
    (op.PRGCN); the GEMM and the basis decomposition stay in PyTorch."""

    def __init__(self, A, rel, R, f_in, f_out, num_bases=None, aggr="mean", root_weight=True, bias=True):
        super().__init__()
        if aggr not in op.RGCN_AGGRS:
            raise ValueError("aggr=%r: R-GCN aggregates with one of %s" % (aggr, ", ".join(map(repr, op.RGCN_AGGRS))))
        if num_bases is not None and num_bases < 1:
            raise ValueError("num_bases=%r: need at least one basis" % (num_bases,))
        self.A, self.rel, self.R, self.aggr = A, rel, int(R), aggr
        self.f_in, self.f_out = f_in, f_out
        if num_bases is None:
            self.weight = nn.Parameter(torch.empty(self.R, f_in, f_out))
            _glorot(self.weight)
            self.comp = None
        else:
            self.weight = nn.Parameter(torch.empty(num_bases, f_in, f_out))
            _glorot(self.weight)
            self.comp = nn.Parameter(torch.empty(self.R, num_bases))
            _glorot(self.comp)
        self.root = None
        if root_weight:
            self.root = nn.Parameter(torch.empty(f_in, f_out))
            _glorot(self.root)
        self.bias = nn.Parameter(torch.zeros(f_out)) if bias else None

    def relation_weights(self):
        """W [R, f_in, f_out]: the weights, or their basis decomposition."""
        if self.comp is None:
            return self.weight
        return (self.comp @ self.weight.reshape(self.weight.shape[0], -1)).reshape(self.R, self.f_in, self.f_out)

    def forward(self, h):
        Z = op.PRGCN.apply(self.A, h, self.rel, self.R, None, self.aggr)
        W = self.relation_weights().reshape(self.R * self.f_in, self.f_out)
        out = Z.reshape(Z.shape[0], self.R * self.f_in) @ W
        if self.root is not None:
            out = out + h @ self.root
        if self.bias is not None:
            out = out + self.bias
        return out


class PRGCN(nn.Module):
    """`nlayers` R-GCN layers of width f on the plan handle A with a ReLU between them, over the synthetic relations
    relation_hash(A.edge_pairs(), R); forward(H) gives the logits."""

    def __init__(self, A, features, nlayers, R, num_bases=None):
        super().__init__()
        self.A = A
        rel = relation_hash(A.edge_pairs(), R)
        self.layers = nn.ModuleList([RGCNLayer(A, rel, R, features, features, num_bases) for _ in range(nlayers)])

    def forward(self, H):
        h = H
        for i, layer in enumerate(self.layers):
            h = layer(h)
            if i + 1 < len(self.layers):
                h = F.relu(h)
        return h


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, relations=None, bases=None, transport="auto",
        out=sys.stdout, seed=None, epochs=50):
    if relations is None or relations < 1:
        raise ValueError("relations=%r: PRGCN needs --relations R >= 1" % (relations,))
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PRGCN", None, nfeatures,
                 False, transport=transport, out=out, seed=seed, epochs=epochs,
                 model=lambda plan: PRGCN(plan, nfeatures, nlayers, relations, bases))


USAGE = ("usage: PRGCN.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> --relations <R> "
         "[--bases <B>] [--seed N]")


def main(argv):
    def valid(size, nlayers, nfeatures, kw):
        return (min(size, nlayers, nfeatures) >= 1 and kw.get("relations", 0) >= 1
                and kw.get("bases", 1) >= 1)
    try:
        parsed = parse_args(argv, USAGE, {"--relations": ("relations", int), "--bases": ("bases", int)}, valid=valid,
                            unknown_flag_text=USAGE)
    except ValueError:
        print(USAGE, flush=True)
        sys.exit(2)
    if parsed[2][4] != "nccl":
        print(USAGE, flush=True)
        sys.exit(2)
    launch(run, *parsed)


if __name__ == "__main__":
    main(sys.argv[1:])
