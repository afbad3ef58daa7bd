"""PGINE trainer CLI — GINE layers with an edge-feature stream over the H100 operator.

    python PGINE.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--seed 0] [--transport auto|p2p|nccl]

The network is a stack of GINE layers (Hu et al., "Strategies for Pre-training Graph Neural Networks"; PyG's
GINEConv(nn, edge_dim=1)) with a residual ReLU. The edge input is each stored entry's fp32 value of A (the plan's
lp.vals, in the order of PgcnPlan.edge_pairs()) as [nnz, 1], which each layer's lin_edge = Linear(1, f) maps to width f:

    Z = PGINE(plan, h, lin_edge(e0))                 Z[i] = sum over the stored entries (i, j) of relu(h[j] + E_e)
    h = h + relu(mlp((1 + eps) h + Z))               mlp = Linear(f, f), ReLU, Linear(f, f)

with eps = 0, fixed, and the logits are the last h. Parameters are drawn with torch's default initialisation in this
order, per layer: lin_edge, mlp[0], mlp[2]. Everything else is PGATED.py's surface: flags -a -p -b -s -l -f; rank/size
from SLURM_PROCID / SLURM_NPROCS with torchrun's RANK / WORLD_SIZE as a fallback; inputs H[i, :] = i and labels i % f;
parameters built on the CPU under --seed, then moved to the device and averaged over ranks; Adam lr 1e-3; 50 epochs;
gradients all-reduced / world_size; stdout `Epoch {:05d} | Loss {:.4f}` (each rank's loss is sum_owned nll / n, the
printed loss their all-reduced sum) and `Elapsed time {:.4f}`. h is exchanged in every layer, so the plan is built with
f_max = f; the edge features stay on the rank that owns their row. `-b gloo` is refused: the H100 path has no CPU
fallback.
"""
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import op
from .pgcn import launch, parse_args, train


class GINELayer(nn.Module):
    """One GINE layer (residual, ReLU) on the plan handle A (a bound PgcnPlan with f_max >= f): forward(h, e0) -> h,
    h [rows, f] in the plan's layout, e0 [nnz_local, 1] the edge input in edge_pairs() order. eps is GIN's self weight,
    a parameter when train_eps."""

    def __init__(self, A, features, eps=0.0, train_eps=False):
        super().__init__()
        self.A = A
        self.lin_edge = nn.Linear(1, features)
        self.mlp = nn.Sequential(nn.Linear(features, features), nn.ReLU(), nn.Linear(features, features))
        if train_eps:
            self.eps = nn.Parameter(torch.tensor([float(eps)]))
        else:
            self.register_buffer("eps", torch.tensor([float(eps)]))

    def forward(self, h, e0):
        Z = op.PGINE.apply(self.A, h, self.lin_edge(e0))
        return h + F.relu(self.mlp((1 + self.eps) * h + Z))


class PGINE(nn.Module):
    """`nlayers` GINE layers of width f on the plan handle A; forward(H) gives the logits."""

    def __init__(self, A, features, nlayers, eps=0.0, train_eps=False):
        super().__init__()
        self.A = A
        self.layers = nn.ModuleList([GINELayer(A, features, eps, train_eps) for _ in range(nlayers)])
        self.register_buffer("edge_input", torch.from_numpy(A.lp.vals.astype("float32")).reshape(-1, 1),
                             persistent=False)

    def forward(self, H):
        h = H
        for layer in self.layers:
            h = layer(h, self.edge_input)
        return h


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        epochs=50):
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PGINE", None, nfeatures,
                 False, transport=transport, out=out, seed=seed, epochs=epochs,
                 model=lambda plan: PGINE(plan, nfeatures, nlayers))


USAGE = "usage: PGINE.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> [--seed N]"


def main(argv):
    try:
        parsed = parse_args(argv, USAGE, valid=lambda size, nlayers, nfeatures, kw: min(size, nlayers, nfeatures) >= 1,
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
