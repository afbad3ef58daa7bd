"""PGATED trainer CLI — residual gated graph convolutions (ResGatedGraphConv) over the H100 operator.

    python PGATED.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--seed 0] [--transport auto|p2p|nccl]

One layer is PyG's ResGatedGraphConv(f, f, act=Sigmoid(), root_weight=True, bias=True) over the stored pattern,
followed by ReLU:

    k, q, v = lin_key(H), lin_query(H), lin_value(H)          Linear(f, f) with bias each
    N = PSpMMGated(A, k, q, v)                                N[i] = sum_{(i, j) stored} sigmoid(k[i] + q[j]) * v[j]
    out = relu(N + lin_skip(H) + bias),  lin_skip = Linear(f, f, bias=False), bias = zeros(f)

drawn in that order with torch's default initialisation. Everything else is PSAGE.py's surface: flags -a -p -b -s -l
-f; rank/size from SLURM_PROCID / SLURM_NPROCS with torchrun's RANK / WORLD_SIZE as a fallback; inputs H[i, :] = i and
labels i % f; L layers f -> f; parameters built on the CPU under --seed, then moved to the device and averaged over
ranks; Adam lr 1e-3; 50 epochs; gradients all-reduced / world_size; stdout `Epoch {:05d} | Loss {:.4f}` (each rank's
loss is sum_owned nll / n, the printed loss their all-reduced sum) and `Elapsed time {:.4f}`. [q | v] is exchanged in
every layer, so the plan is built with f_max = 2f. `-b gloo` is refused: the H100 path has no CPU fallback.
"""
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from .op import PSpMMGated
from .pgcn import launch, parse_args, train


class PGATED(nn.Module):
    """One ResGatedGraphConv layer with a ReLU on the plan handle A (a bound PgcnPlan with f_max >= 2 out_features)."""

    def __init__(self, A, in_features, out_features):
        super().__init__()
        self.A = A
        self.lin_key = nn.Linear(in_features, out_features)
        self.lin_query = nn.Linear(in_features, out_features)
        self.lin_value = nn.Linear(in_features, out_features)
        self.lin_skip = nn.Linear(in_features, out_features, bias=False)
        self.bias = nn.Parameter(torch.zeros(out_features))

    def forward(self, H):
        N = PSpMMGated.apply(self.A, self.lin_key(H), self.lin_query(H), self.lin_value(H))
        return F.relu(N + self.lin_skip(H) + self.bias)


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        epochs=50):
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PGATED",
                 lambda plan: PGATED(plan, nfeatures, nfeatures), 2 * nfeatures, False,
                 transport=transport, out=out, seed=seed, epochs=epochs)


USAGE = "usage: PGATED.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> [--seed N]"


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
