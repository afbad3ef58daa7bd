"""PSAGE trainer CLI — GraphSAGE with the max-pool aggregator over the H100 operator.

    python PSAGE.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--seed 0] [--transport auto|p2p|nccl]

One layer is the "pool" form of DGL's SAGEConv(aggregator_type="pool") with PyG's aggr="max":

    P = relu(pool(H)),  pool = Linear(f, f, bias=True)
    N = PSpMMMax(A, P)                      the element-wise maximum over each row's stored entries (op.PSpMMMax)
    out = relu(self_lin(H) + neigh_lin(N)),  self_lin, neigh_lin = Linear(f, f, bias=False)

drawn in that order with torch's default initialisation. Everything else is PGAT.py's surface: flags -a -p -b -s -l -f;
rank/size from SLURM_PROCID / SLURM_NPROCS with torchrun's RANK / WORLD_SIZE as a fallback; inputs H[i, :] = i and labels
i % f; L layers f -> f; parameters built on the CPU under --seed, then moved to the device and averaged over ranks;
Adam lr 1e-3; 50 epochs; gradients all-reduced / world_size; stdout `Epoch {:05d} | Loss {:.4f}` (each rank's loss is
sum_owned nll / n, the printed loss their all-reduced sum) and `Elapsed time {:.4f}`. The halo rows are exchanged in
every layer. `-b gloo` is refused: the H100 path has no CPU fallback.
"""
import sys

import torch.nn as nn
import torch.nn.functional as F

from .op import PSpMMMax
from .pgcn import launch, parse_args, train


class PSAGE(nn.Module):
    """One GraphSAGE layer with the max-pool aggregator on the plan handle A (a bound PgcnPlan)."""

    def __init__(self, A, in_features, out_features):
        super().__init__()
        self.A = A
        self.pool = nn.Linear(in_features, in_features, bias=True)
        self.self_lin = nn.Linear(in_features, out_features, bias=False)
        self.neigh_lin = nn.Linear(in_features, out_features, bias=False)

    def forward(self, H):
        N = PSpMMMax.apply(self.A, F.relu(self.pool(H)))
        return F.relu(self.self_lin(H) + self.neigh_lin(N))


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        epochs=50):
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PSAGE",
                 lambda plan: PSAGE(plan, nfeatures, nfeatures), nfeatures, False,
                 transport=transport, out=out, seed=seed, epochs=epochs)


USAGE = "usage: PSAGE.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> [--seed N]"


def main(argv):
    try:
        parsed = parse_args(argv, USAGE, valid=lambda size, nlayers, nfeatures, kw: min(size, nlayers, nfeatures) >= 1,
                            unknown_flag_text=USAGE)
    except ValueError:
        print(USAGE, flush=True)
        sys.exit(2)
    launch(run, *parsed)


if __name__ == "__main__":
    main(sys.argv[1:])
