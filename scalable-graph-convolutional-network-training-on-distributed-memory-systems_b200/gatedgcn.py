"""PGATEDGCN trainer CLI — GatedGCN layers with an edge-feature stream over the H100 operator.

    python PGATEDGCN.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 16 [--seed 0] [--transport auto|p2p|nccl]

The network is GatedGCN (Bresson & Laurent, in the form of Dwivedi et al.'s benchmarking-gnns) without BatchNorm. The
edge input is each stored entry's fp32 value of A (the plan's lp.vals, in the order of PgcnPlan.edge_pairs()) as
[nnz, 1], which an edge encoder Linear(1, f) maps to width f. Each layer then updates the node features h and the edge
features e:

    Ax, Bx, Dx, Ex = A(h), B(h), D(h), E(h)          Linear(f, f) with bias each
    Ce = C(e)                                        Linear(f, f) with bias
    Z, ehat = PGatedGCN(plan, Dx, Ex, Bx, Ce)        ehat = Dx[i] + Ex[j] + Ce,  Z[i] = sum s Bx[j] / (sum s + 1e-6)
    h = h + relu(Ax + Z),  e = e + relu(ehat)

and the logits are the last h. Parameters are drawn with torch's default initialisation in this order: the edge
encoder, then per layer A, B, D, E, C. Everything else is PGATED.py's surface: flags -a -p -b -s -l -f; rank/size from
SLURM_PROCID / SLURM_NPROCS with torchrun's RANK / WORLD_SIZE as a fallback; inputs H[i, :] = i and labels i % f;
parameters built on the CPU under --seed, then moved to the device and averaged over ranks; Adam lr 1e-3; 50 epochs;
gradients all-reduced / world_size; stdout `Epoch {:05d} | Loss {:.4f}` (each rank's loss is sum_owned nll / n, the
printed loss their all-reduced sum) and `Elapsed time {:.4f}`. [Ex | Bx] is exchanged in every layer, so the plan is
built with f_max = 2f; the edge features stay on the rank that owns their row. `-b gloo` is refused: the H100 path has
no CPU fallback.
"""
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from .op import GATEDGCN_EPS, PGatedGCN
from .pgcn import launch, parse_args, train


class GatedGCNLayer(nn.Module):
    """One GatedGCN layer (residual, ReLU, no BatchNorm) on the plan handle A (a bound PgcnPlan with f_max >= 2f):
    forward(h, e) -> (h, e), h [rows, f] in the plan's layout, e [nnz_local, f] in edge_pairs() order."""

    def __init__(self, A, features, eps=GATEDGCN_EPS):
        super().__init__()
        self.A = A
        self.eps = eps
        self.lin_A = nn.Linear(features, features)
        self.lin_B = nn.Linear(features, features)
        self.lin_D = nn.Linear(features, features)
        self.lin_E = nn.Linear(features, features)
        self.lin_C = nn.Linear(features, features)

    def forward(self, h, e):
        Z, ehat = PGatedGCN.apply(self.A, self.lin_D(h), self.lin_E(h), self.lin_B(h), self.lin_C(e), self.eps)
        return h + F.relu(self.lin_A(h) + Z), e + F.relu(ehat)


class PGATEDGCN(nn.Module):
    """The edge encoder and `nlayers` GatedGCN layers of width f on the plan handle A; forward(H) gives the logits."""

    def __init__(self, A, features, nlayers, eps=GATEDGCN_EPS):
        super().__init__()
        self.A = A
        self.edge_encoder = nn.Linear(1, features)
        self.layers = nn.ModuleList([GatedGCNLayer(A, features, eps) for _ in range(nlayers)])
        self.register_buffer("edge_input", torch.from_numpy(A.lp.vals.astype("float32")).reshape(-1, 1),
                             persistent=False)

    def forward(self, H):
        h, e = H, self.edge_encoder(self.edge_input)
        for layer in self.layers:
            h, e = layer(h, e)
        return h


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, transport="auto", out=sys.stdout, seed=None,
        epochs=50):
    return train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, "PGATEDGCN", None, 2 * nfeatures,
                 False, transport=transport, out=out, seed=seed, epochs=epochs,
                 model=lambda plan: PGATEDGCN(plan, nfeatures, nlayers))


USAGE = "usage: PGATEDGCN.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> [--seed N]"


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
