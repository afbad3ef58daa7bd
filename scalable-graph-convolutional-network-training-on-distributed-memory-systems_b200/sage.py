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
import getopt
import os
import sys
import time

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from . import graphio, plan as planmod
from .op import PSpMMMax
from .pgcn import average_gradients, initialize_parameters, init_process


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
    if backend != "nccl":
        raise RuntimeError("backend '%s': the H100 PSAGE path runs on CUDA devices over NCCL/NVLink only "
                           "(no CPU fallback); use -b nccl" % backend)
    device = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(device)
    A = graphio.read_adjacency(path_A)
    partvec = graphio.read_partvec(path_partvec, A.shape[0])
    graphio.check_partvec(partvec, size)
    lp_host = planmod.build_local_plan(A, partvec, rank, size)
    n = lp_host.n
    plan = planmod.PgcnPlan(lp_host, nfeatures, device=device)
    used = plan.init_comm(transport=transport)
    plan.bind_values()
    lp = plan.lp

    own = torch.from_numpy(lp.owned).to(device)
    H = own.to(torch.float32).unsqueeze(1).repeat(1, nfeatures).contiguous()
    labels = own % nfeatures

    if seed is not None:
        torch.manual_seed(seed)
    model = nn.Sequential(*[PSAGE(plan, nfeatures, nfeatures) for _ in range(nlayers)]).to(device)
    if size > 1:
        initialize_parameters(model, size)
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)

    torch.cuda.synchronize()
    start = time.time()
    losses = []
    for ep in range(epochs):
        logits = model(H)
        loss = F.nll_loss(F.log_softmax(logits, 1), labels, reduction="sum") / n
        optimizer.zero_grad()
        loss.backward()
        if size > 1:
            average_gradients(model, size)
        optimizer.step()
        total = loss.detach().clone()
        if size > 1:
            dist.all_reduce(total, op=dist.ReduceOp.SUM)
        losses.append(float(total))
        if rank == 0:
            print("Epoch {:05d} | Loss {:.4f}".format(ep, losses[-1]), file=out, flush=True)
    torch.cuda.synchronize()
    elapsed = torch.tensor([time.time() - start], device=device)
    if size > 1:
        dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)
    if rank == 0:
        print("Elapsed time {:.4f}".format(elapsed.item()), file=out, flush=True)
    result = {"losses": losses, "elapsed": float(elapsed.item()), "transport": used, "stats": dict(plan.stats)}
    plan.close()
    return result


USAGE = "usage: PSAGE.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> [--seed N]"


def main(argv):
    size = int(os.environ.get("SLURM_NPROCS", os.environ.get("WORLD_SIZE", "1")))
    rank = int(os.environ.get("SLURM_PROCID", os.environ.get("RANK", "0")))
    os.environ["RANK"] = str(rank)
    try:
        opts, _ = getopt.getopt(argv, "a:p:b:s:l:f:", ["transport=", "seed="])
    except getopt.GetoptError:
        print(USAGE, flush=True)
        sys.exit(2)
    path_A = path_partvec = None
    backend = "nccl"
    nlayers = nfeatures = None
    kw = {}
    try:
        for opt, arg in opts:
            if opt == "-a":
                path_A = arg
            elif opt == "-p":
                path_partvec = arg
            elif opt == "-b":
                backend = arg
            elif opt == "-s":
                size = int(arg)
            elif opt == "-l":
                nlayers = int(arg)
            elif opt == "-f":
                nfeatures = int(arg)
            elif opt == "--transport":
                kw["transport"] = arg
            elif opt == "--seed":
                kw["seed"] = int(arg)
    except ValueError:
        print(USAGE, flush=True)
        sys.exit(2)
    if (path_A is None or path_partvec is None or nlayers is None or nfeatures is None or nlayers < 1 or nfeatures < 1
            or size < 1):
        print(USAGE, flush=True)
        sys.exit(2)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    os.environ["WORLD_SIZE"] = str(size)
    init_process(rank, size, run, nlayers, nfeatures, path_A, path_partvec, backend, **kw)


if __name__ == "__main__":
    main(sys.argv[1:])
