"""PGCN trainer CLI — the reference's surface (GPU/PGCN.py:136-286) over the H100 operator.

    python PGCN.py -a A.mtx -p A.mtx.8.hp -b nccl -s 8 -l 2 -f 128

Kept from the reference: flags -a -p -b -s -l -f (GPU/PGCN.py:262-278); rank/size from
SLURM_PROCID / SLURM_NPROCS (:258-260) with torchrun's RANK / WORLD_SIZE as a fallback; rendezvous
from MASTER_ADDR / MASTER_PORT; device cuda:{rank % ndev} (:169); inputs H[i, :] = i (:186-188) and
labels i % f (:192); L x (PSpMM -> Linear(f, f, bias=False) -> ReLU) (:136-148, :194-196); parameter
averaging at start (:156-160); Adam lr 1e-3 (:200); 1 warm-up + 4 timed epochs (:202-226); gradient
all-reduce / world_size (:150-154); stdout fields `Epoch {:05d} | Loss {:.4f}`, the per-rank stats
dict, `Elapsed time {:.4f}`, `total_vol: .. total_nmsg: ..` (:224-238).

Different by design (SURVEY.md §8a/§8b): every tensor is [m_local, f] instead of [n, f]; the loss is
the reference's value computed from owned rows only, loss = (sum_owned nll + (n - m) * log f) / n,
which has exactly the reference's gradients (its non-owned rows are all-zero logits); the elapsed
time is bracketed by torch.cuda.synchronize(); `-b gloo` is refused — the H100 path has no CPU
fallback (the CPU oracle lives under oracle/ and is test infrastructure).
`--ref-quirks` reproduces quirk Q1 (halo rows counted twice in layer 1 because `run` feeds a fully
populated H into `H + X`, GPU/PGCN.py:117,186) so loss curves can be compared with seeded weights.
"""
import getopt
import math
import os
import sys
import time

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from . import plan as planmod
from .op import PSpMM, PSpMMRelu, communicate_fgm, spmm_local, aggregate_backward


class _PSpMMQuirkQ1(torch.autograd.Function):
    """Layer-1 aggregation as the reference computes it when fed an unmasked H: A_loc (H + 1_halo H),
    i.e. halo rows weigh twice (quirk Q1). Backward is the regular one."""

    @staticmethod
    def forward(ctx, A, H):
        ctx.plan = A
        halo = communicate_fgm(A, H, backward=False)
        return spmm_local(A, H, 2.0 * halo if A.lp.h else None)

    @staticmethod
    def backward(ctx, g):
        return None, aggregate_backward(ctx.plan, g)


class PGCN(nn.Module):
    """GPU/PGCN.py:136-148 with the plan handle in place of the sparse tensor."""

    def __init__(self, A, in_features, out_features, quirk_q1=False, fused=False):
        super().__init__()
        self.linear = nn.Linear(in_features, out_features, bias=False)
        self.A = A
        self.quirk_q1 = quirk_q1
        self.fused = fused and not quirk_q1

    def forward(self, H):
        if self.fused:
            # relu(A (H W^T)): dense step on the m owned rows first, relu fused into the aggregation's store
            return PSpMMRelu.apply(self.A, self.linear(H))
        H = _PSpMMQuirkQ1.apply(self.A, H) if self.quirk_q1 else PSpMM.apply(self.A, H)
        H = self.linear(H)
        return F.relu(H)


def average_gradients(model, world_size):
    for param in model.parameters():                      # GPU/PGCN.py:150-154
        dist.all_reduce(param.grad.data, op=dist.ReduceOp.SUM)
        param.grad.data /= world_size


def initialize_parameters(model, world_size):
    for param in model.parameters():                      # GPU/PGCN.py:156-160
        dist.all_reduce(param.data, op=dist.ReduceOp.SUM)
        param.data /= world_size


def _cuda_device(rank, backend, name):
    if backend != "nccl":
        raise RuntimeError("backend '%s': the H100 %s path runs on CUDA devices over NCCL/NVLink only "
                           "(no CPU fallback); use -b nccl" % (backend, name))
    device = torch.device("cuda", rank % torch.cuda.device_count())      # GPU/PGCN.py:169
    torch.cuda.set_device(device)
    return device


def train(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, name, layer, f_max, grad_H,
          transport="auto", out=sys.stdout, seed=None, epochs=50, model=None):
    """The training loop of PGAT.py and PSAGE.py (`name`): a bound plan of width f_max, inputs H[i, :] = i (requiring
    grad when grad_H) and labels i % f, nlayers layers `layer(plan)` (f -> f) built under `seed` and averaged over
    ranks, Adam lr 1e-3, `epochs` epochs of the loss sum_owned nll / n with gradients averaged over ranks. Rank 0 prints
    `Epoch {:05d} | Loss {:.4f}` (the all-reduced loss) per epoch and `Elapsed time {:.4f}`. Returns the losses, the
    elapsed time, the transport and plan.stats. model: a factory model(plan) of the whole network (H -> logits), built
    under `seed` in place of the stack of `layer`s, for a network that is not a plain sequence of layers (PGATEDGCN.py:
    an edge-feature stream beside the node features)."""
    device = _cuda_device(rank, backend, name)
    lp_host = planmod.read_local_plan(path_A, path_partvec, rank, size)
    n = lp_host.n
    plan = planmod.PgcnPlan(lp_host, f_max, device=device)
    used = plan.init_comm(transport=transport)
    plan.bind_values()
    lp = plan.lp

    own = torch.from_numpy(lp.owned).to(device)
    H = own.to(torch.float32).unsqueeze(1).repeat(1, nfeatures).contiguous().requires_grad_(grad_H)
    labels = own % nfeatures

    if seed is not None:
        torch.manual_seed(seed)
    factory = model
    model = (factory(plan) if factory is not None else nn.Sequential(*[layer(plan) for _ in range(nlayers)])).to(device)
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


def reference_loss(logits_own, labels_own, n):
    """F.nll_loss(log_softmax(logits), labels) over ALL n rows as the reference computes it
    (GPU/PGCN.py:204-205), from the owned rows: non-owned rows are all-zero logits -> nll = log f."""
    m, f = logits_own.shape
    nll = F.nll_loss(F.log_softmax(logits_own, 1), labels_own, reduction="sum") if m else logits_own.sum()
    return (nll + (n - m) * math.log(f)) / n


def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, ref_quirks=False, transport="auto",
        out=sys.stdout, seed=None, fused=False):
    device = _cuda_device(rank, backend, "PGCN")
    cache = os.environ.get("PGCN_PLAN_CACHE")
    if cache:                                                            # optional on-disk plan cache (§8f rank 2)
        lp_host = planmod.cached_local_plan(path_A, path_partvec, rank, size, cache)
    else:
        lp_host = planmod.read_local_plan(path_A, path_partvec, rank, size)
    n = lp_host.n
    plan = planmod.PgcnPlan(lp_host, nfeatures, device=device)           # :178-182
    if ref_quirks:
        transport = "nccl"            # the quirk emulation drives the exchange step by step (NCCL entry points)
    used = plan.init_comm(transport=transport)
    plan.autotune(nfeatures)
    lp = plan.lp

    own = torch.from_numpy(lp.owned).to(device)
    H = own.to(torch.float32).unsqueeze(1).repeat(1, nfeatures).contiguous().requires_grad_(True)   # :186-188
    labels = own % nfeatures                                                                          # :192

    if seed is not None:
        torch.manual_seed(seed)
    model = nn.Sequential(*[PGCN(plan, nfeatures, nfeatures, quirk_q1=(ref_quirks and i == 0), fused=fused)
                            for i in range(nlayers)]).to(device)        # :194-198
    if size > 1:
        initialize_parameters(model, size)
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)            # :200

    def epoch():
        logits = model(H)
        loss = reference_loss(logits, labels, n)
        optimizer.zero_grad()
        loss.backward()
        if size > 1:
            average_gradients(model, size)
        optimizer.step()
        return loss

    epoch()                                                              # warm-up epoch, :202-209
    torch.cuda.synchronize()
    start = time.time()
    losses = []
    for ep in range(4):                                                  # :212-224
        loss = epoch()
        losses.append(float(loss))
        if rank == 0:
            print("Epoch {:05d} | Loss {:.4f}".format(ep, losses[-1]), file=out, flush=True)
    torch.cuda.synchronize()
    elapsed = torch.tensor([time.time() - start], device=device)
    if size > 1:
        dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)                   # :228

    print(plan.stats, file=out, flush=True)                              # :230
    tot = torch.tensor([plan.stats["send_volume"], plan.stats["send_nmsg"]], device=device)
    if size > 1:
        dist.all_reduce(tot, op=dist.ReduceOp.SUM)                       # :233-234
    if rank == 0:
        print("Elapsed time {:.4f}".format(elapsed.item()), file=out, flush=True)
        print("total_vol: {} total_nmsg: {}".format(int(tot[0]), int(tot[1])), file=out, flush=True)
    result = {"losses": losses, "total_vol": int(tot[0]), "total_nmsg": int(tot[1]), "elapsed": float(elapsed.item()),
              "transport": used}
    plan.close()
    return result


def init_process(rank, size, fn, nlayers, nfeatures, path_A, path_partvec, backend, **kw):
    if backend == "nccl" and torch.cuda.is_available():
        torch.cuda.set_device(rank % torch.cuda.device_count())
    dist.init_process_group(backend, rank=rank, world_size=size)         # GPU/PGCN.py:242
    env = {k: os.environ.get(k) for k in ("MASTER_ADDR", "MASTER_PORT", "RANK", "WORLD_SIZE")}
    print("[{}] Initializing process group with: {}".format(os.getpid(), env), flush=True)
    try:
        return fn(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, **kw)
    finally:
        dist.destroy_process_group()


def parse_args(argv, usage, options=None, valid=None, unknown_flag_text="a:p:b:"):
    """The command line of every trainer: rank and size from SLURM_PROCID / SLURM_NPROCS (GPU/PGCN.py:258-260) with
    torchrun's RANK / WORLD_SIZE as a fallback, the flags -a -p -b -s -l -f (:262-278), --transport, --seed and the
    trainer's own `options`, {"--name": (keyword, type)} with type None for a switch. Returns (rank, size, args, kw):
    the positional arguments of `run` after rank and size, and its keywords. An unknown flag prints `unknown_flag_text`
    (by default the reference's, :264); a missing flag, or options that valid(size, nlayers, nfeatures, kw) refuses,
    print `usage`; both exit with status 2. A malformed number raises ValueError."""
    size = int(os.environ.get("SLURM_NPROCS", os.environ.get("WORLD_SIZE", "1")))
    rank = int(os.environ.get("SLURM_PROCID", os.environ.get("RANK", "0")))
    os.environ["RANK"] = str(rank)
    options = dict(options or {}, **{"--transport": ("transport", str), "--seed": ("seed", int)})
    try:
        opts, _ = getopt.getopt(argv, "a:p:b:s:l:f:", [o[2:] + ("=" if t else "") for o, (_, t) in options.items()])
    except getopt.GetoptError:
        print(unknown_flag_text, flush=True)
        sys.exit(2)
    path_A = path_partvec = None
    backend = "nccl"
    nlayers = nfeatures = None
    kw = {}
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
        else:
            key, typ = options[opt]
            kw[key] = typ(arg) if typ else True
    if (path_A is None or path_partvec is None or nlayers is None or nfeatures is None
            or (valid is not None and not valid(size, nlayers, nfeatures, kw))):
        print(usage, flush=True)
        sys.exit(2)
    return rank, size, (nlayers, nfeatures, path_A, path_partvec, backend), kw


def launch(fn, rank, size, args, kw):
    """fn(rank, size, *args, **kw) in the process group, with the rendezvous at MASTER_ADDR / MASTER_PORT (default
    127.0.0.1:29500)."""
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    os.environ["WORLD_SIZE"] = str(size)
    init_process(rank, size, fn, *args, **kw)


USAGE = "usage: PGCN.py -a <A.mtx> -p <partvec> -b nccl -s <nparts> -l <nlayers> -f <nfeatures>"


def main(argv):
    # --fused: relu(A (H W^T)) with the clamp fused into the aggregation (SURVEY §8f rank 1)
    launch(run, *parse_args(argv, USAGE, {"--ref-quirks": ("ref_quirks", None), "--fused": ("fused", None)}))


if __name__ == "__main__":
    main(sys.argv[1:])
