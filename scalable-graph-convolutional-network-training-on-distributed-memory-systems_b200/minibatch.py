"""Host side of the mini-batch variant (GPU/PGCN-Mini-batch.py) — SURVEY.md §8f rank 3, loader part only.

The reference pre-samples `nbatches = (n // batch_size + 1) * 3` vertex sets with `random.sample` (seed 1,
GPU/PGCN-Mini-batch.py:201-203,220-230), keeps for each the induced sub-matrix (entries whose row AND column are
in the batch, :58-69), and recomputes the per-peer maps and the rank's rows per batch with the same per-nnz
Python loop as the full-batch trainer (:40-56, :71-82). The same operator then runs on the per-batch matrix.

Here each batch becomes an ordinary LocalPlan (plan.build_local_plan on the induced sub-matrix, global shape and
the global part vector kept), so PSpMM / PgcnPlan run unchanged on it; every batch plan shares the rank's [m, f]
row layout (rows outside the batch are simply empty).

The training driver (`run` / `main`, same flags as the reference plus `-n batch_size`, GPU/PGCN-Mini-batch.py:199-342):
one device plan per pre-sampled batch, all of them sharing ONE NCCL communicator (`pgcn_comm_share`), swapped per
step exactly where the reference swaps `[bA, send_map, recv_map]` (:256-259); 3 GCN layers like the reference's
`SequentialGCN` (:176-187; `-l` is parsed and ignored there, honoured here with default 3); one warm-up epoch, four
timed epochs, the loss summed over batches starting from 1 (:277), the reference's output lines.
"""
import pickle
import random

import numpy as np
import scipy.sparse as sp

from . import plan as planmod


def read_partvec_pickle(path):
    """The mini-batch trainer reads a PICKLED list of part ids (GPU/PGCN-Mini-batch.py:216-217), written by
    GPU/SHP/main.py."""
    with open(path, "rb") as f:
        return np.asarray(pickle.load(f), dtype=np.int64)


def sample_adjacency_matrix(A, indices):
    """GPU/PGCN-Mini-batch.py:58-69, vectorised: entries with row in `indices` and column in `indices`;
    shape and entry order of A preserved."""
    A = A.tocoo()
    mask = np.zeros(A.shape[0], dtype=bool)
    mask[np.asarray(indices, dtype=np.int64)] = True
    keep = mask[A.row] & mask[A.col]
    return sp.coo_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)


def batch_index_sets(n, batch_size, seed=1):
    """The reference's sampling sequence: random.seed(seed); (n // batch_size + 1) * 3 draws of
    random.sample(range(n), batch_size) (GPU/PGCN-Mini-batch.py:201-203,220-225)."""
    rnd = random.Random(seed)
    nbatches = (n // batch_size + 1) * 3
    return [np.array(rnd.sample(range(n), batch_size), dtype=np.int64) for _ in range(nbatches)]


def batch_local_plans(A, partvec, rank, size, batch_size, seed=1, index_sets=None):
    """One LocalPlan per pre-sampled batch for this rank (the reference's `batches` list,
    GPU/PGCN-Mini-batch.py:220-230: [bA, batch_send_map, batch_recv_map])."""
    sets = batch_index_sets(A.shape[0], batch_size, seed) if index_sets is None else index_sets
    return [planmod.build_local_plan(sample_adjacency_matrix(A, idx), partvec, rank, size) for idx in sets], sets


# ---- training driver ---------------------------------------------------------------------------------------------

def run(rank, size, nlayers, nfeatures, path_A, path_partvec, backend, batch_size, out=None, seed=None,
        cuda_graph=False):
    """GPU/PGCN-Mini-batch.py:199-310 on the H100 path. Returns {"losses", "elapsed", "total_vol", "total_nmsg"}.

    cuda_graph=True: after the (eager) warm-up epoch, the forward and backward of every batch plan are captured once
    in a CUDA graph (all graphs share one memory pool) and replayed in the eager step order; the gradient average and
    the optimizer step stay eager, so the losses are the eager ones. A step of a small batch is launch-bound: the
    replay saves the per-kernel launch and the Python autograd overhead."""
    import sys
    import time
    import torch
    import torch.distributed as dist
    import torch.nn as nn
    from . import graphio
    from .op import PSpMM
    from .pgcn import reference_loss, average_gradients, initialize_parameters
    import torch.nn.functional as F
    out = sys.stdout if out is None else out
    if backend != "nccl":
        raise RuntimeError("backend '%s': the H100 PGCN path runs on CUDA devices over NCCL/NVLink only "
                           "(no CPU fallback); use -b nccl" % backend)
    device = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(device)
    A = graphio.read_adjacency(path_A)                                         # :213
    partvec = read_partvec_pickle(path_partvec) if not path_partvec.endswith((".hp", ".gp", ".rp", ".txt")) \
        else graphio.read_partvec(path_partvec, A.shape[0])                    # :216-217 (pickled list)
    graphio.check_partvec(partvec, size)
    n = A.shape[0]
    lps, _ = batch_local_plans(A, partvec, rank, size, batch_size, seed=1)     # :220-230, random.seed(1)
    plans = [planmod.PgcnPlan(lp, nfeatures, device=device) for lp in lps]
    if size > 1:
        plans[0].init_comm(transport="nccl")                                   # one communicator ...
        for p in plans[1:]:
            p.share_comm(plans[0])                                             # ... borrowed by every other batch plan
    lp0 = lps[0]
    own = torch.from_numpy(lp0.owned).to(device)
    H = own.to(torch.float32).unsqueeze(1).repeat(1, nfeatures).contiguous().requires_grad_(True)   # :234-236
    labels = own % nfeatures                                                                          # :239
    if seed is not None:
        torch.manual_seed(seed)

    class Layer(nn.Module):                                                    # :163-174, plan passed per call
        def __init__(self):
            super().__init__()
            self.linear = nn.Linear(nfeatures, nfeatures, bias=False)

        def forward(self, plan, X):
            return F.relu(self.linear(PSpMM.apply(plan, X)))

    layers = nn.ModuleList([Layer() for _ in range(nlayers)]).to(device)
    if size > 1:
        initialize_parameters(layers, size)
    optimizer = torch.optim.Adam(layers.parameters(), lr=1e-3)                 # :249

    def forward_loss(plan):
        X = H
        for layer in layers:
            X = layer(plan, X)
        return reference_loss(X, labels, n)                         # nll over all n rows (:262-263)

    def update():
        if size > 1:
            average_gradients(layers, size)
        optimizer.step()

    def step(plan):
        loss = forward_loss(plan)
        optimizer.zero_grad()
        loss.backward()
        update()
        return loss.detach()

    if cuda_graph:
        for plan in plans:
            plan.prepare(nfeatures)
    for plan in plans:                                                         # warm-up epoch (:251-268)
        step(plan)
    if cuda_graph:
        step = _graphed_steps(plans, forward_loss, update, optimizer, layers)
    torch.cuda.synchronize()
    start = time.time()
    losses = []
    for epoch in range(4):                                                     # :271-291
        loss_epoch = torch.ones((), device=device)
        for plan in plans:
            loss_epoch = loss_epoch + step(plan)
        if size > 1:
            dist.all_reduce(loss_epoch, op=dist.ReduceOp.SUM)
        losses.append(float(loss_epoch))
        if rank == 0:
            print("Epoch {:05d} | Loss {:.4f}".format(epoch, losses[-1]), file=out, flush=True)
    torch.cuda.synchronize()
    elapsed = torch.tensor([time.time() - start], device=device)
    vol = torch.tensor([sum(p.stats["send_volume"] for p in plans), sum(p.stats["send_nmsg"] for p in plans)],
                       device=device, dtype=torch.int64)
    if size > 1:
        dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)
        dist.all_reduce(vol, op=dist.ReduceOp.SUM)
    if rank == 0:
        print("Elapsed time {:.4f}".format(float(elapsed)), file=out, flush=True)
        print("total_vol: %d total_nmsg: %d" % (int(vol[0]), int(vol[1])), file=out, flush=True)
    res = {"losses": losses, "elapsed": float(elapsed), "total_vol": int(vol[0]), "total_nmsg": int(vol[1]),
           "nbatches": len(plans)}
    for p in plans[1:] + plans[:1]:
        p.close()
    return res


def _graphed_steps(plans, forward_loss, update, optimizer, layers):
    """Capture forward + backward of every batch plan in a CUDA graph of its own, all graphs in one memory pool.
    Returns step(plan): replay that plan's graph, add the exchange stats its capture recorded, run `update` (gradient
    average and optimizer step) eagerly, and return the graph's loss tensor (read it before the next replay: the next
    graph may reuse its memory)."""
    import torch
    params = list(layers.parameters())
    grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in params]
    for p, g in zip(params, grads):
        p.grad = g                       # static gradient buffers: backward inside the graph accumulates into them
    pool = torch.cuda.graph_pool_handle()
    graphs = {}
    for plan in plans:
        before = dict(plan.stats)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=pool):
            optimizer.zero_grad(set_to_none=False)
            loss = forward_loss(plan)
            loss.backward()
        # the capture ran no kernel: its exchange counts belong to every replay instead
        delta = {k: plan.stats[k] - before[k] for k in before}
        plan.stats.update(before)
        if any(p.grad is None or p.grad.data_ptr() != g_.data_ptr() for p, g_ in zip(params, grads)):
            raise RuntimeError("backward inside the CUDA graph replaced a gradient buffer instead of accumulating")
        graphs[id(plan)] = (g, loss.detach(), delta)

    def step(plan):
        g, loss, delta = graphs[id(plan)]
        g.replay()
        for k, v in delta.items():
            plan.stats[k] += v
        update()
        return loss
    return step


def main(argv):
    """python -m pgcn_b200.minibatch -a A.mtx -p partvec.pkl -b nccl -s k -l 3 -f F -n batch_size [--cuda-graph]
    (SLURM_NPROCS / SLURM_PROCID or WORLD_SIZE / RANK, MASTER_ADDR / MASTER_PORT as the reference)."""
    import getopt
    import os
    import sys
    import torch.distributed as dist
    size = int(os.environ.get("SLURM_NPROCS", os.environ.get("WORLD_SIZE", "1")))
    rank = int(os.environ.get("SLURM_PROCID", os.environ.get("RANK", "0")))
    try:
        opts, _ = getopt.getopt(argv, "a:p:b:s:l:f:n:", ["seed=", "cuda-graph"])
    except getopt.GetoptError:
        print("a:p:b:", flush=True)
        sys.exit(2)
    kw = dict(path_A=None, path_partvec=None, backend="nccl", nlayers=3, nfeatures=None, batch_size=None, seed=None,
              cuda_graph=False)
    for opt, arg in opts:
        if opt == "-a": kw["path_A"] = arg
        elif opt == "-p": kw["path_partvec"] = arg
        elif opt == "-b": kw["backend"] = arg
        elif opt == "-s": size = int(arg)
        elif opt == "-l": kw["nlayers"] = int(arg)
        elif opt == "-f": kw["nfeatures"] = int(arg)
        elif opt == "-n": kw["batch_size"] = int(arg)
        elif opt == "--seed": kw["seed"] = int(arg)
        elif opt == "--cuda-graph": kw["cuda_graph"] = True
    if None in (kw["path_A"], kw["path_partvec"], kw["nfeatures"], kw["batch_size"]):
        print("usage: minibatch -a <A.mtx> -p <partvec.pkl> -b nccl -s <nparts> -l <nlayers> -f <nfeatures> -n <batch_size>", flush=True)
        sys.exit(2)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    os.environ["RANK"] = str(rank); os.environ["WORLD_SIZE"] = str(size)
    import torch
    dist.init_process_group("nccl", rank=rank, world_size=size,
                            device_id=torch.device("cuda", rank % max(torch.cuda.device_count(), 1)))
    try:
        return run(rank, size, kw["nlayers"], kw["nfeatures"], kw["path_A"], kw["path_partvec"], kw["backend"],
                   kw["batch_size"], seed=kw["seed"], cuda_graph=kw["cuda_graph"])
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    import sys
    main(sys.argv[1:])
