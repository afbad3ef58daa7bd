"""The GPU test harness, shared by every GPU test file: device, stream and operand helpers, the test graphs, the ranks
of one process over the peer transport, CUDA-graph capture-and-replay checks, the command-line loss-curve run and the
multi-process spawner. A new feature's tests start from here.
"""
import os
import queue
import subprocess
import sys
import time
import traceback

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from helpers import GOLDEN, Golden
from pgcn_b200 import cabi, graphio, plan as planmod

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -24
# How long a spawned rank or a command-line run may take. pytest.ini ends a test at 420 s with os._exit, which would
# leave the workers running: the harness ends a stuck run first, with room for two runs in one test.
TIMEOUT = 180


def dev():
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: -m gpu tests must run on a GPU machine")
    return torch.device("cuda", 0)


def stream():
    return torch.cuda.current_stream().cuda_stream


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev())


def shifted(x):
    """A copy of x whose data starts 4 bytes into its buffer."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    return v


def bits(x):
    return x.detach().cpu().numpy().view(np.uint32) if x.dtype == torch.float32 else x.detach().cpu().numpy()


def identical(u, w):
    """Equal values and equal bits (so no NaN, and a zero keeps its sign)."""
    return torch.equal(u, w) and np.array_equal(bits(u), bits(w))


# ---- test graphs -----------------------------------------------------------------------------------------------------

def hub_graph():
    """R-MAT (6000 vertices) with a hub row of 3000 entries, rows of one entry (rows 20..29) and empty rows (10..19)."""
    A = sp.coo_matrix(graphio.synthetic_graph(6000, 120000, seed=31))
    keep = (A.row < 10) | (A.row >= 30)
    row = np.concatenate([A.row[keep], np.zeros(3000, np.int64), np.arange(20, 30)])
    col = np.concatenate([A.col[keep], np.arange(3000) * 2, np.arange(20, 30) + 100])
    B = sp.csr_matrix((np.ones(len(row), np.float32), (row, col)), shape=A.shape)
    B.sum_duplicates()
    return B.tocoo()


def karate():
    """The karate matrix of tests/golden/pgat_karate_k1.npz."""
    z = np.load(os.path.join(GOLDEN, "pgat_karate_k1.npz"))
    n = int(z["n"])
    return sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n))


def problem(case):
    """(A, partvec, k) of a golden case, "hub" (one rank), "karate" (pgat_karate_k3: three ranks) or a small R-MAT graph
    ("rmat": one rank, "rmat_k2": two)."""
    if case == "hub":
        A = hub_graph()
        return A, np.zeros(A.shape[0], dtype=np.int64), 1
    if case == "karate":
        z = np.load(os.path.join(GOLDEN, "pgat_karate_k3.npz"))
        n = int(z["n"])
        return sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n)), z["partvec"].astype(np.int64), 3
    if case.startswith("rmat"):
        n = 6000
        A = graphio.synthetic_graph(n, 120000, seed=31)
        k = 2 if case == "rmat_k2" else 1
        return A, (graphio.random_partvec(n, k, seed=5) if k > 1 else np.zeros(n, dtype=np.int64)), k
    g = Golden(case)
    return g.A, g.partvec, g.k


def edges(lp):
    """(rows, cols) of the local plan's stored entries."""
    return np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64))), lp.colidx.astype(np.int64)


def one_rank_plan(case, f):
    """(A, plan): problem(case) on one rank, values bound."""
    A, _, _ = problem(case)
    plan = planmod.build_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1, f, device=dev())
    plan.bind_values()
    return A, plan


# ---- several ranks in this process -----------------------------------------------------------------------------------

def linked_plans(lps, f, overlap, bind=True):
    """One plan per local plan, linked over the peer transport when there are several."""
    plans = [planmod.PgcnPlan(lp, f, device=dev()) for lp in lps]
    if len(plans) > 1:
        planmod.link_local_plans(plans)
    for p in plans:
        p.set_option("overlap", overlap)
        if bind:
            p.bind_values()
    return plans


def run_ranks(plans, fn, streams):
    """fn(r) for every rank on its own stream (the ranks' kernels wait for each other on the device), then sync."""
    torch.cuda.synchronize()
    out = [None] * len(plans)
    for r, s in enumerate(streams):
        with torch.cuda.stream(s):
            out[r] = fn(r)
    torch.cuda.synchronize()
    return out


# ---- CUDA-graph capture and replay -----------------------------------------------------------------------------------

REPLAYS = (0, 1, 2, 1)


def check_one_rank_capture(plan, step, load, eager, prepare=None, leaves=()):
    """Capture step() (named outputs of the static buffers) and replay it on the inputs REPLAYS after load(i); each
    replay must give the bits of eager(i). With `prepare` (widths), a capture before plan.prepare is refused first,
    the gradients of `leaves` are cleared, and the plan is prepared for those widths; without, it is prepared
    already."""
    if prepare is not None:
        with pytest.raises(RuntimeError, match="pgcn_plan_prepare"):
            with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=torch.cuda.Stream()):
                step()
        for u in leaves:
            u.grad = None
        for f in prepare:
            plan.prepare(f)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for i in REPLAYS:
        load(i)
        graph.replay()
        got = {name: u.detach().clone() for name, u in outs.items()}
        want = eager(i)
        for name, u in got.items():
            assert identical(u, want[name].detach()), "replay %d: %s differs from eager" % (i, name)


def check_two_rank_capture(plans, streams, buffers, load, step):
    """Capture step(r, bufs) on each rank's stream and replay it on the inputs REPLAYS: load(bufs, i) fills every
    rank's buffers (buffers(r) makes them, "x" the rank's m x f input) and step returns named outputs, which must have
    the bits of the same step run eagerly on fresh buffers. After the second step one more fused forward per rank
    makes the later replays meet the other exchange parity."""
    k = len(plans)
    cap = [buffers(r) for r in range(k)]
    graphs, outs = [], []
    for r in range(k):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=streams[r]):
            outs.append(step(r, cap[r]))
        graphs.append(graph)
    lib = cabi.load()
    for it, i in enumerate(REPLAYS):
        load(cap, i)
        run_ranks(plans, lambda r: graphs[r].replay(), streams)
        got = [{name: u.detach().clone() for name, u in outs[r].items()} for r in range(k)]
        eager = [buffers(r) for r in range(k)]
        load(eager, i)
        res = run_ranks(plans, lambda r: step(r, eager[r]), streams)
        for r in range(k):
            for name, u in got[r].items():
                assert identical(u, res[r][name].detach()), "step %d rank %d: %s replay differs from eager" % (
                    it, r, name)
        if it == 1:
            def forward(r):
                x = eager[r]["x"]
                cabi.check(lib.pgcn_forward(plans[r].handle, x.data_ptr(), torch.empty_like(x).data_ptr(), x.shape[1],
                                            stream()), plans[r].handle)
            run_ranks(plans, forward, streams)


# ---- command line ----------------------------------------------------------------------------------------------------

def run_cli(tmp_path, script, extra, port):
    """Train karate() on one rank with `script` (PGAT.py or PSAGE.py): 2 layers, f = 4, seed 7, plus `extra` flags.
    Returns the Epoch lines."""
    from scipy.io import mmwrite
    A = karate()
    n = A.shape[0]
    a = str(tmp_path / "karate.mtx")
    mmwrite(a, A)
    p = str(tmp_path / "karate.mtx.1.rp")
    graphio.write_partvec(p, np.zeros(n, dtype=np.int64))
    env = dict(os.environ, SLURM_NPROCS="1", SLURM_PROCID="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    out = subprocess.run([sys.executable, os.path.join(ROOT, script), "-a", a, "-p", p, "-b", "nccl", "-s", "1",
                          "-l", "2", "-f", "4", "--seed", "7"] + extra, env=env, capture_output=True, text=True,
                         timeout=TIMEOUT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert any(l.startswith("Elapsed time ") for l in out.stdout.splitlines())
    return [l for l in out.stdout.splitlines() if l.startswith("Epoch")]


def assert_follows(lines, want):
    """The Epoch lines print the fp64 curve `want` (the printed values carry 4 decimals)."""
    assert [l[:11] for l in lines] == ["Epoch %05d" % i for i in range(len(want))]
    np.testing.assert_allclose([float(l.split("Loss")[1]) for l in lines], want, rtol=1e-3, atol=6e-5)


# ---- one process per rank --------------------------------------------------------------------------------------------

def _rank_main(target, rank, k, args, q):
    try:
        q.put((rank, True, target(rank, k, *args)))
    except Exception:
        q.put((rank, False, traceback.format_exc()))


def spawn_ranks(target, k, args=(), timeout=TIMEOUT):
    """Run target(rank, k, *args) in k spawned processes and return {rank: its result}. A rank that raises, or that
    has not returned or exited within `timeout` seconds, fails the test. Every worker is dead and joined when this
    returns or raises, whatever the path."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(target, r, k, args, q), daemon=True) for r in range(k)]
    deadline = time.monotonic() + timeout
    out = {}
    try:
        for p in procs:
            p.start()
        while len(out) < k:
            try:
                rank, ok, payload = q.get(timeout=min(1.0, max(0.0, deadline - time.monotonic())))
            except queue.Empty:
                gone = [r for r, p in enumerate(procs) if r not in out and p.exitcode is not None]
                if gone:
                    try:                              # a result put just before the exit
                        rank, ok, payload = q.get(timeout=1.0)
                    except queue.Empty:
                        pytest.fail("rank %d exited with code %s and no result" % (gone[0], procs[gone[0]].exitcode))
                elif time.monotonic() >= deadline:
                    pytest.fail("ranks %s gave no result within %d s" % ([r for r in range(k) if r not in out],
                                                                         timeout))
                else:
                    continue
            if not ok:
                pytest.fail("rank %d failed:\n%s" % (rank, payload))
            out[rank] = payload
        for p in procs:
            p.join(max(0.0, deadline - time.monotonic()))
        late = [r for r, p in enumerate(procs) if p.is_alive()]
        if late:
            pytest.fail("ranks %s did not exit within %d s" % (late, timeout))
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
        for p in procs:
            if p.pid is not None:
                p.join()
        q.close()
    return out
