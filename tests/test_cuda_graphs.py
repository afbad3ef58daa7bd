"""The fused forward / backward captured in CUDA graphs (PgcnPlan.prepare, then torch.cuda.graph or raw stream
capture) and replayed on new inputs: every replay equals an eager call on the same input bit for bit.

  * one rank: PSpMM forward + backward and PSpMMRelu, register kernel (f = 16, 100) and ring kernel (f = 128, 256:
    64-float slices, full width, autotuned), "local" and "global" layouts;
  * a capture that would need set-up work is refused with an error naming prepare, and leaves plan and stream usable;
    a refused call has enqueued no kernel (a matrix with empty rows, whose zero-fill comes after all set-up);
  * several ranks on this GPU over the peer transport (plan.link_local_plans), eager calls and replays mixed so that the
    device-resident exchange epoch takes both parities in both directions;
  * schedules replaced after the capture are retired, not freed, and the replay still computes the old options;
  * the mini-batch trainer with cuda_graph=True against the eager trainer and the reference's loss curve;
  * on >= 2 GPUs: capture and replay over NCCL and over CUDA IPC peer memory, one process per GPU.
"""
import io
import json
import os
import pickle

import numpy as np
import pytest
import torch

from harness import dev, run_ranks, spawn_ranks
from helpers import GOLDEN, Golden, assert_close_fp32, fp32_tol
from oracle import pgcn_oracle as orc
from pgcn_b200 import cabi, graphio, plan as planmod
from pgcn_b200.op import PSpMM, PSpMMRelu

pytestmark = pytest.mark.gpu


def rand(rs, rows, f):
    return torch.from_numpy(rs.uniform(-1, 1, size=(rows, f)).astype(np.float32)).to(dev())


def eager_fwd_bwd(fn, plan, x, g):
    x = x.clone().requires_grad_(True)
    z = fn.apply(plan, x)
    z.backward(g)
    return z.detach(), x.grad


def check_capture_replays(plan, rows, f, seed):
    """Capture PSpMM and PSpMMRelu, each forward + backward, in one graph; replay it on three inputs."""
    rs = np.random.RandomState(seed)
    xs = [rand(rs, rows, f) for _ in range(3)]
    gs = [rand(rs, rows, f) for _ in range(3)]
    x = torch.zeros((rows, f), device=dev(), requires_grad=True)
    xr = torch.zeros((rows, f), device=dev(), requires_grad=True)
    g_in = torch.zeros((rows, f), device=dev())
    relu = plan.layout == "local"                  # PSpMMRelu takes the compact layout only
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z = PSpMM.apply(plan, x)
        z.backward(g_in)
        if relu:
            zr = PSpMMRelu.apply(plan, xr)
            zr.backward(g_in)
    for i in range(3):
        with torch.no_grad():
            x.copy_(xs[i]); xr.copy_(xs[i]); g_in.copy_(gs[i])
        graph.replay()
        ze, ge = eager_fwd_bwd(PSpMM, plan, xs[i], gs[i])
        assert torch.equal(z, ze) and torch.equal(x.grad, ge), "PSpMM replay %d differs from eager" % i
        if relu:
            zre, gre = eager_fwd_bwd(PSpMMRelu, plan, xs[i], gs[i])
            assert torch.equal(zr, zre) and torch.equal(xr.grad, gre), "PSpMMRelu replay %d differs from eager" % i
    torch.cuda.synchronize()
    return xs[-1], z.detach().clone()


def one_rank_matrix(case):
    if case == "rmat":
        return graphio.synthetic_graph(8000, 160000, seed=21)
    return Golden(case).A


@pytest.mark.parametrize("case", ["gemat11_k1", "rmat"])
@pytest.mark.parametrize("f", [16, 100, 128, 256])
def test_one_rank_capture_equals_eager(case, f):
    A = one_rank_matrix(case)
    n = A.shape[0]
    settings = ["default"] if f % 128 else ["slices", "full", "autotune"]
    for layout in ("local", "global"):
        for s in settings:
            plan = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
            plan.layout = layout
            if s == "slices":
                plan.set_option("ring_tile_floats", 64)
            elif s == "full":
                plan.set_option("ring_tile_floats", f)
            elif s == "autotune":
                plan.autotune(f)
            plan.prepare(f)
            x, z = check_capture_replays(plan, n, f, seed=f)
            Z64 = orc.truth_forward(A, x.cpu().numpy())
            assert_close_fp32(z.cpu().numpy(), Z64, fp32_tol(A, x.cpu().numpy(), int(orc.row_degree(A).max())),
                              "%s f=%d %s %s" % (case, f, layout, s))
            plan.close()


@pytest.mark.parametrize("f", [16, 128])
def test_capture_before_prepare_is_refused(f):
    A = one_rank_matrix("rmat")
    n = A.shape[0]
    plan = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    x = rand(np.random.RandomState(1), n, f)
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="pgcn_plan_prepare"):
        with torch.cuda.graph(graph, stream=s):
            PSpMM.apply(plan, x)
    with torch.cuda.stream(s):                      # the capture was not invalidated: plan and stream still work
        z = PSpMM.apply(plan, x)
    s.synchronize()
    xn = x.cpu().numpy()
    assert_close_fp32(z.cpu().numpy(), orc.truth_forward(A, xn), fp32_tol(A, xn, int(orc.row_degree(A).max())),
                      "eager after refused capture f=%d" % f)
    plan.close()


def test_refused_capture_enqueues_nothing():
    """A capture refused because a ring instance lacks its shared-memory opt-in (the schedule itself is built) leaves
    no kernel in the caller's graph: the zero-fill of the empty rows comes after all set-up."""
    import scipy.sparse as sp
    A = sp.coo_matrix(one_rank_matrix("rmat"))
    keep = (A.row < 10) | (A.row >= 20)                      # rows 10..19 without entries
    A = sp.csr_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)
    n, f = A.shape[0], 128
    assert (orc.row_degree(A) == 0).sum() == 10
    plan = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    x = rand(np.random.RandomState(2), n, f)
    PSpMM.apply(plan, x)                                     # eager: ring schedule and the 16-slot instance
    torch.cuda.synchronize()
    plan.set_option("ring_slots", 32)                        # same schedule, a ring instance not opted in yet
    launches = plan.launch_count()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="pgcn_plan_prepare"):
        with torch.cuda.graph(graph, stream=s):
            PSpMM.apply(plan, x)
    assert plan.launch_count() == launches, "the refused call enqueued %d kernels" % (plan.launch_count() - launches)
    with torch.cuda.stream(s):                              # the capture was not invalidated: plan and stream still work
        z = PSpMM.apply(plan, x)
    s.synchronize()
    xn = x.cpu().numpy()
    assert_close_fp32(z.cpu().numpy(), orc.truth_forward(A, xn), fp32_tol(A, xn, int(orc.row_degree(A).max())),
                      "eager after refused capture with empty rows")
    plan.close()


@pytest.mark.parametrize("overlap", [1, 0])
@pytest.mark.parametrize("case", ["gemat11_k2", "gemat11_k3_hp", "karate_k3_hp", "rmat_k4"])
def test_peer_transport_capture_and_replay(case, overlap):
    if case == "rmat_k4":
        n, f, k = 12000, 128, 4
        A = graphio.synthetic_graph(n, 240000, seed=4)
        pv = graphio.random_partvec(n, k, seed=9)
    else:
        g = Golden(case)
        A, pv, f, k, n = g.A, g.partvec, g.f, g.k, g.n
    lib = cabi.load()
    plans = [planmod.build_plan(A, pv, r, k, f, device=dev()) for r in range(k)]
    planmod.link_local_plans(plans)
    for p in plans:
        p.set_option("overlap", overlap)
        p.prepare(f)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    m = [p.lp.m for p in plans]
    rs = np.random.RandomState(17 + k)
    inputs = [(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.uniform(-1, 1, size=(n, f)).astype(np.float32))
              for _ in range(5)]
    x = [torch.zeros((m[r], f), device=dev()) for r in range(k)]
    gz = [torch.zeros((m[r], f), device=dev()) for r in range(k)]
    z = [torch.zeros((m[r], f), device=dev()) for r in range(k)]
    gh = [torch.zeros((m[r], f), device=dev()) for r in range(k)]

    def fused(r, xr, zr, gr, hr):
        def call():
            st = torch.cuda.current_stream().cuda_stream
            cabi.check(lib.pgcn_forward(plans[r].handle, xr.data_ptr(), zr.data_ptr(), f, st), plans[r].handle)
            cabi.check(lib.pgcn_backward(plans[r].handle, gr.data_ptr(), hr.data_ptr(), f, st), plans[r].handle)
        return call

    graphs = []
    for r in range(k):                               # capture does not run anything: no rank waits for another
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=streams[r]):
            fused(r, x[r], z[r], gz[r], gh[r])()
        graphs.append(graph)

    def load(i):
        H, G = inputs[i]
        for r, p in enumerate(plans):
            x[r].copy_(torch.from_numpy(H[p.lp.owned])); gz[r].copy_(torch.from_numpy(G[p.lp.owned]))
        torch.cuda.synchronize()

    def eager(i, extra_forward=False):
        H, G = inputs[i]
        xe = [torch.from_numpy(H[p.lp.owned]).to(dev()) for p in plans]
        ge = [torch.from_numpy(G[p.lp.owned]).to(dev()) for p in plans]
        ze = [torch.empty_like(t) for t in xe]
        he = [torch.empty_like(t) for t in xe]
        if extra_forward:                            # one more exchange: the replays after it see the other parities
            run_ranks(plans, lambda r: fused(r, xe[r], ze[r], ge[r], he[r])(), streams)
            z1 = [t.clone() for t in ze]
            run_ranks(plans, lambda r: cabi.check(lib.pgcn_forward(
                plans[r].handle, xe[r].data_ptr(), ze[r].data_ptr(), f, torch.cuda.current_stream().cuda_stream),
                plans[r].handle), streams)
            assert all(torch.equal(a, b) for a, b in zip(z1, ze))
            return ze, he, 3
        run_ranks(plans, lambda r: fused(r, xe[r], ze[r], ge[r], he[r])(), streams)
        return ze, he, 2

    calls = 0
    got = {}
    for i, mode in enumerate(["eager", "replay", "replay", "eager", "replay"]):
        if mode == "eager":
            ze, he, c = eager(i, extra_forward=(i == 3))
            calls += c
            got[i] = (ze, he)
        else:
            load(i)
            run_ranks(plans, lambda r: graphs[r].replay(), streams)
            calls += 2
            got[i] = ([t.clone() for t in z], [t.clone() for t in gh])
    for i in (1, 2, 4):                              # the eager result of every replayed input
        ze, he, c = eager(i)
        calls += c
        for r in range(k):
            assert torch.equal(got[i][0][r], ze[r]), "%s forward replay %d rank %d" % (case, i, r)
            assert torch.equal(got[i][1][r], he[r]), "%s backward replay %d rank %d" % (case, i, r)
    for i, (H, G) in enumerate(inputs):
        Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
        tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
        for r, p in enumerate(plans):
            own = p.lp.owned
            assert_close_fp32(got[i][0][r].cpu().numpy(), Z64[own], tolZ[own], "%s fwd step %d r%d" % (case, i, r))
            assert_close_fp32(got[i][1][r].cpu().numpy(), G64[own], tolG[own], "%s bwd step %d r%d" % (case, i, r))
    for p in plans:
        assert p.get_option("epoch") == calls
        p.close()


def test_replaced_schedules_are_retired_until_destroy():
    A = one_rank_matrix("rmat")
    n, f = A.shape[0], 128
    plan = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    plan.prepare(f)
    rs = np.random.RandomState(5)
    x_in, x_next = rand(rs, n, f), rand(rs, n, f)
    x = x_in.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z = PSpMM.apply(plan, x)
    want = PSpMM.apply(plan, x_next)                         # eager, the options of the capture
    assert plan.get_option("retired_schedules") == 0
    plan.set_option("ring_edges_per_block", 64)
    plan.set_option("edges_per_block", 16)
    other = PSpMM.apply(plan, x_next)                        # new schedules; the old ones belong to the graph
    torch.cuda.synchronize()
    assert plan.get_option("retired_schedules") > 0          # checked before the graph reads them again
    x.copy_(x_next)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(z, want)
    xn = x_next.cpu().numpy()
    assert_close_fp32(other.cpu().numpy(), orc.truth_forward(A, xn), fp32_tol(A, xn, int(orc.row_degree(A).max())),
                      "new options")
    plan.close()


def test_minibatch_trainer_with_cuda_graphs(tmp_path):
    from scipy.io import mmwrite
    import scipy.sparse as sp
    from pgcn_b200 import minibatch
    ref = json.load(open(os.path.join(GOLDEN, "karate_minibatch_e2e.json")))
    zg = np.load(os.path.join(GOLDEN, "karate_minibatch.npz"))
    n = int(zg["n"])
    a = str(tmp_path / "karate.mtx")
    mmwrite(a, sp.coo_matrix((zg["val"], (zg["row"], zg["col"])), shape=(n, n)))
    pv = str(tmp_path / "pv1.pkl")
    pickle.dump([0] * n, open(pv, "wb"))
    res = {}
    text = {}
    for graphs in (False, True):
        buf = io.StringIO()
        res[graphs] = minibatch.run(0, 1, ref["layers"], ref["f"], a, pv, "nccl", ref["batch_size"], out=buf,
                                    seed=ref["seed"], cuda_graph=graphs)
        text[graphs] = buf.getvalue()
    np.testing.assert_allclose(res[True]["losses"], ref["losses"], rtol=5e-4)
    np.testing.assert_allclose(res[True]["losses"], res[False]["losses"], rtol=1e-5)
    assert (res[True]["total_vol"], res[True]["total_nmsg"]) == (res[False]["total_vol"], res[False]["total_nmsg"])
    lines = {g: [l for l in text[g].splitlines() if not l.startswith("Elapsed time")] for g in text}
    assert lines[True] == lines[False]


# ---- >= 2 GPUs: one process per GPU --------------------------------------------------------------------------------

def _worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    g = Golden("gemat11_k2")
    d = torch.device("cuda", rank)
    p = planmod.build_plan(g.A, g.partvec, rank, k, g.f, device=d)
    used = p.init_comm(transport=transport)
    p.prepare(g.f)
    own = p.lp.owned
    rs = np.random.RandomState(3)
    ins = [(torch.from_numpy(rs.uniform(-1, 1, size=(g.n, g.f)).astype(np.float32)[own]).to(d),
            torch.from_numpy(rs.uniform(-1, 1, size=(g.n, g.f)).astype(np.float32)[own]).to(d)) for _ in range(3)]
    x = torch.zeros_like(ins[0][0], requires_grad=True)
    gz = torch.zeros_like(ins[0][1])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z = PSpMM.apply(p, x)
        z.backward(gz)
    for xi, gi in ins:
        with torch.no_grad():
            x.copy_(xi); gz.copy_(gi)
        graph.replay()
        zr, hr = z.detach().clone(), x.grad.clone()
        ze, he = eager_fwd_bwd(PSpMM, p, xi, gi)
        torch.cuda.synchronize()
        assert torch.equal(zr, ze) and torch.equal(hr, he)
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used


@pytest.mark.multigpu
@pytest.mark.parametrize("transport,port", [("nccl", 29851), ("p2p", 29852)])
def test_two_gpus_capture_and_replay(transport, port):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    assert spawn_ranks(_worker, 2, (port, transport)) == {0: transport, 1: transport}
