"""The peer-memory transport of the halo exchange on ONE GPU (so a single-GPU machine runs it):

  * every rank's plan in this process on cuda:0, wired with plan.link_local_plans (same-process peers are reached
    through plain device pointers): fused put + epoch-signal kernels, per-peer wait kernels, the per-peer pipelined
    forward (own columns while rows travel, each source's block as it lands) and backward (partials for each peer
    first, leaving while the rest is computed) — against the fp64 truth, the reference's golden outputs, the
    non-overlapped path, and repeated calls (epoch parity of the double-buffered slabs);
  * two PROCESSES sharing cuda:0 through CUDA IPC and PgcnPlan.init_comm(transport="p2p") over gloo.

NCCL refuses two ranks on one device; its path is covered by tests/test_multigpu.py on >= 2 GPUs.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from harness import ROOT, dev
from helpers import Golden, assert_close_fp32, fp32_tol
from oracle import pgcn_oracle as orc
from pgcn_b200 import cabi, graphio, plan as planmod

pytestmark = pytest.mark.gpu


def run_all(plans, fn_name, inputs, f):
    """Enqueue one fused forward/backward per rank, each on its own stream (nothing blocks on the host: the
    ranks' kernels wait for each other on the device), then synchronise."""
    lib = cabi.load()
    outs = [torch.empty((p.lp.m, f), device=dev()) for p in plans]
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    torch.cuda.synchronize()
    for p, x, y, s in zip(plans, inputs, outs, streams):
        cabi.check(getattr(lib, fn_name)(p.handle, x.data_ptr(), y.data_ptr(), f, s.cuda_stream), p.handle)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("case", ["gemat11_k2", "gemat11_k3_hp", "gemat11_k3_rp", "karate_k3_hp", "rmat_k4"])
def test_peer_transport_all_ranks_on_one_gpu(case):
    if case == "rmat_k4":
        n, f, k = 12000, 128, 4
        A = graphio.synthetic_graph(n, 240000, seed=4)
        pv = graphio.random_partvec(n, k, seed=9)
        rs = np.random.RandomState(3)
        H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
        G = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
        g = None
    else:
        g = Golden(case)
        A, pv, H, G, f, k = g.A, g.partvec, g.H, g.G, g.f, g.k
    plans = [planmod.build_plan(A, pv, r, k, f, device=dev()) for r in range(k)]
    assert planmod.link_local_plans(plans) == "p2p"
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
    Hd = [torch.from_numpy(H[p.lp.owned]).to(dev()) for p in plans]
    Gd = [torch.from_numpy(G[p.lp.owned]).to(dev()) for p in plans]
    res = {}
    for overlap in (1, 0):
        for p in plans:
            assert p.get_option("p2p") == 1
            p.set_option("overlap", overlap)
        l0 = sum(p.launch_count() for p in plans)
        Z = run_all(plans, "pgcn_forward", Hd, f)
        Gr = run_all(plans, "pgcn_backward", Gd, f)
        assert sum(p.launch_count() for p in plans) - l0 >= 2 * k * (k - 1)      # put + wait kernels ran
        for r, p in enumerate(plans):
            own = p.lp.owned
            assert_close_fp32(Z[r].cpu().numpy(), Z64[own], tolZ[own], "%s fwd r%d overlap=%d" % (case, r, overlap))
            assert_close_fp32(Gr[r].cpu().numpy(), G64[own], tolG[own], "%s bwd r%d overlap=%d" % (case, r, overlap))
            if g is not None:
                np.testing.assert_allclose(Z[r].cpu().numpy(), g.get(r, "Z1_own"), rtol=2e-5,
                                           atol=2e-6 * max(1.0, np.abs(Z64).max()))
        res[overlap] = (Z, Gr)
    for r in range(k):
        torch.testing.assert_close(res[1][0][r], res[0][0][r], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(res[1][1][r], res[0][1][r], rtol=1e-4, atol=1e-5)
    # repeated exchanges: slabs are re-used every second epoch, results must not change by a bit
    for _ in range(4):
        Z = run_all(plans, "pgcn_forward", Hd, f)
    for r in range(k):
        assert torch.equal(Z[r], res[0][0][r])
    for p in plans:
        p.close()


WORKER = r"""
import os, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import numpy as np, torch, torch.distributed as dist
from helpers import Golden, fp32_tol
from oracle import pgcn_oracle as orc
from pgcn_b200 import plan as planmod
from pgcn_b200.op import PSpMM
rank, k = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=k)
g = Golden(%(case)r)
d = torch.device("cuda", 0)
torch.cuda.set_device(d)
p = planmod.build_plan(g.A, g.partvec, rank, k, g.f, device=d)
used = p.init_comm(transport="p2p", nccl_fallback=False)
assert used == "p2p", used
own = p.lp.owned
Hd = torch.from_numpy(g.H[own]).to(d).requires_grad_(True)
Z = PSpMM.apply(p, Hd)
Z.backward(torch.from_numpy(g.G[own]).to(d))
for _ in range(3):
    Z2 = PSpMM.apply(p, Hd.detach())
torch.cuda.synchronize()
assert torch.equal(Z2, Z.detach())
Z64 = orc.truth_forward(g.A, g.H)[own]; G64 = orc.truth_backward(g.A, g.G)[own]
tz = fp32_tol(g.A, g.H, int(orc.row_degree(g.A).max()))[own]
tg = fp32_tol(g.A.T, g.G, int(orc.row_degree(g.A.T).max()))[own]
assert (np.abs(Z.detach().cpu().numpy() - Z64) <= tz).all()
assert (np.abs(Hd.grad.cpu().numpy() - G64) <= tg).all()
dist.barrier()
p.close()
print("rank %%d ok" %% rank)
"""


def test_peer_transport_two_processes_one_gpu_over_cuda_ipc(tmp_path):
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device")
    case, k = "gemat11_k2", 2
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT, "case": case})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29611", WORLD_SIZE=str(k))
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(k)]
    outs = []
    for pr in procs:
        try:
            out, _ = pr.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            pytest.fail("two-process peer-transport worker timed out")
        outs.append(out)
    for r, (pr, out) in enumerate(zip(procs, outs)):
        assert pr.returncode == 0, "rank %d failed:\n%s" % (r, out[-3000:])
        assert "rank %d ok" % r in out


def test_more_ranks_than_the_peer_transport_takes():
    """k = 17 > 16: plans must build and the step-by-step pieces (pack -> wire order -> SpMM, A^T g -> scatter-add)
    must work — the NCCL transport has no rank limit; only pgcn_p2p_export refuses (ADVICE r1: fixed-size peer arrays)."""
    import ctypes as C
    from test_gpu_parity import forward_all, backward_all
    n, f, k = 1700, 32, 17
    A = graphio.synthetic_graph(n, 20000, seed=8)
    pv = graphio.random_partvec(n, k, seed=2)
    H = np.random.RandomState(1).uniform(-1, 1, size=(n, f)).astype(np.float32)
    plans = [planmod.build_plan(A, pv, r, k, f, device=dev()) for r in range(k)]
    Z = forward_all(plans, H)
    Gd = backward_all(plans, H)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, H)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, H, int(orc.row_degree(A.T).max()))
    for r, p in enumerate(plans):
        own = p.lp.owned
        assert_close_fp32(Z[r].cpu().numpy(), Z64[own], tolZ[own], "k=17 fwd r%d" % r)
        assert_close_fp32(Gd[r].cpu().numpy(), G64[own], tolG[own], "k=17 bwd r%d" % r)
    blob = C.create_string_buffer(cabi.P2P_HANDLE_BYTES)
    assert cabi.load().pgcn_p2p_export(plans[0].handle, blob) < 0          # refused, with a message
    assert b"16" in cabi.load().pgcn_last_error(plans[0].handle)
    for p in plans:
        p.close()


@pytest.mark.parametrize("case,k", [("karate_k3", 3), ("unsym_k4_rp", 4)])
def test_operator_driven_from_the_cpu_partitioner_output(case, k):
    """SURVEY.md §8f rank 4 closed on the GPU: the files the reference's CPU-path partitioner `gcnhgp` wrote
    (A.k / H.k / conn.k / buff.k / config, GCN-HP/main.cpp:117-282) -> graphio.read_cpu_partition -> plans -> the
    fused forward / backward over the peer transport (all ranks on this GPU), with the trainer's first-layer input
    H0 = 1.0 on every owned row (Parallel-GCN/main.c:650-684). Checked rank by rank against the C restatement of
    the GraphBLAS aggregation (AH = A*H on own rows, then += per received block, main.c:271,295) and the fp64 truth;
    the exchanged row counts equal the reference's own buff.k counts where its connectivity rule applies (symmetric
    pattern)."""
    from oracle import build_oracle
    d = os.path.join(ROOT, "tests", "golden", "cpu_path", case)
    P = graphio.read_cpu_partition(d, k)
    A, pv = P["A"].tocoo(), P["partvec"]
    n = A.shape[0]
    f = 4 * max(1, int(P["config"]["widths"][0]))            # a multiple of 4 so the peer-store kernels take it
    plans = [planmod.build_plan(A, pv, r, k, f, device=dev()) for r in range(k)]
    planmod.link_local_plans(plans)
    H = np.ones((n, f), dtype=np.float32) * (1.0 + np.arange(f, dtype=np.float32)[None, :])   # H0 rows identical per column
    G = np.random.RandomState(5).uniform(-1, 1, size=(n, f)).astype(np.float32)
    Hd = [torch.from_numpy(H[p.lp.owned]).to(dev()) for p in plans]
    Gd = [torch.from_numpy(G[p.lp.owned]).to(dev()) for p in plans]
    Z = run_all(plans, "pgcn_forward", Hd, f)
    Gr = run_all(plans, "pgcn_backward", Gd, f)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
    for r, p in enumerate(plans):
        lp = p.lp
        assert_close_fp32(Z[r].cpu().numpy(), Z64[lp.owned], tolZ[lp.owned], "%s fwd r%d" % (case, r))
        assert_close_fp32(Gr[r].cpu().numpy(), G64[lp.owned], tolG[lp.owned], "%s bwd r%d" % (case, r))
        Hcat = np.concatenate([H[lp.owned], H[lp.halo]], 0)
        Zc = build_oracle.grb_aggregate(lp.rowptr, lp.colidx, lp.vals, Hcat, lp.recv_off, lp.m)
        np.testing.assert_allclose(Z[r].cpu().numpy(), Zc, rtol=3e-5, atol=3e-6)
        if case == "karate_k3":                                # symmetric: the reference's buff.k == the plan's counts
            bs, br = P["buff"][r]
            assert sum(bs.values()) == lp.S and sum(br.values()) == lp.h
        p.close()


@pytest.mark.parametrize("case", ["gemat11_k1", "gemat11_k3_hp", "rmat_k4"])
def test_fused_relu_epilogue_equals_reference_layer(case):
    """SURVEY.md §8f rank 1: relu fused into the aggregation's store — relu(A (H W^T)) through pgcn_forward with the
    plan option "relu" — equals the reference layer relu(linear(PSpMM(A, H))) (GPU/PGCN.py:144-148) computed in fp64,
    on one rank (single pass), on 3 / 4 ranks with the per-peer pipelined forward (each row clamped by the launch that
    writes it last) and without overlap; rows with a long neighbour list go through the split-row fixup; the
    backward mask is relu's (out > 0)."""
    from pgcn_b200.op import PSpMMRelu
    if case == "rmat_k4":
        n, f, k = 9000, 128, 4
        A = graphio.synthetic_graph(n, 200000, seed=14)
        pv = graphio.random_partvec(n, k, seed=3)
        H = np.random.RandomState(2).uniform(-1, 1, size=(n, f)).astype(np.float32)
    else:
        g = Golden(case)
        A, pv, H, f, k, n = g.A, g.partvec, g.H, g.f, g.k, g.n
    W = np.random.RandomState(7).uniform(-0.5, 0.5, size=(f, f)).astype(np.float32)
    X = (H.astype(np.float64) @ W.T.astype(np.float64)).astype(np.float32)          # the dense step, done first
    pre64 = orc.truth_forward(A, X)                                                  # A (H W^T) in fp64
    ref = np.maximum(pre64, 0.0)
    tol = fp32_tol(A, X, int(orc.row_degree(A).max()))
    plans = [planmod.build_plan(A, pv, r, k, f, device=dev()) for r in range(k)]
    if k > 1:
        planmod.link_local_plans(plans)
    Xd = [torch.from_numpy(X[p.lp.owned]).to(dev()) for p in plans]
    for overlap in (1, 0):
        for p in plans:
            p.set_option("overlap", overlap); p.set_option("relu", 1)
            p.set_option("ring_edges_per_block", 64); p.set_option("edges_per_block", 16)   # force split rows
        Z = run_all(plans, "pgcn_forward", Xd, f)
        for r, p in enumerate(plans):
            own = p.lp.owned
            z = Z[r].cpu().numpy()
            assert (z >= 0).all()
            # exact zeros where the pre-activation is clearly negative, the fp32 bound elsewhere
            assert_close_fp32(z, ref[own], tol[own], "%s fused relu r%d overlap=%d" % (case, r, overlap))
            assert (z[pre64[own] < -tol[own]] == 0).all()
            p.set_option("relu", 0)
    if k == 1:
        # autograd: d/dX of sum(relu(A X) * G) == A^T (G * mask)
        Xt = Xd[0].clone().requires_grad_(True)
        out = PSpMMRelu.apply(plans[0], Xt)
        Gm = torch.from_numpy(np.random.RandomState(9).uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev())
        out.backward(Gm)
        mask = (pre64 > 0)
        gref = orc.truth_backward(A, Gm.cpu().numpy() * mask)
        sure = np.abs(pre64) > tol                                                    # mask bits fp32 cannot flip
        if sure.all():
            np.testing.assert_allclose(Xt.grad.cpu().numpy(), gref, rtol=1e-4, atol=1e-5 * max(1.0, np.abs(gref).max()))
        assert plans[0].get_option("relu") == 0
    for p in plans:
        p.close()
