"""Max aggregation on the H100 path: pgcn_forward_max, pgcn_backward_max, op.PSpMMMax and PSAGE.py.

  * the forward equals the NumPy oracle (sage_oracle.max_aggregate) bit for bit, Z and arg, on gemat11, a hub graph
    (a row of 3000 entries split into segments, empty rows, rows of one entry) and a matrix with duplicated entries,
    at widths 1 .. 256, with two block sizes (one of them cuts the hub row into about 190 segments), with every operand 4 bytes
    into its buffer, twice;
  * ties everywhere (integer H) give the first entry; NaN (with payloads), +-inf, rows of all -inf and signed zeros give
    the oracle's bits;
  * the backward lies within the fp32 bound of the fp64 routed gradient, is run-to-run identical and gives the same bits
    from the scalar and vector instances; both calls refuse an unbound plan;
  * on 2 and 3 ranks (peer transport, in-process linked plans) Z equals the one-rank Z, arg names the same global
    columns and G lies within the fp32 bound; on two GPUs NCCL gives the peer transport's bits;
  * PSpMMMax's gradient against the oracle on one and three ranks; CUDA-graph capture on one and two ranks;
  * PSAGE.py follows the fp64 loss curve, and the layer on 3 ranks follows the one-rank curve.
"""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import sage_oracle as so
from harness import (assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from helpers import fp32_tol
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PSpMMMax, aggregate_max, aggregate_max_backward

pytestmark = pytest.mark.gpu
WIDTHS = [1, 3, 4, 8, 64, 128, 132, 256]
SCHEDULES = {"default": {}, "segments": {"edges_per_block": 16, "long_row": 32}}


def with_duplicates(lp):
    """lp (k = 1) with a second copy of every 3rd entry appended at the end of its row: duplicated (row, column) entries
    reach the plan, and the transpose holds them in forward order."""
    rows = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
    cols = lp.colidx.astype(np.int64)
    extra = np.arange(0, len(cols), 3)
    r = np.concatenate([rows, rows[extra]])
    c = np.concatenate([cols, cols[extra]])
    order = np.argsort(r, kind="stable")
    r, c = r[order], c[order]
    out = planmod.LocalPlan()
    for name in ("n", "k", "rank", "m", "h", "S", "owned", "halo", "send_idx", "send_gid", "send_off", "recv_off"):
        setattr(out, name, getattr(lp, name))
    out.rowptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=lp.m))]).astype(np.int32)
    out.colidx = c.astype(np.int32)
    out.vals = np.ones(len(c), np.float32)
    tor = np.argsort(c, kind="stable")
    out.t_rowptr = np.concatenate([[0], np.cumsum(np.bincount(c, minlength=lp.m + lp.h))]).astype(np.int32)
    out.t_colidx = r[tor].astype(np.int32)
    out.t_vals = np.ones(len(c), np.float32)
    return out


def one_rank_plan(case, f, opts=None, bind=True):
    A, _, _ = problem("gemat11_k1" if case == "dup" else case)
    lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    if case == "dup":
        lp = with_duplicates(lp)
    plan = planmod.PgcnPlan(lp, f, device=dev())
    for k, v in (opts or {}).items():
        plan.set_option(k, v)
    if bind:
        plan.bind_values()
    return plan


def run_max(plan, H, f):
    lp = plan.lp
    Z = torch.full((lp.m, f), float("nan"), device=dev())
    arg = torch.full((lp.m, f), -7, dtype=torch.int32, device=dev())
    cabi.check(cabi.load().pgcn_forward_max(plan.handle, H.data_ptr(), Z.data_ptr(), arg.data_ptr(), f, stream()),
               plan.handle)
    return Z, arg


def run_max_backward(plan, arg, g, f):
    G = torch.full((plan.lp.m, f), float("nan"), device=dev())
    cabi.check(cabi.load().pgcn_backward_max(plan.handle, arg.data_ptr(), g.data_ptr(), G.data_ptr(), f, stream()),
               plan.handle)
    return G


def backward_tol(lp, gZ):
    """The fp32 bound of a sum of gZ values into each column (pattern values 1)."""
    P = sp.csr_matrix((np.ones(lp.nnz()), lp.colidx, lp.rowptr), shape=(lp.m, lp.m + lp.h))
    return fp32_tol(P.T, np.abs(gZ), int(np.diff(lp.t_rowptr).max()))[:lp.m]


@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_forward_bit_exact_and_backward_within_fp32(case, f, sched):
    plan = one_rank_plan(case, f, SCHEDULES[sched])
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() >= 3000 and (deg == 0).any() and (deg == 1).any()
    rs = np.random.RandomState(f + len(case))
    Hn = rs.standard_normal((lp.m, f)).astype(np.float32)
    gn = rs.uniform(-1, 1, (lp.m, f)).astype(np.float32)
    Zo, ao = so.max_aggregate(lp.rowptr, lp.colidx, Hn)
    H, g = t(Hn), t(gn)
    Z, arg = run_max(plan, H, f)
    assert np.array_equal(bits(Z), Zo.view(np.uint32)) and np.array_equal(bits(arg), ao)
    Z2, arg2 = run_max(plan, H, f)
    assert torch.equal(Z2, Z) and torch.equal(arg2, arg)
    G = run_max_backward(plan, arg, g, f)
    G64 = so.max_backward(lp.colidx, ao, gn, lp.m + lp.h)[:lp.m]
    assert (np.abs(G.cpu().numpy() - G64) <= backward_tol(lp, gn)).all()
    assert torch.equal(run_max_backward(plan, arg, g, f), G)
    # every operand 4 bytes into its buffer: the scalar instances, the same bits
    Hs, gs, args = shifted(H), shifted(g), shifted(arg)
    Zs, argz = shifted(torch.full_like(Z, float("nan"))), shifted(torch.full_like(arg, -7))
    cabi.check(cabi.load().pgcn_forward_max(plan.handle, Hs.data_ptr(), Zs.data_ptr(), argz.data_ptr(), f, stream()),
               plan.handle)
    Gs = shifted(torch.full_like(G, float("nan")))
    cabi.check(cabi.load().pgcn_backward_max(plan.handle, args.data_ptr(), gs.data_ptr(), Gs.data_ptr(), f, stream()),
               plan.handle)
    assert np.array_equal(bits(Zs), bits(Z)) and torch.equal(argz, arg) and np.array_equal(bits(Gs), bits(G))
    plan.close()


@pytest.mark.parametrize("f", [5, 8, 64])
@pytest.mark.parametrize("case,sched", [("hub", "segments"), ("hub", "default"), ("gemat11_k1", "default")])
def test_ties_and_ieee_special_values(case, sched, f):
    plan = one_rank_plan(case, f, SCHEDULES[sched])
    lp = plan.lp
    rs = np.random.RandomState(f)
    # ties everywhere: the first entry of the largest value
    Hn = rs.randint(0, 4, (lp.m, f)).astype(np.float32)
    Z, arg = run_max(plan, t(Hn), f)
    Zo, ao = so.max_aggregate(lp.rowptr, lp.colidx, Hn)
    assert np.array_equal(bits(Z), Zo.view(np.uint32)) and np.array_equal(bits(arg), ao)
    # NaN with payloads, +-inf, signed zeros; the columns of one row all -inf, of another all zeros of both signs
    Hn = rs.standard_normal((lp.m, f)).astype(np.float32)
    u = rs.uniform(size=Hn.shape)
    Hn[u < 0.02] = np.inf
    Hn[(u >= 0.02) & (u < 0.04)] = -np.inf
    Hn[(u >= 0.04) & (u < 0.06)] = -0.0
    Hn[(u >= 0.06) & (u < 0.08)] = 0.0
    nan_at = (u >= 0.08) & (u < 0.09)
    Hn.view(np.uint32)[nan_at] = 0x7fc00000 | rs.randint(1, 1 << 22, nan_at.sum()).astype(np.uint32)
    deg = np.diff(lp.rowptr.astype(np.int64))
    r_zero, r_inf = np.flatnonzero(deg > 1)[:2]
    zc = lp.colidx[lp.rowptr[r_zero]:lp.rowptr[r_zero + 1]]
    Hn[zc] = np.where(rs.uniform(size=(len(zc), f)) < 0.5, -0.0, 0.0).astype(np.float32)
    Hn[lp.colidx[lp.rowptr[r_inf]:lp.rowptr[r_inf + 1]]] = -np.inf
    Z, arg = run_max(plan, t(Hn), f)
    Zo, ao = so.max_aggregate(lp.rowptr, lp.colidx, Hn)
    assert np.array_equal(bits(Z), Zo.view(np.uint32)) and np.array_equal(bits(arg), ao)
    assert np.all(np.isneginf(Zo[r_inf]))
    plan.close()


def test_unbound_plan_is_refused():
    plan = one_rank_plan("gemat11_k1", 8, bind=False)
    lib = cabi.load()
    x = torch.zeros((plan.lp.m, 8), device=dev())
    a = torch.zeros((plan.lp.m, 8), dtype=torch.int32, device=dev())
    assert lib.pgcn_forward_max(plan.handle, x.data_ptr(), x.data_ptr(), a.data_ptr(), 8, stream()) == -5
    assert b"pgcn_plan_bind_values" in lib.pgcn_last_error(plan.handle)
    assert lib.pgcn_backward_max(plan.handle, a.data_ptr(), x.data_ptr(), x.data_ptr(), 8, stream()) == -5
    with pytest.raises(RuntimeError, match="bind_values"):
        PSpMMMax.apply(plan, x)
    plan.bind_values()
    assert lib.pgcn_forward_max(plan.handle, x.data_ptr(), x.data_ptr(), a.data_ptr(), 9, stream()) == -1
    assert lib.pgcn_forward_max(plan.handle, None, x.data_ptr(), a.data_ptr(), 8, stream()) == -1
    assert lib.pgcn_backward_max(plan.handle, None, x.data_ptr(), x.data_ptr(), 8, stream()) == -1
    plan.close()


def tie_free(n, f, seed):
    return (np.random.RandomState(seed).permutation(n * f).reshape(n, f).astype(np.float32) - n * f / 2) / 64.0


def global_cols(lp, arg):
    a = arg.cpu().numpy()
    gid = np.concatenate([lp.owned, lp.halo]).astype(np.int64)
    return np.where(a >= 0, gid[lp.colidx.astype(np.int64)[np.maximum(a, 0)]], -1)


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("case,f", [("gemat11_k2", 128), ("gemat11_k2", 20), ("gemat11_k3_hp", 64),
                                    ("gemat11_k3_hp", 132)])
def test_multi_rank_equals_one_rank(case, f, overlap):
    A, pv, k = problem(case)
    n = A.shape[0]
    Hn = tie_free(n, f, f)
    gn = np.random.RandomState(f + 1).uniform(-1, 1, (n, f)).astype(np.float32)
    one = one_rank_plan(case, f)
    Z1, a1 = run_max(one, t(Hn), f)
    c1 = global_cols(one.lp, a1)
    lp1 = one.lp
    _, ao = so.max_aggregate(lp1.rowptr, lp1.colidx, Hn)
    G64 = so.max_backward(lp1.colidx, ao, gn, n)
    tol = backward_tol(lp1, gn)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    Hr = [t(Hn[lp.owned]) for lp in lps]
    gr = [t(gn[lp.owned]) for lp in lps]
    for rep in range(2):                                  # both epoch parities of the peer slabs
        out = run_ranks(plans, lambda r: run_max(plans[r], Hr[r], f), streams)
        G = run_ranks(plans, lambda r: run_max_backward(plans[r], out[r][1], gr[r], f), streams)
        for r, lp in enumerate(lps):
            w = "%s f=%d overlap=%d rank %d rep %d" % (case, f, overlap, r, rep)
            assert np.array_equal(bits(out[r][0]), bits(Z1)[lp.owned]), w + ": Z"
            assert np.array_equal(global_cols(lp, out[r][1]), c1[lp.owned]), w + ": arg"
            assert (np.abs(G[r].cpu().numpy() - G64[lp.owned]) <= tol[lp.owned]).all(), w + ": G"
    for p in plans + [one]:
        p.close()


@pytest.mark.parametrize("layout", ["local", "global"])
def test_autograd_one_rank(layout):
    plan = one_rank_plan("hub", 32)
    plan.layout = layout
    lp = plan.lp
    rs = np.random.RandomState(4)
    Hn = rs.standard_normal((lp.m, 32)).astype(np.float32)
    gn = rs.uniform(-1, 1, (lp.m, 32)).astype(np.float32)
    H = t(Hn).requires_grad_(True)
    Z = PSpMMMax.apply(plan, H)
    Z.backward(t(gn))
    Zo, ao = so.max_aggregate(lp.rowptr, lp.colidx, Hn)
    assert np.array_equal(bits(Z), Zo.view(np.uint32))
    G64 = so.max_backward(lp.colidx, ao, gn, lp.m)
    assert (np.abs(H.grad.cpu().numpy() - G64) <= backward_tol(lp, gn)).all()
    plan.close()


def test_autograd_three_ranks():
    A, pv, k = problem("gemat11_k3_hp")
    n, f = A.shape[0], 16
    Hn = tie_free(n, f, 3)
    gn = np.random.RandomState(5).uniform(-1, 1, (n, f)).astype(np.float32)
    one = one_rank_plan("gemat11_k3_hp", f)
    _, ao = so.max_aggregate(one.lp.rowptr, one.lp.colidx, Hn)
    G64 = so.max_backward(one.lp.colidx, ao, gn, n)
    tol = backward_tol(one.lp, gn)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    H = [t(Hn[lp.owned]).requires_grad_(True) for lp in lps]
    Z = run_ranks(plans, lambda r: PSpMMMax.apply(plans[r], H[r]), streams)
    run_ranks(plans, lambda r: Z[r].backward(t(gn[lps[r].owned])), streams)
    for r, lp in enumerate(lps):
        assert (np.abs(H[r].grad.cpu().numpy() - G64[lp.owned]) <= tol[lp.owned]).all(), "rank %d" % r
    for p in plans + [one]:
        p.close()


def test_one_rank_capture_and_refusal_before_prepare():
    f = 64
    plan = one_rank_plan("hub", f, SCHEDULES["segments"])
    m = plan.lp.m
    x, g = torch.zeros((m, f), device=dev()), torch.zeros((m, f), device=dev())
    rs = np.random.RandomState(2)
    ins = [(t(rs.standard_normal((m, f)).astype(np.float32)), t(rs.uniform(-1, 1, (m, f)).astype(np.float32)))
           for _ in range(3)]

    def step(x, g):
        Z, arg = aggregate_max(plan, x)
        return dict(Z=Z, arg=arg, G=aggregate_max_backward(plan, arg, g))

    def load(i):
        x.copy_(ins[i][0]); g.copy_(ins[i][1])

    check_one_rank_capture(plan, lambda: step(x, g), load, lambda i: step(*ins[i]), prepare=(f,))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n = 128, A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(6)
    ins = [(tie_free(n, f, i), rs.uniform(-1, 1, (n, f)).astype(np.float32)) for i in range(3)]

    def buffers(r):
        return dict(x=torch.zeros((lps[r].m, f), device=dev()), g=torch.zeros((lps[r].m, f), device=dev()))

    def load(bufs, i):
        Hn, gn = ins[i]
        for r, lp in enumerate(lps):
            bufs[r]["x"].copy_(t(Hn[lp.owned])); bufs[r]["g"].copy_(t(gn[lp.owned]))
        torch.cuda.synchronize()

    def step(r, b):
        Z, arg = aggregate_max(plans[r], b["x"])
        return dict(Z=Z, arg=arg, G=aggregate_max_backward(plans[r], arg, b["g"]))

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


def _nccl_worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    A, pv, _ = problem("gemat11_k2")
    n, f = A.shape[0], 128
    p = planmod.build_plan(A, pv, rank, k, f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    Hd = torch.from_numpy(tie_free(n, f, 1)[own]).cuda().requires_grad_(True)
    Z = PSpMMMax.apply(p, Hd)
    Z.backward(torch.from_numpy(np.random.RandomState(2).uniform(-1, 1, (n, f)).astype(np.float32)[own]).cuda())
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, Z.detach().cpu().numpy(), Hd.grad.cpu().numpy()


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29861, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29862, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        assert np.array_equal(a[r][1].view(np.uint32), b[r][1].view(np.uint32))
        assert np.array_equal(a[r][2].view(np.uint32), b[r][2].view(np.uint32))


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PSAGE.py", [], 29681)
    assert_follows(lines, so.intended_training(karate(), 2, 4, 7))


def test_layer_on_three_ranks_follows_the_one_rank_curve():
    """sage.run's training loop with the three ranks of karate_k3 in this process (peer transport), against the same
    loop on one rank and against the fp64 oracle with gradients averaged over three ranks."""
    import torch.nn as nn
    import torch.nn.functional as F
    from pgcn_b200.sage import PSAGE
    A, pv, k = problem("karate")
    n, f, L, epochs = A.shape[0], 4, 2, 50

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = nn.Sequential(*[PSAGE(p, f, f) for _ in range(L)]).to(dev())
            models.append(m)
            opts.append(torch.optim.Adam(m.parameters(), lr=1e-3))
        H = [t(np.repeat(lp.owned.astype(np.float32)[:, None], f, axis=1)) for lp in lps]
        y = [torch.from_numpy(lp.owned % f).to(dev()) for lp in lps]
        losses = []
        for _ in range(epochs):
            logits = run_ranks(plans, lambda r: models[r](H[r]), streams)
            loss = [F.nll_loss(F.log_softmax(logits[r], 1), y[r], reduction="sum") / n for r in range(kk)]
            for o in opts:
                o.zero_grad()
            run_ranks(plans, lambda r: loss[r].backward(), streams)
            with torch.no_grad():
                for ps in zip(*[m.parameters() for m in models]):
                    avg = sum(q.grad for q in ps) / kk
                    for q in ps:
                        q.grad.copy_(avg)
            for o in opts:
                o.step()
            losses.append(float(sum(float(x) for x in loss)))
        return losses

    lp1 = [planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)]
    one = [planmod.PgcnPlan(lp1[0], f, device=dev())]
    one[0].bind_values()
    curve1 = train(one, lp1)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    curve3 = train(plans, lps)
    np.testing.assert_allclose(curve1, so.intended_training(A, L, f, 7), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, so.intended_training(A, L, f, 7, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
    for p in plans + one:
        p.close()
