"""Gated aggregation on the H100 path: pgcn_gated_forward / _backward_rows / _backward_cols, pgcn_halo_rows_add,
op.PSpMMGated and PGATED.py.

The fp32 bound. Every output element is one fp32 sum of d terms (d the row's entry count for Z and dK, the column's for
dQ and dV, across all ranks), each term a product of a gate value with an operand. The kernels' gate is
eta = rcp_rn(1 + expf(-x)) on x = fl(K[i] + Q[j]), the oracle's x (gated_oracle.terms rounds it the same way), so a
gate carries expf's 2 ulp plus one rounding each for the sum and the reciprocal: 4 ulp; eta (1 - eta) =
eta * (expf(-x) * eta) adds 2 + 4 + 2 more, 12 in all; the final product with gZ[i] or V[j] one more. The halo partials
of dQ and dV add at most k - 1 <= 2 roundings at their owner. So every element lies within
(d + C) 2^-24 sum|terms| with C = 16, plus 1e-30 for exact zeros.

  * forward and the three gradients against fp64 on gemat11, the hub graph (a split row of 3000 entries, empty rows,
    rows of one entry) and a local plan with duplicated entries, at widths 1 .. 256; run-to-run bits; every operand 4
    bytes into its buffer (the scalar instances) gives the vector instances' bits;
  * a graph whose rows all fall under the chunk and the same graph walked with a chunk of 4: both within the bound;
  * +-inf and NaN in K, Q or V: NaN and +-inf exactly where the fp32 reference has them;
  * torch.profiler, in a process of its own, sees every instance of tests/gated_kernel_instances.txt, each checked;
  * 2 and 3 ranks over the peer transport within the bound of the one-rank fp64 result; pgcn_halo_rows_add against a
    NumPy scatter-add; on two GPUs NCCL gives the peer transport's bits;
  * PSpMMGated's autograd in both layouts on one rank and on three; CUDA-graph capture on one and two ranks, and a
    capture before the first eager call refused before it enqueues work;
  * PGATED.py follows the fp64 loss curve, and the layer on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gated_oracle as go
from harness import (EPS, ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PSpMMGated, aggregate_gated, aggregate_gated_backward
from test_max_aggregation import with_duplicates

pytestmark = pytest.mark.gpu
CONST = 16
WIDTHS = [1, 3, 4, 8, 64, 128, 132, 256]


def one_rank_plan(case, f):
    """A bound one-rank plan of width 2f on problem(case) ("dup": gemat11 with duplicated entries)."""
    A, _, _ = problem("gemat11_k1" if case == "dup" else case)
    lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    if case == "dup":
        lp = with_duplicates(lp)
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev())
    plan.bind_values()
    return plan


def inputs(n, f, seed):
    rs = np.random.RandomState(seed)
    return tuple((rs.standard_normal((n, f)) * s).astype(np.float32) for s in (2.0, 2.0, 1.0, 1.0))   # K, Q, V, gZ


def reference(lp, K, Q, V, gZ):
    """{name: (fp64 value, bound)} of one rank's plan (h = 0) on global inputs."""
    out = go.terms(lp.rowptr, lp.colidx, lp.m, K, Q, V, gZ)
    drow = np.diff(lp.rowptr.astype(np.int64))[:, None]
    dcol = np.diff(lp.t_rowptr.astype(np.int64))[:lp.m, None]
    return {name: (val, (d + CONST) * EPS * mag + 1e-30) for (name, (val, mag)), d in
            zip(sorted(out.items()), [drow, dcol, dcol, drow])}       # dK, dQ, dV, Z


def within(got, ref, what):
    val, tol = ref
    g = got.detach().cpu().numpy().astype(np.float64)
    err = np.abs(g - val)
    bad = ~(err <= tol)
    assert not bad.any(), "%s: %d elements beyond the fp32 bound, worst err %.3e" % (what, int(bad.sum()),
                                                                                      float(np.nanmax(err)))


def run_all(plan, K, QV, QVh, gZ, f, walks=None):
    """(Z, dK, dQV) from the three C calls, outputs NaN-filled first; walks default to the plan's."""
    fwd, tr = walks or plan.gated_walks()
    lib, lp = cabi.load_gated(), plan.lp
    Z, dK = torch.full((lp.m, f), float("nan"), device=dev()), torch.full((lp.m, f), float("nan"), device=dev())
    dQV = torch.full((lp.m + lp.h, 2 * f), float("nan"), device=dev())
    w1 = torch.empty((fwd.nslots, f), device=dev())
    w2 = torch.empty((tr.nslots, 2 * f), device=dev())
    hp = QVh.data_ptr() if QVh is not None else None
    cabi.check_gated(lib.pgcn_gated_forward(C.byref(fwd.c), lp.m, lp.h, K.data_ptr(), QV.data_ptr(), hp, Z.data_ptr(),
                                            w1.data_ptr(), f, stream()))
    cabi.check_gated(lib.pgcn_gated_backward_rows(C.byref(fwd.c), lp.m, lp.h, K.data_ptr(), QV.data_ptr(), hp,
                                                  gZ.data_ptr(), dK.data_ptr(), w1.data_ptr(), f, stream()))
    cabi.check_gated(lib.pgcn_gated_backward_cols(C.byref(tr.c), lp.m, lp.h, K.data_ptr(), QV.data_ptr(), hp,
                                                  gZ.data_ptr(), dQV.data_ptr(), w2.data_ptr(), f, stream()))
    torch.cuda.synchronize()
    return Z, dK, dQV


def check_one_rank(plan, Kn, Qn, Vn, gn, f, walks=None, shift=False):
    lp = plan.lp
    ops = [t(Kn), t(np.concatenate([Qn, Vn], 1)), t(gn)]
    if shift:
        ops = [shifted(x) for x in ops]
    K, QV, gZ = ops
    Z, dK, dQV = run_all(plan, K, QV, None, gZ, f, walks)
    ref = reference(lp, Kn, Qn, Vn, gn)
    for name, got in (("Z", Z), ("dK", dK), ("dQ", dQV[:, :f]), ("dV", dQV[:, f:])):
        within(got, ref[name], "%s f=%d" % (name, f))
    return Z, dK, dQV


@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_run_to_run_and_scalar_bits(case, f):
    if case != "gemat11_k1" and f not in (3, 8, 128, 256):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
        assert plan.gated_walks()[0].nslots > 0
    Kn, Qn, Vn, gn = inputs(lp.m, f, f + len(case))
    first = check_one_rank(plan, Kn, Qn, Vn, gn, f)
    again = check_one_rank(plan, Kn, Qn, Vn, gn, f)
    scalar = check_one_rank(plan, Kn, Qn, Vn, gn, f, shift=True)
    for a, b, s in zip(first, again, scalar):
        assert np.array_equal(bits(a), bits(b)) and np.array_equal(bits(a), bits(s))
    plan.close()


@pytest.mark.parametrize("f", [4, 5, 64])
def test_forced_small_chunk_stays_within_the_bound(f):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    chunk = cabi.load_gated().pgcn_gated_chunk()
    assert np.diff(lp.rowptr.astype(np.int64)).max() <= chunk and np.diff(lp.t_rowptr.astype(np.int64)).max() <= chunk
    assert plan.gated_walks()[0].nslots == plan.gated_walks()[1].nslots == 0
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    Kn, Qn, Vn, gn = inputs(lp.m, f, 9)
    check_one_rank(plan, Kn, Qn, Vn, gn, f)
    check_one_rank(plan, Kn, Qn, Vn, gn, f, walks=small)
    plan.close()


@pytest.mark.parametrize("f", [5, 8])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values(case, f):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    Kn, Qn, Vn, gn = inputs(lp.m, f, 3 * f)
    rs = np.random.RandomState(f)
    for x in (Kn, Qn, Vn):
        u = rs.uniform(size=x.shape)
        x[u < 0.01] = np.inf
        x[(u >= 0.01) & (u < 0.02)] = -np.inf
        x[(u >= 0.02) & (u < 0.025)] = np.nan
    Z, dK, dQV = run_all(plan, t(Kn), t(np.concatenate([Qn, Vn], 1)), None, t(gn), f)
    ref = go.fp32_reference(lp.rowptr, lp.colidx, lp.m, Kn, Qn, Vn, gn)
    for name, got in (("Z", Z), ("dK", dK), ("dQ", dQV[:, :f]), ("dV", dQV[:, f:])):
        g, w = got.cpu().numpy(), ref[name]
        assert np.isnan(w).any() and (name == "dV" or np.isinf(w).any()), name       # dV: gZ is finite, eta <= 1
        assert np.array_equal(np.isnan(g), np.isnan(w)), name
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    plan.close()


def key(name):
    """Instance name without return type, parameter list, casts and spaces, bools as 0 / 1: the manifest's and the
    profiler's spellings of one instance give the same key."""
    s = name.strip()
    for a, b in (("(int)", ""), ("(bool)", ""), ("true", "1"), ("false", "0")):
        s = s.replace(a, b)
    if s.startswith("void "):
        s = s[5:]
    return s.split("(")[0].replace(" ", "")


def _instances_worker(rank, k):
    """The keys of the gated kernels torch.profiler sees while every instance runs (vector and scalar, split rows
    through the fixup), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for f, shift in ((8, False), (5, False), (8, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        walks = (planmod.GatedWalk(lp.rowptr, lp.colidx, 64, dev()),
                 planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 64, dev()))
        assert walks[0].c.nsplits > 0 and walks[1].c.nsplits > 0
        Kn, Qn, Vn, gn = inputs(lp.m, f, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                check_one_rank(plan, Kn, Qn, Vn, gn, f, walks=walks, shift=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "gated_" in e.name}
            if len(names) == 6:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    # in a process of its own: a profiler session leaves the profiler attached to the process, and later sessions in
    # it then lose the records of their first kernels
    with open(os.path.join(ROOT, "tests", "gated_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


def rank_inputs(lps, arrays):
    return [[t(a[lp.owned]) for a in arrays] for lp in lps]


@pytest.mark.parametrize("case,f", [("gemat11_k2", 64), ("gemat11_k2", 6), ("gemat11_k3_hp", 16),
                                    ("gemat11_k3_hp", 132)])
def test_multi_rank_within_the_bound_of_one_rank(case, f):
    A, pv, k = problem(case)
    n = A.shape[0]
    Kn, Qn, Vn, gn = inputs(n, f, f + k)
    one = one_rank_plan(case, f)
    ref = reference(one.lp, Kn, Qn, Vn, gn)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = rank_inputs(lps, (Kn, Qn, Vn, gn))

    def step(r):
        K, Q, V, g = ins[r]
        Z, QV, QVh = aggregate_gated(plans[r], K, Q, V)
        return (Z,) + aggregate_gated_backward(plans[r], K, QV, QVh, g)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "dK", "dQ", "dV"), out[r]):
                val, tol = ref[name]
                within(got, (val[lp.owned], tol[lp.owned]), "%s %s rank %d rep %d" % (case, name, r, rep))
        if first is None:
            first = [[bits(x) for x in o] for o in out]
        else:
            assert all(np.array_equal(a, bits(b)) for fo, o in zip(first, out) for a, b in zip(fo, o))
    for p in plans + [one]:
        p.close()


def test_halo_rows_add_equals_a_numpy_scatter_add():
    A, pv, k = problem("gemat11_k3_hp")
    w = 12
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    # rows in several send lists: the sum really takes several peers' partials
    assert any(np.bincount(lp.send_idx).max() > 1 for lp in lps)
    plans = linked_plans(lps, w, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(8)
    X = [rs.uniform(-1, 1, (lp.h, w)).astype(np.float32) for lp in lps]
    G0 = [rs.uniform(-1, 1, (lp.m, w)).astype(np.float32) for lp in lps]
    want = [g.astype(np.float64) for g in G0]
    mag = [np.abs(g.astype(np.float64)) for g in G0]
    local = np.zeros(A.shape[0], dtype=np.int64)
    for lp in lps:
        local[lp.owned] = np.arange(lp.m)
    for lp, x in zip(lps, X):
        owner = pv[lp.halo]
        for r in range(k):
            sel = owner == r
            np.add.at(want[r], local[lp.halo[sel]], x[sel].astype(np.float64))
            np.add.at(mag[r], local[lp.halo[sel]], np.abs(x[sel].astype(np.float64)))
    lib = cabi.load()
    for rep in range(2):
        G = [t(g) for g in G0]
        Xd = [t(x) for x in X]
        run_ranks(plans, lambda r: cabi.check(lib.pgcn_halo_rows_add(plans[r].handle, Xd[r].data_ptr(),
                                                                     G[r].data_ptr(), w, stream()), plans[r].handle),
                  streams)
        for r in range(k):
            err = np.abs(G[r].cpu().numpy() - want[r])
            assert (err <= (k + 1) * EPS * mag[r] + 1e-30).all(), "rank %d rep %d" % (r, rep)
    for p in plans:
        p.close()


def test_halo_rows_add_refusals():
    plan = planmod.PgcnPlan(planmod.build_local_plan(*problem("gemat11_k2")[:2], 0, 2), 8, device=dev())
    lib = cabi.load()
    x = torch.zeros((max(plan.lp.m, plan.lp.h), 8), device=dev())
    assert lib.pgcn_halo_rows_add(plan.handle, x.data_ptr(), x.data_ptr(), 8, stream()) == -5
    assert b"pgcn_plan_bind_values" in lib.pgcn_last_error(plan.handle)
    plan.bind_values()
    assert lib.pgcn_halo_rows_add(plan.handle, x.data_ptr(), x.data_ptr(), 9, stream()) == -1
    assert lib.pgcn_halo_rows_add(plan.handle, None, x.data_ptr(), 8, stream()) == -1
    assert lib.pgcn_halo_rows_add(plan.handle, x.data_ptr(), None, 8, stream()) == -1
    plan.close()


def _nccl_worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    A, pv, _ = problem("gemat11_k2")
    n, f = A.shape[0], 64
    p = planmod.build_plan(A, pv, rank, k, 2 * f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    K, Q, V, g = (torch.from_numpy(a[own]).cuda().requires_grad_(True) for a in inputs(n, f, 1))
    Z = PSpMMGated.apply(p, K, Q, V)
    Z.backward(g.detach())
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), K.grad, Q.grad, V.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29871, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29872, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        for x, y in zip(a[r][1], b[r][1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("layout", ["local", "global"])
def test_autograd_one_rank(layout):
    f = 32
    plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp = plan.lp
    Kn, Qn, Vn, gn = inputs(lp.m, f, 4)
    K, Q, V = (t(a).requires_grad_(True) for a in (Kn, Qn, Vn))
    Z = PSpMMGated.apply(plan, K, Q, V)
    Z.backward(t(gn))
    ref = reference(lp, Kn, Qn, Vn, gn)
    for name, got in (("Z", Z), ("dK", K.grad), ("dQ", Q.grad), ("dV", V.grad)):
        within(got, ref[name], "%s %s" % (layout, name))
    plan.close()


def test_autograd_three_ranks_and_global_layout():
    A, pv, k = problem("gemat11_k3_hp")
    n, f = A.shape[0], 16
    Kn, Qn, Vn, gn = inputs(n, f, 3)
    one = one_rank_plan("gemat11_k3_hp", f)
    ref = reference(one.lp, Kn, Qn, Vn, gn)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    for layout in ("local", "global"):
        for p in plans:
            p.layout = layout
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [[t(pick(a, lp)).requires_grad_(True) for a in (Kn, Qn, Vn)] for lp in lps]
        Z = run_ranks(plans, lambda r: PSpMMGated.apply(plans[r], *leaves[r]), streams)
        run_ranks(plans, lambda r: Z[r].backward(t(pick(gn, lps[r]))), streams)
        for r, lp in enumerate(lps):
            rows = lp.owned if layout == "local" else np.arange(n)
            for name, got in zip(("Z", "dK", "dQ", "dV"), [Z[r]] + [x.grad for x in leaves[r]]):
                val, tol = ref[name]
                if layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                    within(got, (val, tol), "global %s rank %d" % (name, r))
                else:
                    within(got, (val[rows], tol[rows]), "local %s rank %d" % (name, r))
    for p in plans + [one]:
        p.close()


def test_one_rank_capture_and_refusal_before_the_first_eager_call():
    f = 64
    plan = one_rank_plan("hub", f)
    m = plan.lp.m
    K, Q, V, g = (torch.zeros((m, f), device=dev()) for _ in range(4))

    def step(K, Q, V, g):
        Z, QV, QVh = aggregate_gated(plan, K, Q, V)
        dK, dQ, dV = aggregate_gated_backward(plan, K, QV, QVh, g)
        return dict(Z=Z, dK=dK, dQ=dQ, dV=dV)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    with pytest.raises(RuntimeError, match="gated_walks"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(K, Q, V, g)
    assert plan.launch_count() == launches and plan._gated_walks is None
    ins = [tuple(t(a) for a in inputs(m, f, 20 + i)) for i in range(3)]

    def load(i):
        for dst, src in zip((K, Q, V, g), ins[i]):
            dst.copy_(src)

    plan.prepare(2 * f)
    step(*ins[0])                                         # the first eager call builds the walks
    check_one_rank_capture(plan, lambda: step(K, Q, V, g), load, lambda i: step(*ins[i]))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n = 64, A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    for p in plans:
        p.prepare(2 * f)
        p.gated_walks()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, f, 30 + i) for i in range(3)]

    def buffers(r):
        return {name: torch.zeros((lps[r].m, f), device=dev()) for name in ("x", "q", "v", "g")}

    def load(bufs, i):
        for r, lp in enumerate(lps):
            for name, a in zip(("x", "q", "v", "g"), ins[i]):
                bufs[r][name].copy_(t(a[lp.owned]))
        torch.cuda.synchronize()

    def step(r, b):
        Z, QV, QVh = aggregate_gated(plans[r], b["x"], b["q"], b["v"])
        dK, dQ, dV = aggregate_gated_backward(plans[r], b["x"], QV, QVh, b["g"])
        return dict(Z=Z, dK=dK, dQ=dQ, dV=dV)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGATED.py", [], 29691)
    assert_follows(lines, go.intended_training(karate(), 2, 4, 7))


def test_layer_on_three_ranks_follows_the_one_rank_curve():
    """gated.run's training loop with the three ranks of karate_k3 in this process (peer transport), against the same
    loop on one rank and against the fp64 oracle with gradients averaged over three ranks."""
    import torch.nn as nn
    import torch.nn.functional as F
    from pgcn_b200.gated import PGATED
    A, pv, k = problem("karate")
    n, f, L, epochs = A.shape[0], 4, 2, 50

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = nn.Sequential(*[PGATED(p, f, f) for _ in range(L)]).to(dev())
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
    one = [planmod.PgcnPlan(lp1[0], 2 * f, device=dev())]
    one[0].bind_values()
    curve1 = train(one, lp1)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    curve3 = train(plans, lps)
    np.testing.assert_allclose(curve1, go.intended_training(A, L, f, 7), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, go.intended_training(A, L, f, 7, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
    for p in plans + one:
        p.close()
