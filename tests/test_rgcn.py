"""R-GCN's relational aggregation on the H100 path: pgcn_rgcn_forward / pgcn_rgcn_backward, PgcnPlan.relation_walks,
op.PRGCN and PRGCN.py.

The fp32 bound is rgcn_oracle.terms': a first-order propagation of the kernels' roundings (the product when there is a
weight, every sum d roundings of its sum|terms|, the fp32 mean weight against 1 / c), doubled.

  * Z and dX against fp64 on gemat11, the hub graph (a split row of 3000 entries, empty rows, rows of one entry) and a
    local plan with duplicated entries, at widths 1 .. 256 and R in {1, 2, 3, 8}, for "add", "mean" and weighted "add";
    run-to-run bits; every operand 4 bytes into its buffer (the scalar instances) gives the vector instances' bits;
  * the same graph walked with a chunk of 4; +-0, +-inf and NaN in X and w where the formula has them; a plan with
    m R f > 2^31 checked on its last rows and columns;
  * exact identities: R = 1 "add" with X >= 0 is pgcn_gine_forward with E = 0 to the bit; relabelling the relations
    permutes Z's relation axis (and leaves dX) bit for bit; a relation that never occurs gives +0;
  * torch.profiler, in a process of its own, sees every instance of tests/rgcn_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport within the bound of the one-rank fp64 result; on two GPUs NCCL gives the
    peer transport's bits;
  * PRGCN's autograd in both layouts and on 3 ranks; CUDA-graph capture on one and two ranks, and a capture before the
    first eager call refused before it enqueues work;
  * PRGCN.py follows the fp64 loss curve, and the network on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import rgcn_oracle as ro
from harness import (ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PRGCN, aggregate_rgcn, aggregate_rgcn_backward, rgcn_weights
from pgcn_b200.rgcn import relation_hash
from test_gatedgcn import key
from test_gine import _eager, one_rank_plan, within

pytestmark = pytest.mark.gpu
WIDTHS = [1, 3, 4, 5, 31, 32, 127, 128, 129, 256]
RELATIONS = [1, 2, 3, 8]
MODES = [("add", False), ("mean", False), ("add", True)]


def inputs(m, ncols, nnz, R, f, seed):
    """X [ncols, f], gZ [m, R, f] and w [nnz], fp32."""
    rs = np.random.RandomState(seed)
    X = rs.standard_normal((ncols, f)).astype(np.float32)
    gZ = rs.standard_normal((m, R, f)).astype(np.float32)
    return X, gZ, rs.uniform(-2, 2, nnz).astype(np.float32)


def relations(lp, R, seed):
    return np.random.RandomState(seed).randint(0, R, lp.nnz())


def run_all(plan, walks, X, gZ, w, f, tr_perm=None):
    """{"Z": [m, R, f], "dX": [m + h, f]} from the two C calls (one rank, h = 0), outputs NaN-filled first."""
    lib, lp, R = cabi.load_rgcn(), plan.lp, walks.R
    perm_t = plan.transposed_entries() if tr_perm is None else tr_perm
    o = {"Z": torch.full((lp.m, R, f), float("nan"), device=dev()),
         "dX": torch.full((lp.m + lp.h, f), float("nan"), device=dev())}
    w1 = torch.empty((walks.fwd.nslots, f), device=dev())
    w2 = torch.empty((walks.tr.nslots, f), device=dev())
    p = lambda x: None if x is None else x.data_ptr()
    cabi.check_rgcn(lib.pgcn_rgcn_forward(C.byref(walks.fwd.c), p(walks.perm_f), lp.m, lp.h, R, p(X), None, p(w),
                                          p(o["Z"]), p(w1), f, stream()))
    cabi.check_rgcn(lib.pgcn_rgcn_backward(C.byref(walks.tr.c), p(perm_t), lp.m, lp.h, R, p(gZ), p(w), p(o["dX"]),
                                           p(w2), f, stream()))
    torch.cuda.synchronize()
    return o


def check_one_rank(plan, rel, R, ins, f, aggr, weighted, walks=None, shift=False):
    lp = plan.lp
    Xn, gn, wn = ins
    rt = torch.from_numpy(rel)
    walks = walks or plan.relation_walks(rt, R)
    w = torch.from_numpy(wn).to(dev()) if weighted else None
    kw = rgcn_weights(plan, walks, w, aggr)
    ops = [t(Xn), t(gn), kw]
    if shift:
        ops = [None if x is None else shifted(x) for x in ops]
    out = run_all(plan, walks, *ops, f)
    ref = ro.terms(lp.rowptr, lp.colidx, lp.m, rel, R, Xn, gn, wn if weighted else None, aggr)
    what = "f=%d R=%d %s%s" % (f, R, aggr, " weighted" if weighted else "")
    within(out["Z"], ref["Z"], "Z " + what)
    within(out["dX"], ref["dX"], "dX " + what)
    return out


@pytest.mark.parametrize("R", RELATIONS)
@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_and_run_to_run_and_scalar_bits(case, f, R):
    if case != "gemat11_k1" and f not in (3, 4, 5, 32, 129, 256):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
    rel = relations(lp, R, f + R)
    if case == "hub" and R == 1:
        assert plan.relation_walks(torch.from_numpy(rel), R).fwd.nslots > 0          # a split virtual row
    ins = inputs(lp.m, lp.m, lp.nnz(), R, f, f + 7 * R)
    for aggr, weighted in MODES:
        first = check_one_rank(plan, rel, R, ins, f, aggr, weighted)
        again = check_one_rank(plan, rel, R, ins, f, aggr, weighted)
        scalar = check_one_rank(plan, rel, R, ins, f, aggr, weighted, shift=True)
        for name in ("Z", "dX"):
            assert np.array_equal(bits(first[name]), bits(again[name])), name
            assert np.array_equal(bits(first[name]), bits(scalar[name])), name
    plan.close()


@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("f", [4, 5, 64])
def test_forced_small_chunk_stays_within_the_bound(f, R):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    rel = relations(lp, R, 2)
    walks = plan.relation_walks(torch.from_numpy(rel), R)
    rows = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
    vptr = np.concatenate([[0], np.cumsum(np.bincount(rows * R + rel, minlength=lp.m * R))])
    small = walks._replace(fwd=planmod.GatedWalk(vptr, walks.fwd.idx.cpu().numpy(), 4, dev()),
                           tr=planmod.GatedWalk(lp.t_rowptr, walks.tr.idx.cpu().numpy(), 4, dev()))
    assert small.fwd.nslots > 0 and small.tr.nslots > 0
    ins = inputs(lp.m, lp.m, lp.nnz(), R, f, 9)
    for aggr, weighted in MODES:
        check_one_rank(plan, rel, R, ins, f, aggr, weighted, walks=small)
    plan.close()


@pytest.mark.parametrize("f", [5, 8])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values(case, f):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    R = 3
    rel = relations(lp, R, f)
    Xn, gn, wn = inputs(lp.m, lp.m, lp.nnz(), R, f, 3 * f)
    rs = np.random.RandomState(f)
    for x in (Xn, wn):
        u = rs.uniform(size=x.shape)
        x[u < 0.005] = np.inf
        x[(u >= 0.005) & (u < 0.01)] = -np.inf
        x[(u >= 0.01) & (u < 0.0125)] = np.nan
        x[(u >= 0.0125) & (u < 0.05)] = 0.0
        x[(u >= 0.05) & (u < 0.09)] = -0.0
    walks = plan.relation_walks(torch.from_numpy(rel), R)
    for aggr, weighted in MODES:
        kw = rgcn_weights(plan, walks, t(wn) if weighted else None, aggr)
        out = run_all(plan, walks, t(Xn), t(gn), kw, f)
        ref = ro.fp32_reference(lp.rowptr, lp.colidx, lp.m, rel, R, Xn, gn, wn if weighted else None, aggr)
        for name in ("Z", "dX"):
            g, w = out[name].cpu().numpy(), ref[name]
            assert np.isnan(g).any() or (name == "dX" and not weighted), name     # gZ is finite
            assert np.array_equal(np.isnan(g), np.isnan(w)), (aggr, weighted, name)
            assert np.array_equal(np.isposinf(g), np.isposinf(w)), (aggr, weighted, name)
            assert np.array_equal(np.isneginf(g), np.isneginf(w)), (aggr, weighted, name)
        # sums start at +0: a (row, relation) pair whose terms are all -0 gives +0
        Z = out["Z"].cpu().numpy()
        assert not np.signbit(Z[Z == 0]).any()
    plan.close()


def test_virtual_row_offsets_beyond_2_31():
    """m R f > 2^31 (m = 20000, R = 256, f = 512): the last rows' Z and the last columns' dX within the bound, from
    fp64 over the last rows' entries."""
    import scipy.sparse as sp
    m, band, R, f = 20000, 8, 256, 512
    assert m * R * f > 2 ** 31
    rows = np.repeat(np.arange(m), band)
    cols = (rows + np.tile(np.arange(band), m)) % m
    A = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(m, m))
    lp = planmod.build_local_plan(A, np.zeros(m, dtype=np.int64), 0, 1)
    plan = planmod.PgcnPlan(lp, f, device=dev())
    plan.bind_values()
    rel = np.random.RandomState(3).randint(0, R, lp.nnz())
    rel[-band:] = R - 1                                                # the last virtual row is not empty
    walks = plan.relation_walks(torch.from_numpy(rel), R)
    g = torch.Generator(device=dev()).manual_seed(5)
    X = torch.randn((m, f), device=dev(), generator=g)
    gZ = torch.randn((m, R, f), device=dev(), generator=g)
    w = rgcn_weights(plan, walks, None, "mean")
    Z, _ = aggregate_rgcn(plan, walks, X, w)
    dX = aggregate_rgcn_backward(plan, walks, gZ, w)
    torch.cuda.synchronize()
    last = 100
    e0 = int(lp.rowptr[m - last])
    sub_ptr = lp.rowptr[m - last:].astype(np.int64) - e0
    cpu = lambda x: x.cpu().numpy()
    ref = ro.terms(sub_ptr, lp.colidx[e0:], m, rel[e0:], R, cpu(X), cpu(gZ[m - last:]), None, "mean")
    within(Z[m - last:], ref["Z"], "m R f > 2^31: Z")
    done = slice(m - last + band, m)                                # every entry of these columns is in the last rows
    val, tol = ref["dX"]
    within(dX[done], (val[done], tol[done]), "m R f > 2^31: dX")
    assert float(Z[-1, R - 1].abs().sum()) > 0
    plan.close()


# ---- exact identities ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("f", [4, 5, 129])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_one_relation_sum_is_gine_with_zero_edges(case, f):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    X = t(np.abs(inputs(lp.m, lp.m, 1, 1, f, f)[0]))
    X[::7] = 0.0
    walks = plan.relation_walks(torch.zeros(lp.nnz(), dtype=torch.int64), 1)
    Z = run_all(plan, walks, X, torch.zeros((lp.m, 1, f), device=dev()), None, f)["Z"]
    fwd, _ = plan.gated_walks()
    Zg = torch.full((lp.m, f), float("nan"), device=dev())
    E = torch.zeros((lp.nnz(), f), device=dev())
    work = torch.empty((fwd.nslots, f), device=dev())
    cabi.check_gine(cabi.load_gine().pgcn_gine_forward(C.byref(fwd.c), lp.m, 0, X.data_ptr(), None, E.data_ptr(),
                                                       Zg.data_ptr(), work.data_ptr(), f, stream()))
    torch.cuda.synchronize()
    assert np.array_equal(bits(Z[:, 0]), bits(Zg))
    plan.close()


@pytest.mark.parametrize("aggr,weighted", MODES)
def test_relabelling_permutes_the_relation_axis_and_an_absent_relation_is_zero(aggr, weighted):
    f, R = 32, 5
    plan = one_rank_plan("hub", f)
    lp = plan.lp
    rel = relations(lp, R - 1, 4)                                    # relation R - 1 never occurs
    pi = np.array([3, 0, 4, 1, 2])
    Xn, gn, wn = inputs(lp.m, lp.m, lp.nnz(), R, f, 11)
    w = t(wn) if weighted else None
    a = plan.relation_walks(torch.from_numpy(rel), R)
    b = plan.relation_walks(torch.from_numpy(pi[rel]), R)
    gperm = np.empty_like(gn)
    gperm[:, pi] = gn
    out_a = run_all(plan, a, t(Xn), t(gn), rgcn_weights(plan, a, w, aggr), f)
    out_b = run_all(plan, b, t(Xn), t(gperm), rgcn_weights(plan, b, w, aggr), f)
    za, zb = bits(out_a["Z"]), bits(out_b["Z"])
    assert np.array_equal(zb[:, pi], za)
    assert np.array_equal(bits(out_a["dX"]), bits(out_b["dX"]))
    assert not za[:, R - 1].any() and not zb[:, pi[R - 1]].any()     # exact +0
    plan.close()


def _instances_worker(rank, k):
    """The keys of the relational kernels torch.profiler sees while every instance runs (vector and scalar, with and
    without weights, split rows through the fixup), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    R = 2
    for f, shift in ((8, False), (5, False), (8, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        rel = relations(lp, R, 1)
        walks = plan.relation_walks(torch.from_numpy(rel), R)
        rows = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
        vptr = np.concatenate([[0], np.cumsum(np.bincount(rows * R + rel, minlength=lp.m * R))])
        small = walks._replace(fwd=planmod.GatedWalk(vptr, walks.fwd.idx.cpu().numpy(), 64, dev()),
                               tr=planmod.GatedWalk(lp.t_rowptr, walks.tr.idx.cpu().numpy(), 64, dev()))
        assert small.fwd.c.nsplits > 0 and small.tr.c.nsplits > 0
        ins = inputs(lp.m, lp.m, lp.nnz(), R, f, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for aggr, weighted in (("add", False), ("mean", False)):
                    check_one_rank(plan, rel, R, ins, f, aggr, weighted, walks=small, shift=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "rgcn_" in e.name}
            if len(names) == 3:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    with open(os.path.join(ROOT, "tests", "rgcn_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


# ---- several ranks ---------------------------------------------------------------------------------------------------

def _synthetic(plan, R):
    return relation_hash(plan.edge_pairs(), R)


# f a multiple of 4, the widths the peer transport's halo exchange takes; f = 132 takes two passes of 128 features
@pytest.mark.parametrize("case,f,R", [("gemat11_k2", 64, 3), ("gemat11_k2", 8, 8), ("gemat11_k3_hp", 16, 2),
                                      ("gemat11_k3_hp", 132, 4)])
def test_multi_rank_within_the_bound_of_one_rank(case, f, R):
    A, pv, k = problem(case)
    n = A.shape[0]
    one = one_rank_plan(case, f)
    lp1 = one.lp
    rel1 = _synthetic(one, R).cpu().numpy()
    Xn, gn, _ = inputs(n, n, 1, R, f, f + k)
    ref = {aggr: ro.terms(lp1.rowptr, lp1.colidx, n, rel1, R, Xn, gn, None, aggr) for aggr in ("add", "mean")}
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rels = [_synthetic(p, R) for p in plans]
    ins = [(t(Xn[lp.owned]), t(gn[lp.owned])) for lp in lps]

    def step(r, aggr):
        X, g = ins[r]
        walks = plans[r].relation_walks(rels[r], R)
        w = rgcn_weights(plans[r], walks, None, aggr)
        Z, _ = aggregate_rgcn(plans[r], walks, X, w)
        return Z, aggregate_rgcn_backward(plans[r], walks, g, w)

    for aggr in ("add", "mean"):
        first = None
        for rep in range(2):                              # both epoch parities of the peer slabs
            out = run_ranks(plans, lambda r: step(r, aggr), streams)
            for r, lp in enumerate(lps):
                Z, dX = out[r]
                (zv, zt), (xv, xt) = ref[aggr]["Z"], ref[aggr]["dX"]
                within(Z, (zv[lp.owned], zt[lp.owned]), "%s %s Z rank %d rep %d" % (case, aggr, r, rep))
                within(dX, (xv[lp.owned], xt[lp.owned]), "%s %s dX rank %d rep %d" % (case, aggr, r, rep))
            if first is None:
                first = [[bits(x) for x in o] for o in out]
            else:
                assert all(np.array_equal(a, bits(b)) for fo, o in zip(first, out) for a, b in zip(fo, o))
    for p in plans + [one]:
        p.close()


def _nccl_worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    A, pv, _ = problem("gemat11_k2")
    n, f, R = A.shape[0], 64, 3
    p = planmod.build_plan(A, pv, rank, k, f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    Xn, gn, _ = inputs(n, n, 1, R, f, 1)
    X, g = torch.from_numpy(Xn[own]).cuda().requires_grad_(True), torch.from_numpy(gn[own]).cuda()
    Z = PRGCN.apply(p, X, _synthetic(p, R), R)
    (Z * g).sum().backward()
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), X.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29893, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29894, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        for x, y in zip(a[r][1], b[r][1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("layout", ["local", "global"])
def test_autograd_one_rank(layout):
    f, R = 32, 3
    plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp = plan.lp
    rel = relations(lp, R, 4)
    Xn, gn, wn = inputs(lp.m, lp.m, lp.nnz(), R, f, 4)
    rt = torch.from_numpy(rel)
    for aggr, weighted in MODES:
        w = t(wn) if weighted else None
        X = t(Xn).requires_grad_(True)
        Z = PRGCN.apply(plan, X, rt, R, w, aggr)
        assert tuple(Z.shape) == (lp.m, R, f)
        (Z * t(gn)).sum().backward()
        ref = ro.terms(lp.rowptr, lp.colidx, lp.m, rel, R, Xn, gn, wn if weighted else None, aggr)
        within(Z, ref["Z"], "%s %s Z" % (layout, aggr))
        within(X.grad, ref["dX"], "%s %s dX" % (layout, aggr))
        walks = plan.relation_walks(rt, R)
        out = run_all(plan, walks, t(Xn), t(gn), rgcn_weights(plan, walks, w, aggr), f)
        assert np.array_equal(bits(Z), bits(out["Z"])) and np.array_equal(bits(X.grad), bits(out["dX"]))
    # a weight that asks for a gradient is refused
    with pytest.raises(ValueError, match="no gradient for its edge weights"):
        PRGCN.apply(plan, t(Xn), rt, R, t(wn).requires_grad_(True), "add")
    plan.close()


def _autograd_three_ranks_worker(rank, k):
    """PRGCN through autograd on the three ranks of gemat11_k3_hp in this process, in both layouts: per layout and
    rank (Z, dX) as numpy, and the owned rows."""
    A, pv, k = problem("gemat11_k3_hp")
    n, f, R = A.shape[0], 16, 3
    _, gn0, _ = inputs(n, n, 1, R, f, 3)
    Xn = inputs(n, n, 1, R, f, 3)[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rels = [_synthetic(p, R) for p in plans]
    res = {}
    for layout in ("local", "global"):
        for p in plans:
            p.layout = layout
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank).reshape((-1,) + (1,) * (a.ndim - 1)), a, np.float32(7.0)))   # non-owned rows ignored
        leaves = [t(pick(Xn, lp)).requires_grad_(True) for lp in lps]
        out = run_ranks(plans, lambda r: PRGCN.apply(plans[r], leaves[r], rels[r], R), streams)
        run_ranks(plans, lambda r: (out[r] * t(pick(gn0, lps[r]))).sum().backward(), streams)
        res[layout] = [tuple(x.detach().cpu().numpy() for x in (out[r], leaves[r].grad)) for r in range(k)]
    for p in plans:
        p.close()
    return res, [lp.owned for lp in lps]


def test_autograd_three_ranks_and_global_layout():
    A, pv, k = problem("gemat11_k3_hp")
    n, f, R = A.shape[0], 16, 3
    one = one_rank_plan("gemat11_k3_hp", f)
    lp1 = one.lp
    rel1 = _synthetic(one, R).cpu().numpy()
    one.close()
    Xn, gn, _ = inputs(n, n, 1, R, f, 3)
    ref = ro.terms(lp1.rowptr, lp1.colidx, n, rel1, R, Xn, gn, None, "mean")
    res, owned = _eager(_autograd_three_ranks_worker)
    for layout, per_rank in res.items():
        for r, (Z, dX) in enumerate(per_rank):
            for name, got in (("Z", Z), ("dX", dX)):
                val, tol = ref[name]
                if layout == "global":
                    mask = (pv == r).reshape((-1,) + (1,) * (val.ndim - 1))
                    val, tol = np.where(mask, val, 0.0), np.where(mask, tol, 0.0)
                else:
                    val, tol = val[owned[r]], tol[owned[r]]
                within(torch.from_numpy(got), (val, tol), "%s %s rank %d" % (layout, name, r))


def test_one_rank_capture_and_refusal_before_the_first_eager_call():
    f, R = 64, 4
    plan = one_rank_plan("hub", f)
    m = plan.lp.m
    rel = torch.from_numpy(relations(plan.lp, R, 5))
    X, g = torch.zeros((m, f), device=dev()), torch.zeros((m, R, f), device=dev())

    def step(X, g):
        walks = plan.relation_walks(rel, R)
        w = rgcn_weights(plan, walks, None, "mean")
        Z, _ = aggregate_rgcn(plan, walks, X, w)
        return dict(Z=Z, dX=aggregate_rgcn_backward(plan, walks, g, w))

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    with pytest.raises(RuntimeError, match="relation_walks"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(X, g)
    assert plan.launch_count() == launches and plan._relation_walks == {}
    ins = []
    for i in range(3):
        Xn, gn, _ = inputs(m, m, 1, R, f, 20 + i)
        ins.append((t(Xn), t(gn)))

    def load(i):
        for dst, src in zip((X, g), ins[i]):
            dst.copy_(src)

    plan.prepare(f)
    step(*ins[0])                                         # the first eager call builds the tables
    check_one_rank_capture(plan, lambda: step(X, g), load, lambda i: step(*ins[i]))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n, R = 64, A.shape[0], 3
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    rels = [_synthetic(p, R) for p in plans]
    for p, rel in zip(plans, rels):
        p.prepare(f)
        p.relation_walks(rel, R)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, n, 1, R, f, 30 + i) for i in range(3)]

    def buffers(r):
        return {"x": torch.zeros((lps[r].m, f), device=dev()), "g": torch.zeros((lps[r].m, R, f), device=dev())}

    def load(bufs, i):
        Xn, gn, _ = ins[i]
        for r, lp in enumerate(lps):
            bufs[r]["x"].copy_(t(Xn[lp.owned]))
            bufs[r]["g"].copy_(t(gn[lp.owned]))
        torch.cuda.synchronize()

    def step(r, b):
        walks = plans[r].relation_walks(rels[r], R)
        w = rgcn_weights(plans[r], walks, None, "mean")
        Z, _ = aggregate_rgcn(plans[r], walks, b["x"], w)
        return dict(Z=Z, dX=aggregate_rgcn_backward(plans[r], walks, b["g"], w))

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


@pytest.mark.parametrize("bases", [None, 2])
def test_cli_follows_the_fp64_loss_curve(tmp_path, bases):
    extra = ["--relations", "3"] + ([] if bases is None else ["--bases", str(bases)])
    lines = run_cli(tmp_path, "PRGCN.py", extra, 29697 if bases is None else 29698)
    assert_follows(lines, ro.intended_training(karate(), 2, 4, 3, 7, bases))


def _three_rank_worker(rank, k):
    """(curve1, curve3): rgcn's network trained by rgcn.run's loop on one rank, then on the three ranks of karate_k3
    in this process (peer transport), gradients averaged over the ranks."""
    import torch.nn.functional as F
    from pgcn_b200.rgcn import PRGCN as Network
    A, pv, k = problem("karate")
    n, f, L, R, epochs = A.shape[0], 4, 2, 3, 50

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = Network(p, f, L, R).to(dev())
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
    for p in plans + one:
        p.close()
    return curve1, curve3


def test_network_on_three_ranks_follows_the_one_rank_curve():
    """rgcn.run's training loop with the three ranks of karate_k3 in one process, against the same loop on one rank
    and against the fp64 oracle with gradients averaged over three ranks."""
    A, _, _ = problem("karate")
    curve1, curve3 = _eager(_three_rank_worker)
    np.testing.assert_allclose(curve1, ro.intended_training(A, 2, 4, 3, 7), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, ro.intended_training(A, 2, 4, 3, 7, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
