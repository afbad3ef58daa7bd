"""GINE on the H100 path: pgcn_gine_forward / pgcn_gine_backward, op.PGINE and PGINE.py.

The fp32 bound is gine_oracle.terms': a first-order propagation of the kernels' roundings (the add before the ReLU,
every sum d roundings of its sum|terms|), doubled. dE has no bound: it is gZ[i] or 0, and must be torch's bits.

  * Z and dX against fp64 on gemat11, the hub graph (a split row of 3000 entries, empty rows, rows of one entry) and a
    local plan with duplicated entries, at widths 1 .. 256; dE bit-equal to torch's relu backward of
    X[cols] + E; a NULL dE leaves dX's bits; run-to-run bits; every operand 4 bytes into its buffer (the scalar
    instances) gives the vector instances' bits;
  * the same graph walked with a chunk of 4; +-0, +-inf and NaN in X and E where torch has them; a plan with
    nnz * f > 2^31 checked on its last entries, rows and columns;
  * torch.profiler, in a process of its own, sees every instance of tests/gine_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport within the bound of the one-rank fp64 result, dE bit-equal to one rank's
    through edge_pairs(); on two GPUs NCCL gives the peer transport's bits;
  * PGINE's autograd in both layouts and on 3 ranks; CUDA-graph capture on one and two ranks, and a capture before the
    first eager call refused before it enqueues work;
  * PGINE.py follows the fp64 loss curve, and the network on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gine_oracle as gio
from harness import (ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PGINE, aggregate_gine, aggregate_gine_backward
from test_gatedgcn import edge_rows, key
from test_max_aggregation import with_duplicates

pytestmark = pytest.mark.gpu
WIDTHS = [1, 3, 4, 5, 6, 31, 32, 64, 127, 128, 129, 256]


def one_rank_plan(case, f):
    """A bound one-rank plan of width f on problem(case) ("dup": gemat11 with duplicated entries)."""
    A, _, _ = problem("gemat11_k1" if case == "dup" else case)
    lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    if case == "dup":
        lp = with_duplicates(lp)
    plan = planmod.PgcnPlan(lp, f, device=dev())
    plan.bind_values()
    return plan


def inputs(n, nnz, f, seed):
    """X, gZ ([n, f]) and E ([nnz, f]), fp32; X and E of one scale, so that about half the messages are cut."""
    rs = np.random.RandomState(seed)
    X, gZ = (rs.standard_normal((n, f)).astype(np.float32) for _ in range(2))
    return X, gZ, rs.standard_normal((nnz, f)).astype(np.float32)


def within(got, ref, what):
    val, tol = ref
    g = got.detach().cpu().numpy().astype(np.float64)
    err = np.abs(g - val)
    bad = ~(err <= tol + 1e-30)
    assert not bad.any(), "%s: %d elements beyond the fp32 bound, worst err %.3e" % (what, int(bad.sum()),
                                                                                      float(np.nanmax(err)))


def torch_dE(lp, X, E, gZ):
    """torch's gradient of E through relu(X[cols] + E) for the output gradient gZ[rows] (X, E, gZ device tensors)."""
    r = torch.from_numpy(np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))).to(dev())
    c = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev())
    e = E.detach().clone().requires_grad_(True)
    torch.relu(X[c] + e).backward(gZ[r])
    return e.grad


def run_all(plan, X, E, gZ, f, walks=None, with_dE=True):
    """{name: tensor} from the two C calls (one rank, h = 0), outputs NaN-filled first."""
    fwd, tr = walks or plan.gated_walks()
    perm = plan.transposed_entries()
    lib, lp = cabi.load_gine(), plan.lp
    nan = lambda *s: torch.full(s, float("nan"), device=dev())
    o = {"Z": nan(lp.m, f), "dE": nan(lp.nnz(), f) if with_dE else None, "dX": nan(lp.m + lp.h, f)}
    w1 = torch.empty((fwd.nslots, f), device=dev())
    w2 = torch.empty((tr.nslots, f), device=dev())
    p = lambda x: None if x is None else x.data_ptr()
    cabi.check_gine(lib.pgcn_gine_forward(C.byref(fwd.c), lp.m, lp.h, p(X), None, p(E), p(o["Z"]), p(w1), f,
                                          stream()))
    cabi.check_gine(lib.pgcn_gine_backward(C.byref(tr.c), p(perm), lp.m, lp.h, p(X), None, p(E), p(gZ), p(o["dE"]),
                                           p(o["dX"]), p(w2), f, stream()))
    torch.cuda.synchronize()
    return o


def check_one_rank(plan, ins, f, walks=None, shift=False, with_dE=True):
    lp = plan.lp
    Xn, gn, En = ins
    ops = [t(Xn), t(En), t(gn)]
    if shift:
        ops = [shifted(x) for x in ops]
    out = run_all(plan, *ops, f, walks, with_dE)
    ref = gio.terms(lp.rowptr, lp.colidx, lp.m, Xn, En, gn)
    within(out["Z"], ref["Z"], "Z f=%d" % f)
    within(out["dX"], ref["dX"], "dX f=%d" % f)
    if with_dE:
        assert np.array_equal(bits(out["dE"]), bits(torch_dE(lp, *ops[:2], ops[2]))), "dE f=%d" % f
    return out


@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_dE_bits_and_run_to_run(case, f):
    if case != "gemat11_k1" and f not in (3, 4, 5, 32, 129, 256):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
        assert plan.gated_walks()[0].nslots > 0
    ins = inputs(lp.m, lp.nnz(), f, f + len(case))
    first = check_one_rank(plan, ins, f)
    again = check_one_rank(plan, ins, f)
    scalar = check_one_rank(plan, ins, f, shift=True)
    no_dE = check_one_rank(plan, ins, f, with_dE=False)
    for name in ("Z", "dE", "dX"):
        assert np.array_equal(bits(first[name]), bits(again[name])), name
        assert np.array_equal(bits(first[name]), bits(scalar[name])), name
    assert np.array_equal(bits(first["dX"]), bits(no_dE["dX"]))          # a NULL dE leaves dX's bits
    assert np.array_equal(bits(first["Z"]), bits(no_dE["Z"]))
    plan.close()


@pytest.mark.parametrize("f", [4, 5, 64])
def test_forced_small_chunk_stays_within_the_bound(f):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    assert plan.gated_walks()[0].nslots == plan.gated_walks()[1].nslots == 0
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    ins = inputs(lp.m, lp.nnz(), f, 9)
    whole = check_one_rank(plan, ins, f)
    split = check_one_rank(plan, ins, f, walks=small)
    assert np.array_equal(bits(whole["dE"]), bits(split["dE"]))          # dE does not depend on the chunking
    plan.close()


@pytest.mark.parametrize("f", [5, 8])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values(case, f):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    Xn, gn, En = inputs(lp.m, lp.nnz(), f, 3 * f)
    rs = np.random.RandomState(f)
    for x in (Xn, En):
        u = rs.uniform(size=x.shape)
        x[u < 0.005] = np.inf
        x[(u >= 0.005) & (u < 0.01)] = -np.inf
        x[(u >= 0.01) & (u < 0.0125)] = np.nan
        x[(u >= 0.0125) & (u < 0.05)] = 0.0
        x[(u >= 0.05) & (u < 0.09)] = -0.0
    X, E, gZ = t(Xn), t(En), t(gn)
    out = run_all(plan, X, E, gZ, f)
    r = torch.from_numpy(np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))).to(dev())
    c = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev())
    Zt = torch.zeros((lp.m, f), device=dev()).index_add_(0, r, torch.relu(X[c] + E))
    dXt = torch.zeros((lp.m, f), device=dev()).index_add_(0, c, torch_dE(lp, X, E, gZ))
    assert np.array_equal(bits(out["dE"]), bits(torch_dE(lp, X, E, gZ)))
    for name, w in (("Z", Zt), ("dX", dXt)):
        g, w = out[name].cpu().numpy(), w.cpu().numpy()
        assert np.isnan(g).any() or name == "dX", name
        assert np.array_equal(np.isnan(g), np.isnan(w)), name
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    ref = gio.fp32_reference(lp.rowptr, lp.colidx, lp.m, Xn, En, gn)
    assert np.array_equal(np.isnan(out["Z"].cpu().numpy()), np.isnan(ref["Z"]))
    plan.close()


def test_entry_offsets_beyond_2_31():
    """A banded graph with nnz * f > 2^31 (f = 256): the last entries' dE bits, and the last rows' Z and the last
    columns' dX within the bound, from fp64 over the last rows' entries."""
    import scipy.sparse as sp
    m, band, f = 40000, 216, 256
    rows = np.repeat(np.arange(m), band)
    cols = (rows + np.tile(np.arange(band), m)) % m
    A = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(m, m))
    lp = planmod.build_local_plan(A, np.zeros(m, dtype=np.int64), 0, 1)
    nnz = lp.nnz()
    assert nnz * f > 2 ** 31
    plan = planmod.PgcnPlan(lp, f, device=dev())
    plan.bind_values()
    g = torch.Generator(device=dev()).manual_seed(5)
    X, gZ = (torch.randn((m, f), device=dev(), generator=g) for _ in range(2))
    E = torch.randn((nnz, f), device=dev(), generator=g)
    Z, X_halo = aggregate_gine(plan, X, E)
    dX, dE = aggregate_gine_backward(plan, X, X_halo, E, gZ)
    torch.cuda.synchronize()
    last = 400                                                      # rows m - 400 .. m - 1
    e0 = int(lp.rowptr[m - last])
    sub_ptr = lp.rowptr[m - last:].astype(np.int64) - e0
    sub_col = lp.colidx[e0:]
    cpu = lambda x: x.cpu().numpy()
    ref = gio.terms(sub_ptr, sub_col, m, cpu(X), cpu(E[e0:]), cpu(gZ[m - last:]))
    r = torch.from_numpy(np.repeat(np.arange(m - last, m), np.diff(sub_ptr))).to(dev())
    c = torch.from_numpy(sub_col.astype(np.int64)).to(dev())
    e = E[e0:].clone().requires_grad_(True)
    torch.relu(X[c] + e).backward(gZ[r])
    assert np.array_equal(bits(dE[e0:]), bits(e.grad))
    within(Z[m - last:], ref["Z"], "nnz*f > 2^31: Z")
    cols_done = slice(m - 100, m)                                   # every entry of these columns is in the last rows
    val, tol = ref["dX"]
    within(dX[cols_done], (val[cols_done], tol[cols_done]), "nnz*f > 2^31: dX")
    plan.close()


def _instances_worker(rank, k):
    """The keys of the GINE kernels torch.profiler sees while every instance runs (vector and scalar, split rows
    through the fixup), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for f, shift in ((8, False), (5, False), (8, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        walks = (planmod.GatedWalk(lp.rowptr, lp.colidx, 64, dev()),
                 planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 64, dev()))
        assert walks[0].c.nsplits > 0 and walks[1].c.nsplits > 0
        ins = inputs(lp.m, lp.nnz(), f, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                check_one_rank(plan, ins, f, walks=walks, shift=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "gine_" in e.name}
            if len(names) == 4:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    with open(os.path.join(ROOT, "tests", "gine_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


# ---- several ranks ---------------------------------------------------------------------------------------------------

# f a multiple of 4, the widths the peer transport's halo exchange takes; f = 132 takes two passes of 128 features
@pytest.mark.parametrize("case,f", [("gemat11_k2", 64), ("gemat11_k2", 8), ("gemat11_k3_hp", 16),
                                    ("gemat11_k3_hp", 132)])
def test_multi_rank_within_the_bound_of_one_rank(case, f):
    A, pv, k = problem(case)
    n = A.shape[0]
    one = one_rank_plan(case, f)
    lp1 = one.lp
    Xn, gn, En = inputs(n, lp1.nnz(), f, f + k)
    ref = gio.terms(lp1.rowptr, lp1.colidx, n, Xn, En, gn)
    X1, E1, g1 = t(Xn), t(En), t(gn)
    Z1, H1 = aggregate_gine(one, X1, E1)
    _, dE1 = aggregate_gine_backward(one, X1, H1, E1, g1)
    dE1 = bits(dE1)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    pos = []
    for p, lp in zip(plans, lps):
        pos.append(edge_rows(lp1, lp))
        assert np.array_equal(p.edge_pairs().cpu().numpy().astype(np.int64),
                              one.edge_pairs().cpu().numpy().astype(np.int64)[pos[-1]])
    ins = [(t(Xn[lp.owned]), t(En[q]), t(gn[lp.owned])) for lp, q in zip(lps, pos)]

    def step(r):
        X, E, g = ins[r]
        Z, X_halo = aggregate_gine(plans[r], X, E)
        return (Z,) + aggregate_gine_backward(plans[r], X, X_halo, E, g)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            Z, dX, dE = out[r]
            within(Z, (ref["Z"][0][lp.owned], ref["Z"][1][lp.owned]), "%s Z rank %d rep %d" % (case, r, rep))
            within(dX, (ref["dX"][0][lp.owned], ref["dX"][1][lp.owned]), "%s dX rank %d rep %d" % (case, r, rep))
            assert np.array_equal(bits(dE), dE1[pos[r]]), "%s dE rank %d rep %d" % (case, r, rep)
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
    n, f = A.shape[0], 64
    p = planmod.build_plan(A, pv, rank, k, f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    Xn, gn, _ = inputs(n, 1, f, 1)
    E = torch.randn((p.lp.nnz(), f), generator=torch.Generator().manual_seed(rank)).cuda().requires_grad_(True)
    X, g = torch.from_numpy(Xn[own]).cuda().requires_grad_(True), torch.from_numpy(gn[own]).cuda()
    Z = PGINE.apply(p, X, E)
    (Z * g).sum().backward()
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), X.grad, E.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29891, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29892, "p2p"))
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
    Xn, gn, En = inputs(lp.m, lp.nnz(), f, 4)
    X, E = t(Xn).requires_grad_(True), t(En).requires_grad_(True)
    Z = PGINE.apply(plan, X, E)
    (Z * t(gn)).sum().backward()
    ref = gio.terms(lp.rowptr, lp.colidx, lp.m, Xn, En, gn)
    within(Z, ref["Z"], layout + " Z")
    within(X.grad, ref["dX"], layout + " dX")
    out = run_all(plan, t(Xn), t(En), t(gn), f)
    assert np.array_equal(bits(E.grad), bits(out["dE"])) and np.array_equal(bits(X.grad), bits(out["dX"]))
    # E without a gradient: dE reaches the kernel as NULL, and dX keeps its bits
    X2 = t(Xn).requires_grad_(True)
    PGINE.apply(plan, X2, t(En)).backward(t(gn))
    assert np.array_equal(bits(X2.grad), bits(out["dX"]))
    plan.close()


def _autograd_three_ranks_worker(rank, k):
    """PGINE through autograd on the three ranks of gemat11_k3_hp in this process, in both layouts: per layout and
    rank (Z, dX, dE) as numpy, with the one-rank dE bits and the entry map."""
    A, pv, k = problem("gemat11_k3_hp")
    n, f = A.shape[0], 16
    one = one_rank_plan("gemat11_k3_hp", f)
    lp1 = one.lp
    Xn, gn, En = inputs(n, lp1.nnz(), f, 3)
    X1, E1 = t(Xn), t(En)
    Z1, H1 = aggregate_gine(one, X1, E1)
    dE1 = bits(aggregate_gine_backward(one, X1, H1, E1, t(gn))[1])
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    pos = [edge_rows(lp1, lp) for lp in lps]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    res = {}
    for layout in ("local", "global"):
        for p in plans:
            p.layout = layout
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [(t(pick(Xn, lp)).requires_grad_(True), t(En[q]).requires_grad_(True)) for lp, q in zip(lps, pos)]
        out = run_ranks(plans, lambda r: PGINE.apply(plans[r], *leaves[r]), streams)
        run_ranks(plans, lambda r: (out[r] * t(pick(gn, lps[r]))).sum().backward(), streams)
        res[layout] = [tuple(x.detach().cpu().numpy() for x in (out[r], leaves[r][0].grad, leaves[r][1].grad))
                       for r in range(k)]
    for p in plans + [one]:
        p.close()
    return res, dE1, pos, [lp.owned for lp in lps]


def _eager(worker, *args):
    """spawn_ranks(worker, 1) with CUDA_MODULE_LOADING=EAGER: with lazy loading, the first launch of a kernel (torch's
    as well as this library's) waits for the device, where an earlier rank's exchange waits for this rank's half,
    which the blocked thread never enqueues. Ranks in separate processes, as in a real job, do not share that wait."""
    old = os.environ.get("CUDA_MODULE_LOADING")
    os.environ["CUDA_MODULE_LOADING"] = "EAGER"
    try:
        return spawn_ranks(worker, 1, args)[0]
    finally:
        if old is None:
            del os.environ["CUDA_MODULE_LOADING"]
        else:
            os.environ["CUDA_MODULE_LOADING"] = old


def test_autograd_three_ranks_and_global_layout():
    A, pv, k = problem("gemat11_k3_hp")
    n, f = A.shape[0], 16
    lp1 = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    Xn, gn, En = inputs(n, lp1.nnz(), f, 3)
    ref = gio.terms(lp1.rowptr, lp1.colidx, n, Xn, En, gn)
    res, dE1, pos, owned = _eager(_autograd_three_ranks_worker)
    for layout, per_rank in res.items():
        for r, (Z, dX, dE) in enumerate(per_rank):
            for name, got in (("Z", Z), ("dX", dX)):
                val, tol = ref[name]
                if layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                else:
                    val, tol = val[owned[r]], tol[owned[r]]
                within(torch.from_numpy(got), (val, tol), "%s %s rank %d" % (layout, name, r))
            assert np.array_equal(dE.view(np.uint32), dE1[pos[r]]), "%s dE rank %d" % (layout, r)


def test_one_rank_capture_and_refusal_before_the_first_eager_call():
    f = 64
    plan = one_rank_plan("hub", f)
    m, nnz = plan.lp.m, plan.lp.nnz()
    X, g = torch.zeros((m, f), device=dev()), torch.zeros((m, f), device=dev())
    E = torch.zeros((nnz, f), device=dev())

    def step(X, E, g):
        Z, X_halo = aggregate_gine(plan, X, E)
        dX, dE = aggregate_gine_backward(plan, X, X_halo, E, g)
        return dict(Z=Z, dX=dX, dE=dE)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    with pytest.raises(RuntimeError, match="gated_walks"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(X, E, g)
    assert plan.launch_count() == launches and plan._gated_walks is None and plan._transposed_entries is None
    plan.gated_walks()
    with pytest.raises(RuntimeError, match="transposed_entries"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(X, E, g)
    assert plan.launch_count() == launches and plan._transposed_entries is None
    ins = []
    for i in range(3):
        Xn, gn, En = inputs(m, nnz, f, 20 + i)
        ins.append((t(Xn), t(En), t(gn)))

    def load(i):
        for dst, src in zip((X, E, g), ins[i]):
            dst.copy_(src)

    plan.prepare(f)
    step(*ins[0])                                         # the first eager call builds the tables
    check_one_rank_capture(plan, lambda: step(X, E, g), load, lambda i: step(*ins[i]))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n = 64, A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
        p.gated_walks()
        p.transposed_entries()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, max(lp.nnz() for lp in lps), f, 30 + i) for i in range(3)]

    def buffers(r):
        return {"x": torch.zeros((lps[r].m, f), device=dev()), "g": torch.zeros((lps[r].m, f), device=dev()),
                "e": torch.zeros((lps[r].nnz(), f), device=dev())}

    def load(bufs, i):
        Xn, gn, En = ins[i]
        for r, lp in enumerate(lps):
            bufs[r]["x"].copy_(t(Xn[lp.owned]))
            bufs[r]["g"].copy_(t(gn[lp.owned]))
            bufs[r]["e"].copy_(t(En[:lp.nnz()]))
        torch.cuda.synchronize()

    def step(r, b):
        Z, X_halo = aggregate_gine(plans[r], b["x"], b["e"])
        dX, dE = aggregate_gine_backward(plans[r], b["x"], X_halo, b["e"], b["g"])
        return dict(Z=Z, dX=dX, dE=dE)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGINE.py", [], 29695)
    assert_follows(lines, gio.intended_training(karate(), 2, 4, 7))


def _three_rank_worker(rank, k):
    """(curve1, curve3): gine's network trained by gine.run's loop on one rank, then on the three ranks of karate_k3 in
    this process (peer transport), gradients averaged over the ranks."""
    import torch.nn.functional as F
    from pgcn_b200.gine import PGINE as Network
    A, pv, k = problem("karate")
    n, f, L, epochs = A.shape[0], 4, 2, 50

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = Network(p, f, L).to(dev())
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
    """gine.run's training loop with the three ranks of karate_k3 in one process, against the same loop on one rank
    and against the fp64 oracle with gradients averaged over three ranks."""
    A, _, _ = problem("karate")
    curve1, curve3 = _eager(_three_rank_worker)
    np.testing.assert_allclose(curve1, gio.intended_training(A, 2, 4, 7), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, gio.intended_training(A, 2, 4, 7, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
