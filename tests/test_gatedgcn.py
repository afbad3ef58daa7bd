"""GatedGCN on the H100 path: pgcn_gatedgcn_forward / _backward_rows / _backward_cols, PgcnPlan.transposed_entries,
op.PGatedGCN and PGATEDGCN.py.

The fp32 bound is gatedgcn_oracle.terms': a first-order propagation of the kernels' roundings (each gate and each
s (1 - s) within CONST = 16 ulp, every sum d roundings of its sum|terms|), doubled.

  * Z, den and the four gradients against fp64 on gemat11, the hub graph (a split row of 3000 entries, empty rows, rows
    of one entry) and a local plan with duplicated entries, at widths 1 .. 256, with the edge gradient given and absent;
    ehat bit-equal to torch's (Dx[rows] + Ex[cols]) + Ce; an absent edge gradient gives the bits of a zero one;
    run-to-run bits; every operand 4 bytes into its buffer (the scalar instances) gives the vector instances' bits;
  * the same graph walked with a chunk of 4; +-inf and NaN in the operands where the fp32 reference has them; a plan with
    nnz * f > 2^31 checked on its last entries, rows and columns;
  * torch.profiler, in a process of its own, sees every instance of tests/gatedgcn_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport within the bound of the one-rank fp64 result, edges matched by edge_pairs();
    on two GPUs NCCL gives the peer transport's bits;
  * PGatedGCN's autograd in both layouts; CUDA-graph capture on one and two ranks, and a capture before the first eager
    call refused before it enqueues work;
  * PGATEDGCN.py follows the fp64 loss curve, and the network on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gatedgcn_oracle as gco
from harness import (ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PGatedGCN, aggregate_gatedgcn, aggregate_gatedgcn_backward
from test_max_aggregation import with_duplicates

pytestmark = pytest.mark.gpu
WIDTHS = [1, 3, 4, 31, 32, 64, 127, 128, 129, 256]
EPS = 1e-6
NAMES = ("Ehat", "Z", "den", "dCe", "dDx", "dEx", "dBx")


def one_rank_plan(case, f):
    """A bound one-rank plan of width 2f on problem(case) ("dup": gemat11 with duplicated entries)."""
    A, _, _ = problem("gemat11_k1" if case == "dup" else case)
    lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    if case == "dup":
        lp = with_duplicates(lp)
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev())
    plan.bind_values()
    return plan


def inputs(n, nnz, f, seed):
    """Dx, Ex, Bx, gZ ([n, f]) and Ce, gE ([nnz, f]), fp32."""
    rs = np.random.RandomState(seed)
    node = [(rs.standard_normal((n, f)) * s).astype(np.float32) for s in (1.5, 1.5, 1.0, 1.0)]
    edge = [(rs.standard_normal((nnz, f)) * s).astype(np.float32) for s in (1.5, 1.0)]
    return node + edge


def within(got, ref, what):
    val, tol = ref
    g = got.detach().cpu().numpy().astype(np.float64)
    err = np.abs(g - val)
    bad = ~(err <= tol + 1e-30)
    assert not bad.any(), "%s: %d elements beyond the fp32 bound, worst err %.3e" % (what, int(bad.sum()),
                                                                                      float(np.nanmax(err)))


def run_all(plan, Dx, EB, Ce, gZ, gE, f, walks=None, eps=EPS):
    """{name: tensor} from the three C calls (one rank, h = 0), outputs NaN-filled first."""
    fwd, tr = walks or plan.gated_walks()
    perm = plan.transposed_entries()
    lib, lp = cabi.load_gatedgcn(), plan.lp
    nan = lambda *s: torch.full(s, float("nan"), device=dev())
    nnz = lp.nnz()
    o = {"Z": nan(lp.m, f), "den": nan(lp.m, f), "Ehat": nan(nnz, f), "U": nan(lp.m, f), "dCe": nan(nnz, f),
         "dDx": nan(lp.m, f), "dEB": nan(lp.m + lp.h, 2 * f)}
    w1 = torch.empty((fwd.nslots, 2 * f), device=dev())
    w2 = torch.empty((tr.nslots, 2 * f), device=dev())
    p = lambda x: None if x is None else x.data_ptr()
    cabi.check_gatedgcn(lib.pgcn_gatedgcn_forward(C.byref(fwd.c), lp.m, lp.h, p(Dx), p(EB), None, p(Ce), eps,
                                                  p(o["Z"]), p(o["den"]), p(o["Ehat"]), p(w1), f, stream()))
    cabi.check_gatedgcn(lib.pgcn_gatedgcn_backward_rows(C.byref(fwd.c), lp.m, lp.h, p(EB), None, p(o["Ehat"]), p(gE),
                                                        p(o["Z"]), p(o["den"]), p(gZ), eps, p(o["U"]), p(o["dCe"]),
                                                        p(o["dDx"]), p(w1), f, stream()))
    cabi.check_gatedgcn(lib.pgcn_gatedgcn_backward_cols(C.byref(tr.c), p(perm), lp.m, lp.h, p(o["Ehat"]), p(o["dCe"]),
                                                        p(o["U"]), p(o["dEB"]), p(w2), f, stream()))
    torch.cuda.synchronize()
    o["dEx"], o["dBx"] = o["dEB"][:, :f], o["dEB"][:, f:]
    return o


def check_one_rank(plan, ins, f, use_ge, walks=None, shift=False):
    lp = plan.lp
    Dn, En, Bn, gn, Cn, gEn = ins
    ops = [t(Dn), t(np.concatenate([En, Bn], 1)), t(Cn), t(gn), t(gEn) if use_ge else None]
    if shift:
        ops = [None if x is None else shifted(x) for x in ops]
    out = run_all(plan, *ops, f, walks)
    ref = gco.terms(lp.rowptr, lp.colidx, lp.m, Dn, En, Bn, Cn, gn, gEn if use_ge else None, eps=EPS)
    for name in NAMES:
        within(out[name], ref[name], "%s f=%d gE=%s" % (name, f, use_ge))
    return out


@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_exact_ehat_and_bits(case, f):
    if case != "gemat11_k1" and f not in (3, 4, 32, 129, 256):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
        assert plan.gated_walks()[0].nslots > 0
    ins = inputs(lp.m, lp.nnz(), f, f + len(case))
    Dn, En, Bn, gn, Cn, gEn = ins
    first = check_one_rank(plan, ins, f, True)
    # ehat is torch's (Dx[rows] + Ex[cols]) + Ce to the bit
    r = torch.from_numpy(np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))).to(dev())
    c = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev())
    assert np.array_equal(bits(first["Ehat"]), bits((t(Dn)[r] + t(En)[c]) + t(Cn)))
    again = check_one_rank(plan, ins, f, True)
    scalar = check_one_rank(plan, ins, f, True, shift=True)
    for name in NAMES:
        assert np.array_equal(bits(first[name]), bits(again[name])), name
        assert np.array_equal(bits(first[name]), bits(scalar[name])), name
    # an absent edge gradient is an explicit zero one, to the bit
    none = check_one_rank(plan, ins, f, False)
    zero = run_all(plan, t(Dn), t(np.concatenate([En, Bn], 1)), t(Cn), t(gn), torch.zeros((lp.nnz(), f), device=dev()),
                   f)
    for name in NAMES:
        assert np.array_equal(bits(none[name]), bits(zero[name])), name
    plan.close()


@pytest.mark.parametrize("f", [4, 5, 64])
def test_forced_small_chunk_stays_within_the_bound(f):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    assert plan.gated_walks()[0].nslots == plan.gated_walks()[1].nslots == 0
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    ins = inputs(lp.m, lp.nnz(), f, 9)
    whole = check_one_rank(plan, ins, f, True)
    split = check_one_rank(plan, ins, f, True, walks=small)
    assert np.array_equal(bits(whole["Ehat"]), bits(split["Ehat"]))      # ehat does not depend on the chunking
    plan.close()


@pytest.mark.parametrize("f", [5, 8])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values(case, f):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    ins = inputs(lp.m, lp.nnz(), f, 3 * f)
    Dn, En, Bn, gn, Cn, gEn = ins
    rs = np.random.RandomState(f)
    for x in (Dn, En, Bn, Cn):
        u = rs.uniform(size=x.shape)
        x[u < 0.005] = np.inf
        x[(u >= 0.005) & (u < 0.01)] = -np.inf
        x[(u >= 0.01) & (u < 0.0125)] = np.nan
    out = run_all(plan, t(Dn), t(np.concatenate([En, Bn], 1)), t(Cn), t(gn), t(gEn), f)
    ref = gco.fp32_reference(lp.rowptr, lp.colidx, lp.m, Dn, En, Bn, Cn, gn, gEn, eps=EPS)
    for name in NAMES:
        g, w = out[name].cpu().numpy(), ref[name]
        assert np.isnan(w).any(), name
        assert np.array_equal(np.isnan(g), np.isnan(w)), name
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    plan.close()


def test_entry_offsets_beyond_2_31():
    """A banded graph with nnz * f > 2^31 (f = 256): the last entries' ehat bits, and the last rows' Z and dDx and the
    last columns' dEx and dBx within the bound, from fp64 over the last rows' entries."""
    import scipy.sparse as sp
    m, band, f = 40000, 216, 256
    rows = np.repeat(np.arange(m), band)
    cols = (rows + np.tile(np.arange(band), m)) % m
    A = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(m, m))
    lp = planmod.build_local_plan(A, np.zeros(m, dtype=np.int64), 0, 1)
    nnz = lp.nnz()
    assert nnz * f > 2 ** 31
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev())
    plan.bind_values()
    g = torch.Generator(device=dev()).manual_seed(5)
    Dx, Ex, Bx, gZ = (torch.randn((m, f), device=dev(), generator=g) for _ in range(4))
    Ce = torch.randn((nnz, f), device=dev(), generator=g)
    gE = torch.randn((nnz, f), device=dev(), generator=g)
    Z, Ehat, den, EB, EBh = aggregate_gatedgcn(plan, Dx, Ex, Bx, Ce)
    dDx, dEx, dBx, dCe = aggregate_gatedgcn_backward(plan, Ehat, EB, EBh, Z, den, gZ, gE)
    torch.cuda.synchronize()
    last = 400                                                      # rows m - 400 .. m - 1
    e0 = int(lp.rowptr[m - last])
    sub_ptr = lp.rowptr[m - last:].astype(np.int64) - e0
    sub_col = lp.colidx[e0:]
    cpu = lambda x: x.cpu().numpy()
    Dn = np.zeros((last, f), np.float32)
    Dn[:] = cpu(Dx[m - last:])
    ref = gco.terms(sub_ptr, sub_col, m, Dn, cpu(Ex), cpu(Bx), cpu(Ce[e0:]), cpu(gZ[m - last:]), cpu(gE[e0:]), eps=EPS)
    assert np.array_equal(bits(Ehat[e0:]), ref["Ehat"][0].astype(np.float32).view(np.uint32))
    for name, got in (("Z", Z[m - last:]), ("den", den[m - last:]), ("dDx", dDx[m - last:]), ("dCe", dCe[e0:])):
        within(got, ref[name], "nnz*f > 2^31: " + name)
    cols_done = slice(m - 100, m)                                   # every entry of these columns is in the last rows
    for name, got in (("dEx", dEx), ("dBx", dBx)):
        val, tol = ref[name]
        within(got[cols_done], (val[cols_done], tol[cols_done]), "nnz*f > 2^31: " + name)
    plan.close()


def key(name):
    """Instance name without return type, parameter list, casts and spaces, bools as 0 / 1."""
    s = name.strip()
    for a, b in (("(int)", ""), ("(bool)", ""), ("true", "1"), ("false", "0")):
        s = s.replace(a, b)
    if s.startswith("void "):
        s = s[5:]
    return s.split("(")[0].replace(" ", "")


def _instances_worker(rank, k):
    """The keys of the GatedGCN kernels torch.profiler sees while every instance runs (vector and scalar, split rows
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
                check_one_rank(plan, ins, f, True, walks=walks, shift=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "gatedgcn_" in e.name}
            if len(names) == 6:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    with open(os.path.join(ROOT, "tests", "gatedgcn_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


# ---- several ranks ---------------------------------------------------------------------------------------------------

def edge_rows(lp_one, lp):
    """For every local entry of lp, the index of the same (global row, global column) entry in the one-rank plan
    lp_one (whose local ids are global ids)."""
    n = lp_one.n
    r1 = np.repeat(lp_one.owned, np.diff(lp_one.rowptr.astype(np.int64)))
    k1 = r1 * n + lp_one.owned[lp_one.colidx]
    order = np.argsort(k1, kind="stable")
    r = np.repeat(lp.owned, np.diff(lp.rowptr.astype(np.int64)))
    key = r * n + np.concatenate([lp.owned, lp.halo])[lp.colidx]
    pos = order[np.searchsorted(k1[order], key)]
    assert np.array_equal(k1[pos], key)
    return pos


# 2f a multiple of 4, the widths the peer transport's halo exchange takes; f = 6 and 130 run the scalar instances
@pytest.mark.parametrize("case,f", [("gemat11_k2", 64), ("gemat11_k2", 6), ("gemat11_k3_hp", 16),
                                    ("gemat11_k3_hp", 130)])
def test_multi_rank_within_the_bound_of_one_rank(case, f):
    A, pv, k = problem(case)
    n = A.shape[0]
    one = one_rank_plan(case, f)
    lp1 = one.lp
    Dn, En, Bn, gn, Cn, gEn = inputs(n, lp1.nnz(), f, f + k)
    ref = gco.terms(lp1.rowptr, lp1.colidx, n, Dn, En, Bn, Cn, gn, gEn, eps=EPS)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    # the pairs edge_pairs() gives are the ones edge_rows matches
    pos = []
    for p, lp in zip(plans, lps):
        pos.append(edge_rows(lp1, lp))
        assert np.array_equal(p.edge_pairs().cpu().numpy().astype(np.int64),
                              one.edge_pairs().cpu().numpy().astype(np.int64)[pos[-1]])
    ins = [[t(a[lp.owned]) for a in (Dn, En, Bn, gn)] + [t(Cn[q]), t(gEn[q])] for lp, q in zip(lps, pos)]

    def step(r):
        D, E, B, g, Ce, gE = ins[r]
        Z, Ehat, den, EB, EBh = aggregate_gatedgcn(plans[r], D, E, B, Ce)
        return (Ehat, Z, den) + aggregate_gatedgcn_backward(plans[r], Ehat, EB, EBh, Z, den, g, gE)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Ehat", "Z", "den", "dDx", "dEx", "dBx", "dCe"), out[r]):
                val, tol = ref[name]
                sel = pos[r] if name in ("Ehat", "dCe") else lp.owned
                within(got, (val[sel], tol[sel]), "%s %s rank %d rep %d" % (case, name, r, rep))
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
    p = planmod.build_plan(A, pv, rank, k, 2 * f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    Dn, En, Bn, gn, _, _ = inputs(n, 1, f, 1)
    Ce = torch.randn((p.lp.nnz(), f), generator=torch.Generator().manual_seed(rank)).cuda().requires_grad_(True)
    D, E, B, g = (torch.from_numpy(a[own]).cuda().requires_grad_(True) for a in (Dn, En, Bn, gn))
    Z, Eh = PGatedGCN.apply(p, D, E, B, Ce)
    (Z * g.detach()).sum().backward()
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), Eh.detach(), D.grad, E.grad, B.grad, Ce.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29881, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29882, "p2p"))
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
    Dn, En, Bn, gn, Cn, gEn = inputs(lp.m, lp.nnz(), f, 4)
    D, E, B, Ce = (t(a).requires_grad_(True) for a in (Dn, En, Bn, Cn))
    Z, Eh = PGatedGCN.apply(plan, D, E, B, Ce)
    ((Z * t(gn)).sum() + (Eh * t(gEn)).sum()).backward()
    ref = gco.terms(lp.rowptr, lp.colidx, lp.m, Dn, En, Bn, Cn, gn, gEn, eps=EPS)
    for name, got in (("Z", Z), ("Ehat", Eh), ("dDx", D.grad), ("dEx", E.grad), ("dBx", B.grad), ("dCe", Ce.grad)):
        within(got, ref[name], "%s %s" % (layout, name))
    # only Z used: the edge gradient reaches the kernels as NULL, and gives the bits of a zero one
    D2, E2, B2, C2 = (t(a).requires_grad_(True) for a in (Dn, En, Bn, Cn))
    Z2, _ = PGatedGCN.apply(plan, D2, E2, B2, C2)
    Z2.backward(t(gn))
    out = run_all(plan, t(Dn), t(np.concatenate([En, Bn], 1)), t(Cn), t(gn), None, f)
    for name, got in (("dDx", D2.grad), ("dCe", C2.grad), ("dEx", E2.grad), ("dBx", B2.grad)):
        assert np.array_equal(bits(got), bits(out[name])), name
    plan.close()


def test_autograd_three_ranks_and_global_layout():
    A, pv, k = problem("gemat11_k3_hp")
    n, f = A.shape[0], 16
    one = one_rank_plan("gemat11_k3_hp", f)
    lp1 = one.lp
    Dn, En, Bn, gn, Cn, gEn = inputs(n, lp1.nnz(), f, 3)
    ref = gco.terms(lp1.rowptr, lp1.colidx, n, Dn, En, Bn, Cn, gn, gEn, eps=EPS)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    pos = [edge_rows(lp1, lp) for lp in lps]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    for layout in ("local", "global"):
        for p in plans:
            p.layout = layout
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [[t(pick(a, lp)).requires_grad_(True) for a in (Dn, En, Bn)] + [t(Cn[q]).requires_grad_(True)]
                  for lp, q in zip(lps, pos)]
        out = run_ranks(plans, lambda r: PGatedGCN.apply(plans[r], *leaves[r]), streams)
        run_ranks(plans, lambda r: ((out[r][0] * t(pick(gn, lps[r]))).sum()
                                    + (out[r][1] * t(gEn[pos[r]])).sum()).backward(), streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "dDx", "dEx", "dBx"), [out[r][0]] + [x.grad for x in leaves[r][:3]]):
                val, tol = ref[name]
                if layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                    within(got, (val, tol), "global %s rank %d" % (name, r))
                else:
                    within(got, (val[lp.owned], tol[lp.owned]), "local %s rank %d" % (name, r))
            within(out[r][1], (ref["Ehat"][0][pos[r]], ref["Ehat"][1][pos[r]]), "%s Ehat rank %d" % (layout, r))
            within(leaves[r][3].grad, (ref["dCe"][0][pos[r]], ref["dCe"][1][pos[r]]), "%s dCe rank %d" % (layout, r))
    for p in plans + [one]:
        p.close()


def test_one_rank_capture_and_refusal_before_the_first_eager_call():
    f = 64
    plan = one_rank_plan("hub", f)
    m, nnz = plan.lp.m, plan.lp.nnz()
    D, E, B, g = (torch.zeros((m, f), device=dev()) for _ in range(4))
    Ce, gE = torch.zeros((nnz, f), device=dev()), torch.zeros((nnz, f), device=dev())

    def step(D, E, B, Ce, g, gE):
        Z, Ehat, den, EB, EBh = aggregate_gatedgcn(plan, D, E, B, Ce)
        dDx, dEx, dBx, dCe = aggregate_gatedgcn_backward(plan, Ehat, EB, EBh, Z, den, g, gE)
        return dict(Z=Z, Ehat=Ehat, dDx=dDx, dEx=dEx, dBx=dBx, dCe=dCe)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    with pytest.raises(RuntimeError, match="gated_walks"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(D, E, B, Ce, g, gE)
    assert plan.launch_count() == launches and plan._gated_walks is None and plan._transposed_entries is None
    plan.gated_walks()
    with pytest.raises(RuntimeError, match="transposed_entries"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(D, E, B, Ce, g, gE)
    assert plan.launch_count() == launches and plan._transposed_entries is None
    ins = []
    for i in range(3):
        Dn, En, Bn, gn, Cn, gEn = inputs(m, nnz, f, 20 + i)
        ins.append(tuple(t(a) for a in (Dn, En, Bn, Cn, gn, gEn)))

    def load(i):
        for dst, src in zip((D, E, B, Ce, g, gE), ins[i]):
            dst.copy_(src)

    plan.prepare(2 * f)
    step(*ins[0])                                         # the first eager call builds the tables
    check_one_rank_capture(plan, lambda: step(D, E, B, Ce, g, gE), load, lambda i: step(*ins[i]))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n = 64, A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    for p in plans:
        p.prepare(2 * f)
        p.gated_walks()
        p.transposed_entries()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, max(lp.nnz() for lp in lps), f, 30 + i) for i in range(3)]

    def buffers(r):
        b = {name: torch.zeros((lps[r].m, f), device=dev()) for name in ("x", "e", "b", "g")}
        b.update({name: torch.zeros((lps[r].nnz(), f), device=dev()) for name in ("c", "ge")})
        return b

    def load(bufs, i):
        for r, lp in enumerate(lps):
            for name, a in zip(("x", "e", "b", "g"), ins[i][:4]):
                bufs[r][name].copy_(t(a[lp.owned]))
            for name, a in zip(("c", "ge"), ins[i][4:]):
                bufs[r][name].copy_(t(a[:lp.nnz()]))
        torch.cuda.synchronize()

    def step(r, b):
        Z, Ehat, den, EB, EBh = aggregate_gatedgcn(plans[r], b["x"], b["e"], b["b"], b["c"])
        dDx, dEx, dBx, dCe = aggregate_gatedgcn_backward(plans[r], Ehat, EB, EBh, Z, den, b["g"], b["ge"])
        return dict(Z=Z, Ehat=Ehat, dDx=dDx, dEx=dEx, dBx=dBx, dCe=dCe)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGATEDGCN.py", [], 29693)
    assert_follows(lines, gco.intended_training(karate(), 2, 4, 7))


def _three_rank_worker(rank, k):
    """(curve1, curve3): gatedgcn's network trained by gatedgcn.run's loop on one rank, then on the three ranks of
    karate_k3 in this process (peer transport), gradients averaged over the ranks."""
    import torch.nn.functional as F
    from pgcn_b200.gatedgcn import PGATEDGCN
    A, pv, k = problem("karate")
    n, f, L, epochs = A.shape[0], 4, 2, 50

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = PGATEDGCN(p, f, L).to(dev())
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
    for p in plans + one:
        p.close()
    return curve1, curve3


def test_network_on_three_ranks_follows_the_one_rank_curve():
    """gatedgcn.run's training loop with the three ranks of karate_k3 in one process, against the same loop on one rank
    and against the fp64 oracle with gradients averaged over three ranks. The ranks run in a process of their own with
    CUDA_MODULE_LOADING=EAGER: a rank's backward launches cuBLAS kernels chosen for its own shapes, and with lazy loading
    the first launch of one waits for the device, where an earlier rank's exchange waits for this rank's half, which
    the blocked thread never enqueues. Ranks in separate processes, as in a real job, do not share that wait."""
    A, _, _ = problem("karate")
    old = os.environ.get("CUDA_MODULE_LOADING")
    os.environ["CUDA_MODULE_LOADING"] = "EAGER"
    try:
        curve1, curve3 = spawn_ranks(_three_rank_worker, 1)[0]
    finally:
        if old is None:
            del os.environ["CUDA_MODULE_LOADING"]
        else:
            os.environ["CUDA_MODULE_LOADING"] = old
    np.testing.assert_allclose(curve1, gco.intended_training(A, 2, 4, 7), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, gco.intended_training(A, 2, 4, 7, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
