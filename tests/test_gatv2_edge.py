"""GATv2 attention with edge features on the H100 path: pgcn_gatv2_edge_forward / _backward_rows / _backward_cols,
op.PGATv2EdgeAttention and PGAT.py --v2 --edge-values.

The fp32 bound is tests/gatv2_edge_oracle.attention's, with CONST = 16 as the transformer tests use.

  * the forward, dXL, dXR, datt and dE against fp64 for the transformer tests' (f, heads), on gemat11, the hub graph and
    a plan with duplicated entries, with and without dropout (p = 0.3); run-to-run bits; E 4 bytes into its buffer (the
    scalar instances) gives the vector instances' bits; without dE every other output keeps its bits;
  * the same graph walked with a chunk of 4 stays within the bound;
  * with E = 0 and no dropout, Z and the gradients lie within the fp32 bound of fp64 and within twice that bound of
    op.PGATv2Attention's (the two order the softmax differently, so their bits differ);
  * the entries the dropout keeps are those op.edge_dropout keeps for the same key and counter;
  * +-inf and NaN in E: NaN and +-inf exactly where the fp32 NumPy restatement has them;
  * a graph with nnz * f > 2^31;
  * torch.profiler, in a process of its own, sees every instance of tests/gatv2_edge_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport, with and without dropout, within the bound of the one-rank fp64 result; on
    two GPUs NCCL gives the peer transport's bits;
  * PGATv2EdgeAttention's autograd in both layouts on one rank (one tensor as XL and XR too) and on three; E without a
    gradient; CUDA-graph capture with dropout on one and two ranks, and a capture before the first eager call refused
    before it enqueues work;
  * PGAT.py --v2 --edge-values follows the fp64 loss curve (plain, with --heads 2, with --attn-dropout 0.5), and the
    layer on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gatv2_edge_oracle as geo
from harness import (ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import (EdgeDropout, PGATv2Attention, PGATv2EdgeAttention, aggregate_gatv2_edge,
                          aggregate_gatv2_edge_backward, edge_dropout)
from test_gatedgcn import edge_rows
from test_transformer_attention import FH, follower, global_entries, key, mask, one_rank_plan, within
from test_transformer_edge import in_eager_process

pytestmark = pytest.mark.gpu
CONST = 16
KEY = 0x0123456789ABCDEF           # the key of test_transformer_attention.mask
P = 0.3
SLOPE = 0.2


def edge_term(lp, f):
    """E of the local entries as a function of their global (row, column) and feature, so that every partition of a
    graph gives each entry the same E (duplicated entries share it)."""
    gi, gj = global_entries(lp)
    c = np.arange(f)
    return (np.sin(0.37 * gi[:, None] + 1.13 * gj[:, None] + 0.71 * c) * 0.8).astype(np.float32)


def inputs(n, f, seed):
    """XL, XR, gZ [n, f] and att [heads, f / heads] as a flat [f] (reshaped by the caller)."""
    rs = np.random.RandomState(seed)
    XL, XR, gZ = ((rs.standard_normal((n, f)) * s).astype(np.float32) for s in (1.0, 1.0, 1.0))
    att = (rs.standard_normal(f) * 0.7).astype(np.float32)
    return XL, XR, gZ, att


def reference(lp, XL, XR, att, E, gZ, heads, p=0.0, counter=1):
    """{name: (fp64 value, bound)} of a one-rank plan (h = 0) on global inputs."""
    return geo.attention(lp.rowptr, lp.colidx, lp.m, XL, XR, att.reshape(heads, -1), E, gZ, SLOPE, CONST,
                         mask(lp, heads, p, counter))


def run_all(plan, XL, XR, att, E, gZ, f, heads, drop=None, snap=None, walks=None, G=None):
    """(Z, L, dXR, D, PS, G, datt, dXL) from the three C calls, outputs NaN-filled first; walks default to the plan's,
    G (the row walk's g, which is dE) to a fresh buffer."""
    fwd, tr = walks or plan.gated_walks()
    perm = plan.transposed_entries()
    lib, lp = cabi.load_gatv2_edge(), plan.lp
    cabi.check_gatv2_edge(lib.pgcn_gatv2_edge_load())
    gid = plan.global_ids()
    nan = lambda *s: torch.full(s, float("nan"), device=dev())
    Z, L, dXR, D, dXL = nan(lp.m, f), nan(lp.m, heads), nan(lp.m, f), nan(lp.m, heads), nan(lp.m + lp.h, f)
    PS, datt = nan(lp.nnz(), 2 * heads), nan(f)
    G = nan(lp.nnz(), f) if G is None else G.fill_(float("nan"))
    w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev())
    w1 = torch.empty((lib.pgcn_gatv2_edge_work_rows(C.byref(fwd.c)), f), device=dev())
    w2 = torch.empty((tr.nslots, f), device=dev())
    dargs = (None, 0, 1.0) if drop is None else (snap.data_ptr(), drop.threshold, drop.scale)
    head = (lp.m, lp.h, heads, XL.data_ptr(), None, XR.data_ptr(), att.data_ptr(), E.data_ptr(), SLOPE,
            gid.data_ptr()) + dargs
    cabi.check_gatv2_edge(lib.pgcn_gatv2_edge_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                      w0.data_ptr(), f, stream()))
    cabi.check_gatv2_edge(lib.pgcn_gatv2_edge_backward_rows(
        C.byref(fwd.c), *head, gZ.data_ptr(), Z.data_ptr(), L.data_ptr(), dXR.data_ptr(), D.data_ptr(), PS.data_ptr(),
        G.data_ptr(), datt.data_ptr(), w1.data_ptr(), f, stream()))
    cabi.check_gatv2_edge(lib.pgcn_gatv2_edge_backward_cols(
        C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, heads, gZ.data_ptr(), PS.data_ptr(), G.data_ptr(), dXL.data_ptr(),
        w2.data_ptr(), f, stream()))
    torch.cuda.synchronize()
    return Z, L, dXR, D, PS, G, datt, dXL


NAMES = ("Z", "L", "dXR", "D", "PS", "dE", "datt", "dXL")


def check_one_rank(plan, ins, En, f, heads, p=0.0, walks=None, shift_E=False, shift_G=False):
    """Run the three calls on (XL, XR, gZ, att) and E with a fresh draw at counter 1, check every output against fp64."""
    lp = plan.lp
    XLn, XRn, gn, an = ins
    XL, XR, gZ, att, E = t(XLn), t(XRn), t(gn), t(an), t(En)
    if shift_E:
        E = shifted(E)
    G = shifted(torch.empty((lp.nnz(), f), device=dev())) if shift_G else None
    drop = EdgeDropout(p, KEY, dev()) if p > 0 else None
    snap = drop.draw() if drop else None
    out = run_all(plan, XL, XR, att, E, gZ, f, heads, drop, snap, walks, G)
    Z, L, dXR, D, PS, G, datt, dXL = out
    ref = reference(lp, XLn, XRn, an, En, gn, heads, p)
    for name, got in (("Z", Z), ("L", L), ("dXR", dXR), ("dXL", dXL), ("datt", datt.view(heads, -1)), ("dE", G),
                      ("P", PS[:, :heads]), ("ds", PS[:, heads:])):
        within(got, ref[name], "%s f=%d heads=%d p=%g" % (name, f, heads, p))
    return out


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("f,heads", FH)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_run_to_run_and_scalar_bits(case, f, heads, p):
    if case != "gemat11_k1" and (f, heads) not in ((3, 1), (8, 8), (128, 4), (136, 8), (256, 2)):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
        assert plan.gated_walks()[0].nslots > 0
    ins = inputs(lp.m, f, f + heads + len(case))
    En = edge_term(lp, f)
    first = check_one_rank(plan, ins, En, f, heads, p)
    again = check_one_rank(plan, ins, En, f, heads, p)
    scalar = check_one_rank(plan, ins, En, f, heads, p, shift_E=True)
    scalar_g = check_one_rank(plan, ins, En, f, heads, p, shift_G=True)
    for name, a, b, s, sg in zip(NAMES, first, again, scalar, scalar_g):
        assert np.array_equal(bits(a), bits(b)) and np.array_equal(bits(a), bits(s)), name
        assert np.array_equal(bits(a), bits(sg)), name
    plan.close()


def test_without_dE_every_other_output_keeps_its_bits():
    """The operator without dE: the same node gradients and datt as with it (the row walk writes g to scratch)."""
    f, heads = 64, 4
    plan = one_rank_plan("hub", f)
    lp = plan.lp
    XLn, XRn, gn, an = inputs(lp.m, f, 12)
    XL, XR, gZ, att, E = t(XLn), t(XRn), t(gn), t(an).view(heads, -1), t(edge_term(lp, f))
    outs = []
    for need in (True, False):
        drop = EdgeDropout(P, KEY, dev())
        Z, L, XLh, snap = aggregate_gatv2_edge(plan, XL, XR, att, E, SLOPE, drop)
        outs.append((Z, L) + aggregate_gatv2_edge_backward(plan, XL, XLh, XR, att, E, Z, L, gZ, SLOPE, drop, snap,
                                                           need_dE=need))
    assert outs[1][-1] is None and outs[0][-1] is not None
    for a, b in zip(outs[0][:-1], outs[1][:-1]):
        assert torch.equal(a, b)
    plan.close()


@pytest.mark.parametrize("f,heads", [(4, 1), (5, 1), (64, 4), (136, 8)])
def test_forced_small_chunk_stays_within_the_bound(f, heads):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    ins = inputs(lp.m, f, 9)
    En = edge_term(lp, f)
    for p in (0.0, P):
        check_one_rank(plan, ins, En, f, heads, p)
        check_one_rank(plan, ins, En, f, heads, p, walks=small)
    plan.close()


@pytest.mark.parametrize("case,f,heads", [("gemat11_k1", 64, 4), ("gemat11_k1", 6, 2), ("hub", 136, 8),
                                          ("dup", 24, 1), ("gemat11_k1", 128, 1)])
def test_zero_edge_term_within_the_bound_of_the_attention_without_edges(case, f, heads):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    XLn, XRn, gn, an = inputs(lp.m, f, 41)
    En = np.zeros((lp.nnz(), f), np.float32)
    ref = reference(lp, XLn, XRn, an, En, gn, heads)
    XL, XR, gZ, att, E = t(XLn), t(XRn), t(gn), t(an).view(heads, -1), t(En)
    Z1, L1, XLh, _ = aggregate_gatv2_edge(plan, XL, XR, att, E, SLOPE)
    dXL1, dXR1, datt1, _ = aggregate_gatv2_edge_backward(plan, XL, XLh, XR, att, E, Z1, L1, gZ, SLOPE)
    leaves = [x.clone().requires_grad_(True) for x in (XL, XR, att)]
    Z0 = PGATv2Attention.apply(plan, *leaves, SLOPE)
    Z0.backward(gZ)
    for name, a, b in (("Z", Z1, Z0), ("dXL", dXL1, leaves[0].grad), ("dXR", dXR1, leaves[1].grad),
                       ("datt", datt1, leaves[2].grad)):
        val, tol = ref[name]
        within(a, (val, tol), "edge kernels, E = 0: " + name)
        within(a, (b.detach().cpu().numpy().astype(np.float64), 2 * tol), "PGATv2Attention, E = 0: " + name)
    plan.close()


def test_kept_entries_are_those_of_edge_dropout():
    f, heads = 32, 4
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    ins = inputs(lp.m, f, 5)
    out = check_one_rank(plan, ins, edge_term(lp, f), f, heads, P)
    PS = out[4]
    d = EdgeDropout(P, KEY, dev())
    kept = edge_dropout(plan, torch.ones((lp.nnz(), heads), device=dev()), d)       # counter 1, as check_one_rank
    assert (kept == 0).any() and (kept != 0).any()
    assert torch.equal(PS[:, :heads] == 0, kept == 0)
    plan.close()


@pytest.mark.parametrize("f,heads", [(5, 1), (8, 2)])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values_in_E(case, f, heads):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    XLn, XRn, gn, an = inputs(lp.m, f, 3 * f)
    En = edge_term(lp, f)
    rs = np.random.RandomState(f)
    u = rs.uniform(size=En.shape)
    En[u < 0.004] = np.inf
    En[(u >= 0.004) & (u < 0.008)] = -np.inf
    En[(u >= 0.008) & (u < 0.01)] = np.nan
    Z, L, dXR, _, _, dE, datt, dXL = run_all(plan, t(XLn), t(XRn), t(an), t(En), t(gn), f, heads)
    fwd = plan.gated_walks()[0]
    ref = geo.fp32_reference(lp.rowptr, lp.colidx, XLn, XRn, an.reshape(heads, -1), En, gn, SLOPE,
                             fwd.items.cpu().numpy(), fwd.splits.cpu().numpy())
    has = np.diff(lp.rowptr.astype(np.int64)) > 0
    for name, got in (("Z", Z), ("L", L), ("dXR", dXR), ("dXL", dXL), ("dE", dE), ("datt", datt.view(heads, -1))):
        g, w = got.cpu().numpy(), ref[name]
        if name == "L":
            g, w = g[has], w[has]
        if name != "datt":
            assert np.isnan(w).any(), name
        assert np.array_equal(np.isnan(g), np.isnan(w)), "%s: %d NaN differ" % (name, int((np.isnan(g) != np.isnan(w)).sum()))
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    plan.close()


def test_entry_offsets_beyond_2_31():
    """A banded graph with nnz * f > 2^31 (f = 256, 4 heads): the last rows' Z, L, dXR and their entries' dE, and the
    last columns' dXL, within the bound of fp64 over the last rows' entries."""
    import scipy.sparse as sp
    m, band, f, heads = 40000, 216, 256, 4
    rows = np.repeat(np.arange(m), band)
    cols = (rows + np.tile(np.arange(band), m)) % m
    A = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(m, m))
    lp = planmod.build_local_plan(A, np.zeros(m, dtype=np.int64), 0, 1)
    nnz = lp.nnz()
    assert nnz * f > 2 ** 31
    plan = planmod.PgcnPlan(lp, f, device=dev())
    plan.bind_values()
    g = torch.Generator(device=dev()).manual_seed(5)
    XL, XR, gZ = (torch.randn((m, f), device=dev(), generator=g) for _ in range(3))
    att = torch.randn((heads, f // heads), device=dev(), generator=g)
    E = torch.randn((nnz, f), device=dev(), generator=g)
    Z, L, XLh, _ = aggregate_gatv2_edge(plan, XL, XR, att, E, SLOPE)
    dXL, dXR, _, dE = aggregate_gatv2_edge_backward(plan, XL, XLh, XR, att, E, Z, L, gZ, SLOPE)
    torch.cuda.synchronize()
    last = 400                                                      # rows m - 400 .. m - 1
    e0 = int(lp.rowptr[m - last])
    sub_ptr = lp.rowptr[m - last:].astype(np.int64) - e0
    sub_col = lp.colidx[e0:]
    cpu = lambda x: x.cpu().numpy()
    ref = geo.attention(sub_ptr, sub_col, m, cpu(XL), cpu(XR[m - last:]), cpu(att), cpu(E[e0:]), cpu(gZ[m - last:]),
                        SLOPE, CONST, dcol=np.full(m, band))
    for name, got in (("Z", Z[m - last:]), ("L", L[m - last:]), ("dXR", dXR[m - last:]), ("dE", dE[e0:])):
        within(got, ref[name], "nnz*f > 2^31: " + name)
    done = slice(m - 100, m)                                        # every entry of these columns is in the last rows
    val, tol = ref["dXL"]
    within(dXL[done], (val[done], tol[done]), "nnz*f > 2^31: dXL")
    plan.close()


def _instances_worker(rank, k):
    """The keys of the kernels torch.profiler sees while every instance runs (vector and scalar, split rows through the
    delta and fixup kernels), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for f, heads, shift in ((8, 2, False), (6, 2, False), (8, 2, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        walks = (planmod.GatedWalk(lp.rowptr, lp.colidx, 64, dev()),
                 planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 64, dev()))
        assert walks[0].c.nsplits > 0 and walks[1].c.nsplits > 0
        ins = inputs(lp.m, f, f)
        En = edge_term(lp, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                check_one_rank(plan, ins, En, f, heads, P, walks=walks, shift_E=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "gatv2_edge_" in e.name}
            if len(names) == 7:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    with open(os.path.join(ROOT, "tests", "gatv2_edge_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


# ---- several ranks ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("case,f,heads", [("gemat11_k2", 64, 4), ("gemat11_k2", 8, 2), ("gemat11_k3_hp", 16, 1),
                                          ("gemat11_k3_hp", 136, 8)])
def test_multi_rank_within_the_bound_of_one_rank(case, f, heads, p):
    A, pv, k = problem(case)
    n = A.shape[0]
    XLn, XRn, gn, an = inputs(n, f, f + k)
    one = one_rank_plan(case, f)
    lp1 = one.lp
    E1 = edge_term(lp1, f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    pos = [edge_rows(lp1, lp) for lp in lps]
    att = t(an).view(heads, -1)
    ins = [[t(a[lp.owned]) for a in (XLn, XRn, gn)] + [t(edge_term(lp, f))] for lp in lps]
    drops = [EdgeDropout(p, KEY, dev()) for _ in plans]

    def step(r):
        XL, XR, g, E = ins[r]
        Z, L, XLh, snap = aggregate_gatv2_edge(plans[r], XL, XR, att, E, SLOPE, drops[r])
        return (Z, L) + aggregate_gatv2_edge_backward(plans[r], XL, XLh, XR, att, E, Z, L, g, SLOPE, drops[r], snap)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs; counters 1 and 2
        ref = reference(lp1, XLn, XRn, an, E1, gn, heads, p, rep + 1)
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "L", "dXL", "dXR", "dE"), out[r][:4] + out[r][5:]):
                val, tol = ref[name]
                sel = pos[r] if name == "dE" else lp.owned
                within(got, (val[sel], tol[sel]), "%s %s rank %d rep %d" % (case, name, r, rep))
        # each rank's datt covers its own entries; their sum is the whole graph's
        val, tol = ref["datt"]
        within(sum(o[4] for o in out), (val, tol * k), "%s datt rep %d" % (case, rep))
        if first is None:
            first = [[bits(x) for x in o] for o in out]
        elif p == 0:
            assert all(np.array_equal(a, bits(b)) for fo, o in zip(first, out) for a, b in zip(fo, o))
    for p_ in plans + [one]:
        p_.close()


def _nccl_worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    A, pv, _ = problem("gemat11_k2")
    n, f, heads = A.shape[0], 64, 4
    p = planmod.build_plan(A, pv, rank, k, f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    XLn, XRn, gn, an = inputs(n, f, 1)
    XL, XR = (torch.from_numpy(a[own]).cuda().requires_grad_(True) for a in (XLn, XRn))
    att = torch.from_numpy(an.reshape(heads, -1)).cuda().requires_grad_(True)
    E = torch.from_numpy(edge_term(p.lp, f)).cuda().requires_grad_(True)
    Z = PGATv2EdgeAttention.apply(p, XL, XR, att, E, SLOPE, EdgeDropout(P, KEY, torch.device("cuda", rank)))
    Z.backward(torch.from_numpy(gn[own]).cuda())
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), XL.grad, XR.grad, att.grad, E.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29895, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29896, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        for x, y in zip(a[r][1], b[r][1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("layout", ["local", "global"])
def test_autograd_one_rank(layout):
    f, heads = 32, 4
    plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp = plan.lp
    XLn, XRn, gn, an = inputs(lp.m, f, 4)
    En = edge_term(lp, f)
    XL, XR, att, E = (t(a).requires_grad_(True) for a in (XLn, XRn, an.reshape(heads, -1), En))
    Z = PGATv2EdgeAttention.apply(plan, XL, XR, att, E, SLOPE)
    Z.backward(t(gn))
    ref = reference(lp, XLn, XRn, an, En, gn, heads)
    for name, got in (("Z", Z), ("dXL", XL.grad), ("dXR", XR.grad), ("datt", att.grad), ("dE", E.grad)):
        within(got, ref[name], "%s %s" % (layout, name))
    # E without a gradient: the same other gradients, and none for E
    XL2, XR2, att2 = (t(a).requires_grad_(True) for a in (XLn, XRn, an.reshape(heads, -1)))
    E2 = t(En)
    Z2 = PGATv2EdgeAttention.apply(plan, XL2, XR2, att2, E2, SLOPE)
    Z2.backward(t(gn))
    assert E2.grad is None
    for a, b in ((Z, Z2), (XL.grad, XL2.grad), (XR.grad, XR2.grad), (att.grad, att2.grad)):
        assert torch.equal(a, b)
    # one tensor as XL and XR (share_weights=True): its gradient is the sum of both
    X = t(XLn).requires_grad_(True)
    Z3 = PGATv2EdgeAttention.apply(plan, X, X, t(an.reshape(heads, -1)), t(En), SLOPE)
    Z3.backward(t(gn))
    ref = reference(lp, XLn, XLn, an, En, gn, heads)
    within(Z3, ref["Z"], "shared Z")
    val = ref["dXL"][0] + ref["dXR"][0]
    within(X.grad, (val, ref["dXL"][1] + ref["dXR"][1] + 2.0 ** -23 * np.abs(val)), "shared dX")
    plan.close()


def test_autograd_three_ranks_and_global_layout():
    assert in_eager_process(_autograd_three_ranks_worker)


def _autograd_three_ranks_worker(rank, k):
    A, pv, k = problem("gemat11_k3_hp")
    n, f, heads = A.shape[0], 16, 2
    XLn, XRn, gn, an = inputs(n, f, 3)
    one = one_rank_plan("gemat11_k3_hp", f)
    E1 = edge_term(one.lp, f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    pos = [edge_rows(one.lp, lp) for lp in lps]
    plans = linked_plans(lps, f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    for counter, layout in enumerate(("local", "global"), 1):
        ref = reference(one.lp, XLn, XRn, an, E1, gn, heads, P, counter)
        for p in plans:
            p.layout = layout
        if counter == 1:
            drops = [EdgeDropout(P, KEY, dev()) for _ in plans]
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [[t(pick(a, lp)).requires_grad_(True) for a in (XLn, XRn)]
                  + [t(an.reshape(heads, -1)).requires_grad_(True), t(E1[q]).requires_grad_(True)]
                  for lp, q in zip(lps, pos)]
        Z = run_ranks(plans, lambda r: PGATv2EdgeAttention.apply(plans[r], *leaves[r], SLOPE, drops[r]), streams)
        run_ranks(plans, lambda r: Z[r].backward(t(pick(gn, lps[r]))), streams)
        datt = 0
        for r, lp in enumerate(lps):
            datt = datt + leaves[r][2].grad
            for name, got in zip(("Z", "dXL", "dXR", "dE"), [Z[r]] + [leaves[r][i].grad for i in (0, 1, 3)]):
                val, tol = ref[name]
                if name == "dE":
                    within(got, (val[pos[r]], tol[pos[r]]), "%s dE rank %d" % (layout, r))
                elif layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                    within(got, (val, tol), "global %s rank %d" % (name, r))
                else:
                    within(got, (val[lp.owned], tol[lp.owned]), "local %s rank %d" % (name, r))
        within(datt, (ref["datt"][0], ref["datt"][1] * k), "%s datt" % layout)
    for p in plans + [one]:
        p.close()
    return True


def test_one_rank_capture_with_dropout_and_refusal_before_the_first_eager_call():
    f, heads = 64, 4
    plan = one_rank_plan("hub", f)
    m, nnz = plan.lp.m, plan.lp.nnz()
    XL, XR, g = (torch.zeros((m, f), device=dev()) for _ in range(3))
    att = torch.zeros((heads, f // heads), device=dev())
    E = torch.zeros((nnz, f), device=dev())
    drop = EdgeDropout(P, KEY, dev())

    def step(XL, XR, att, E, g, drop):
        Z, L, XLh, snap = aggregate_gatv2_edge(plan, XL, XR, att, E, SLOPE, drop)
        dXL, dXR, datt, dE = aggregate_gatv2_edge_backward(plan, XL, XLh, XR, att, E, Z, L, g, SLOPE, drop, snap)
        return dict(Z=Z, L=L, dXL=dXL, dXR=dXR, datt=datt, dE=dE)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    plan.gated_walks()                                    # the walks and ids exist; the transposed entries do not yet
    plan.global_ids()
    with pytest.raises(RuntimeError, match="transposed_entries"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(XL, XR, att, E, g, drop)
    assert plan.launch_count() == launches and plan._transposed_entries is None and int(drop.state[1]) == 0
    ins = []
    for i in range(3):
        XLn, XRn, gn, an = inputs(m, f, 20 + i)
        ins.append((t(XLn), t(XRn), t(an).view(heads, -1), t(edge_term(plan.lp, f) * (i + 1)), t(gn)))

    def load(i):
        for dst, src in zip((XL, XR, att, E, g), ins[i]):
            dst.copy_(src)

    plan.prepare(f)
    step(*ins[0], None)                                   # the first eager call builds the transposed entries
    check_one_rank_capture(plan, lambda: step(XL, XR, att, E, g, drop), load,
                           lambda i: step(*ins[i], follower(drop)))
    assert int(drop.state[1]) == 4                        # one draw per replay, none at capture
    plan.close()


def test_two_rank_capture_with_dropout_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n, heads = 64, A.shape[0], 2
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
        p.gated_walks()
        p.global_ids()
        p.transposed_entries()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, f, 30 + i) for i in range(3)]
    made = []

    def buffers(r):
        b = {name: torch.zeros((lps[r].m, f), device=dev()) for name in ("x", "r", "g")}
        b["a"] = torch.zeros((heads, f // heads), device=dev())
        b["e"] = torch.zeros((lps[r].nnz(), f), device=dev())
        b["drop"] = EdgeDropout(P, KEY, dev())
        made.append(b)
        return b

    def load(bufs, i):
        XLn, XRn, gn, an = ins[i]
        for r, lp in enumerate(lps):
            for name, a in zip(("x", "r", "g"), (XLn, XRn, gn)):
                bufs[r][name].copy_(t(a[lp.owned]))
            bufs[r]["a"].copy_(t(an).view(heads, -1))
            bufs[r]["e"].copy_(t(edge_term(lp, f) * (i + 1)))
            if bufs[r] is not made[r]:                    # eager buffers draw with the counter the replay just used
                bufs[r]["drop"] = follower(made[r]["drop"])
        torch.cuda.synchronize()

    def step(r, b):
        Z, L, XLh, snap = aggregate_gatv2_edge(plans[r], b["x"], b["r"], b["a"], b["e"], SLOPE, b["drop"])
        dXL, dXR, datt, dE = aggregate_gatv2_edge_backward(plans[r], b["x"], XLh, b["r"], b["a"], b["e"], Z, L, b["g"],
                                                           SLOPE, b["drop"], snap)
        return dict(Z=Z, dXL=dXL, dXR=dXR, datt=datt, dE=dE)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for r in range(k):
        assert int(made[r]["drop"].state[1]) == 4
    for p in plans:
        p.close()


# ---- the command line ------------------------------------------------------------------------------------------------

def test_cli_edge_values_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", ["--v2", "--edge-values"], 29795)
    assert_follows(lines, geo.intended_training(karate(), 2, 4, 7, 1.0))


def test_cli_edge_values_heads_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", ["--v2", "--edge-values", "--heads", "2"], 29796)
    assert_follows(lines, geo.intended_training(karate(), 2, 4, 7, 1.0, heads=2))


def test_cli_edge_values_attn_dropout_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", ["--v2", "--edge-values", "--attn-dropout", "0.5"], 29797)
    assert_follows(lines, geo.intended_training(karate(), 2, 4, 7, 1.0, p=0.5))


def _three_rank_worker(rank, k):
    """pgat.run's training loop with --v2 --edge-values on one rank and on the three ranks of karate_k3 in this
    process (peer transport): (one-rank curve, three-rank curve)."""
    import torch.nn as nn
    import torch.nn.functional as F
    from pgcn_b200.pgat import PGATv2
    A, pv, k = problem("karate")
    n, f, L, epochs, heads = A.shape[0], 4, 2, 50, 2

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = nn.Sequential(*[PGATv2(p, f, f, 1.0, heads, edge_values=True) for _ in range(L)]).to(dev())
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


def test_edge_values_layer_on_three_ranks_follows_the_one_rank_curve():
    """The layer with --edge-values on one rank and on three, against the fp64 oracle with gradients averaged over
    three ranks, the ranks in a process of their own (in_eager_process)."""
    A, _, _ = problem("karate")
    curve1, curve3 = in_eager_process(_three_rank_worker)
    np.testing.assert_allclose(curve1, geo.intended_training(A, 2, 4, 7, 1.0, heads=2), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, geo.intended_training(A, 2, 4, 7, 1.0, heads=2, k=3), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
