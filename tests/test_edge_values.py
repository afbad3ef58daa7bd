"""Edge values set per call and their gradient: pgcn_plan_bind_values / pgcn_plan_set_values, pgcn_sddmm,
pgcn_forward_keep_halo, PSpMMWeighted.

  * a plan created with v0 and set to v1 computes bit for bit what a plan created with v1 computes (forward, backward,
    fused ReLU; every record set, the transposed views and the per-peer blocks), and set_values(None) brings v0 back;
  * the SDDMM lies within the fp32 dot bound of the fp64 truth, halo columns included, and is run-to-run identical;
  * PSpMMWeighted's dvals and dH against an fp64 reference, two layers with different values on one plan;
  * PSpMM after a weighted call equals a fresh plan; errors; CUDA-graph capture of weighted layers, one rank and two
    ranks over the peer transport with both exchange parities.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from harness import check_one_rank_capture, check_two_rank_capture, dev, linked_plans, problem, run_ranks, stream
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PSpMM, PSpMMWeighted

pytestmark = pytest.mark.gpu


def with_values(lp, v):
    """A copy of the local plan whose forward values are v, the transposed values permuted to match."""
    q = planmod.LocalPlan()
    q.__dict__.update(lp.__dict__)
    q.vals = v.astype(np.float32)
    csr = sp.csr_matrix((q.vals, lp.colidx, lp.rowptr), shape=(lp.m, lp.m + lp.h))
    t = csr.T.tocsr()
    t.sort_indices()
    assert np.array_equal(t.indptr, lp.t_rowptr) and np.array_equal(t.indices, lp.t_colidx)
    q.t_vals = t.data.astype(np.float32)
    return q


def new_values(lp, seed):
    rs = np.random.RandomState(seed)
    return (rs.uniform(0.25, 2.0, lp.nnz()) * rs.choice([-1.0, 1.0], lp.nnz())).astype(np.float32)


def fused_outputs(plans, xs, gs, f, streams):
    """pgcn_forward, pgcn_backward and the fused-ReLU forward of every rank."""
    lib = cabi.load()

    def one(r):
        p = plans[r]
        z = torch.empty_like(xs[r]); g = torch.empty_like(xs[r]); zr = torch.empty_like(xs[r])
        cabi.check(lib.pgcn_forward(p.handle, xs[r].data_ptr(), z.data_ptr(), f, stream()), p.handle)
        cabi.check(lib.pgcn_backward(p.handle, gs[r].data_ptr(), g.data_ptr(), f, stream()), p.handle)
        p.set_option("relu", 1)
        cabi.check(lib.pgcn_forward(p.handle, xs[r].data_ptr(), zr.data_ptr(), f, stream()), p.handle)
        p.set_option("relu", 0)
        return z, g, zr
    return run_ranks(plans, one, streams)


CASES = [("gemat11_k1", 1), ("rmat", 1), ("gemat11_k2", 1), ("gemat11_k2", 0), ("gemat11_k3_hp", 1),
         ("gemat11_k3_hp", 0), ("rmat_k2", 1)]


def setup_case(case, f, overlap):
    A, pv, k = problem(case)
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    rs = np.random.RandomState(f + 7 * k)
    H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    xs = [torch.from_numpy(H[lp.owned]).to(dev()) for lp in lps]
    gs = [torch.from_numpy(G[lp.owned]).to(dev()) for lp in lps]
    return lps, H, G, xs, gs


@pytest.mark.parametrize("case,overlap", CASES)
@pytest.mark.parametrize("f", [16, 40, 128, 256])
def test_set_values_is_bit_exact(case, overlap, f):
    lps, H, G, xs, gs = setup_case(case, f, overlap)
    v1 = [new_values(lp, 100 + r) for r, lp in enumerate(lps)]
    pa = linked_plans(lps, f, overlap, bind=False)
    pb = linked_plans([with_values(lp, v) for lp, v in zip(lps, v1)], f, overlap, bind=False)
    streams = [torch.cuda.Stream(device=dev()) for _ in lps]
    orig = fused_outputs(pa, xs, gs, f, streams)
    for r, p in enumerate(pa):
        p.bind_values()
        with torch.cuda.stream(streams[r]):
            p.set_values(torch.from_numpy(v1[r]).to(dev()))
    got = fused_outputs(pa, xs, gs, f, streams)
    want = fused_outputs(pb, xs, gs, f, streams)
    for r in range(len(lps)):
        for name, a, b in zip(("forward", "backward", "relu forward"), got[r], want[r]):
            assert torch.equal(a, b), "%s f=%d overlap=%d rank %d: %s differs from a plan created with the values" % (
                case, f, overlap, r, name)
    for r, p in enumerate(pa):
        with torch.cuda.stream(streams[r]):
            p.set_values(None)
    back = fused_outputs(pa, xs, gs, f, streams)
    for r in range(len(lps)):
        for a, b in zip(back[r], orig[r]):
            assert torch.equal(a, b), "%s f=%d rank %d: set_values(None) does not restore the creation values" % (case, f, r)
    for p in pa + pb:
        p.close()


def sddmm_truth(lp, gZ, Hcat):
    rows = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
    cols = lp.colidx.astype(np.int64)
    a, b = gZ.astype(np.float64)[rows], Hcat.astype(np.float64)[cols]
    return (a * b).sum(1), (np.abs(a) * np.abs(b)).sum(1)


@pytest.mark.parametrize("case,overlap", CASES)
@pytest.mark.parametrize("f", [16, 40, 128, 256, 384, 512])
def test_sddmm_within_fp32_bound_and_deterministic(case, overlap, f):
    lps, H, G, xs, gs = setup_case(case, f, overlap)
    plans = linked_plans(lps, f, overlap, bind=False)
    streams = [torch.cuda.Stream(device=dev()) for _ in lps]
    lib = cabi.load()

    def one(r):
        p, lp = plans[r], lps[r]
        z = torch.empty_like(xs[r])
        halo = torch.full((lp.h, f), float("nan"), device=dev())
        cabi.check(lib.pgcn_forward_keep_halo(p.handle, xs[r].data_ptr(), z.data_ptr(), halo.data_ptr() if lp.h else None,
                                              f, stream()), p.handle)
        d = []
        for _ in range(2):
            dv = torch.empty(lp.nnz(), device=dev())
            cabi.check(lib.pgcn_sddmm(p.handle, gs[r].data_ptr(), xs[r].data_ptr(), halo.data_ptr() if lp.h else None,
                                      dv.data_ptr(), f, stream()), p.handle)
            d.append(dv)
        return halo, d
    out = run_ranks(plans, one, streams)
    for r, lp in enumerate(lps):
        halo, (d1, d2) = out[r]
        if lp.h:
            assert torch.equal(halo.cpu(), torch.from_numpy(H[lp.halo])), "kept halo rows differ from the sent rows"
        assert torch.equal(d1, d2), "SDDMM is not run-to-run identical"
        truth, mag = sddmm_truth(lp, G[lp.owned], np.concatenate([H[lp.owned], H[lp.halo]], 0))
        err = np.abs(d1.cpu().numpy().astype(np.float64) - truth)
        tol = 2.0 * (f + 2) * 2.0 ** -24 * mag + 1e-30
        assert (err <= tol).all(), "%s f=%d rank %d: %d edges beyond the fp32 dot bound" % (case, f, r, int((err > tol).sum()))
    for p in plans:
        p.close()


@pytest.mark.parametrize("layout", ["local", "global"])
@pytest.mark.parametrize("case,f", [("gemat11_k1", 40), ("rmat", 128), ("rmat", 256)])
def test_weighted_layers_gradients(case, f, layout):
    A, pv, _ = problem(case)
    n = A.shape[0]
    plan = planmod.build_plan(A, pv, 0, 1, f, device=dev())
    plan.layout = layout
    plan.bind_values()
    lp = plan.lp
    rs = np.random.RandomState(f)
    v1n, v2n = new_values(lp, 1), new_values(lp, 2)
    Hn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Gn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    v1 = torch.from_numpy(v1n).to(dev()).requires_grad_(True)
    v2 = torch.from_numpy(v2n).to(dev()).requires_grad_(True)
    x = torch.from_numpy(Hn).to(dev()).requires_grad_(True)
    z1 = PSpMMWeighted.apply(plan, v1, x)
    z2 = PSpMMWeighted.apply(plan, v2, z1)
    z2.backward(torch.from_numpy(Gn).to(dev()))
    # fp64 reference (one rank: local ids are global ids)
    A1 = sp.csr_matrix((v1n.astype(np.float64), lp.colidx, lp.rowptr), shape=(n, n))
    A2 = sp.csr_matrix((v2n.astype(np.float64), lp.colidx, lp.rowptr), shape=(n, n))
    H64, G64 = Hn.astype(np.float64), Gn.astype(np.float64)
    Z1 = A1 @ H64
    Z2 = A2 @ Z1
    G1 = A2.T @ G64
    dH = A1.T @ G1
    rows = np.repeat(np.arange(n), np.diff(lp.rowptr.astype(np.int64)))
    cols = lp.colidx.astype(np.int64)
    dv2 = (G64[rows] * Z1[cols]).sum(1)
    dv1 = (G1[rows] * H64[cols]).sum(1)
    for got, want, what in ((z2, Z2, "Z"), (x.grad, dH, "dH"), (v2.grad, dv2, "dvals layer 2"), (v1.grad, dv1, "dvals layer 1")):
        g = got.detach().cpu().numpy().astype(np.float64)
        np.testing.assert_allclose(g, want, rtol=2e-4, atol=2e-4 * (np.abs(want).max() + 1e-30), err_msg=what)
    plan.close()


def test_psmm_after_weighted_call_equals_fresh_plan():
    A, pv, _ = problem("rmat")
    n, f = A.shape[0], 128
    plan = planmod.build_plan(A, pv, 0, 1, f, device=dev())
    fresh = planmod.build_plan(A, pv, 0, 1, f, device=dev())
    plan.bind_values()
    rs = np.random.RandomState(3)
    x = torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev())
    g = torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev())
    v = torch.from_numpy(new_values(plan.lp, 9)).to(dev()).requires_grad_(True)
    xw = x.clone().requires_grad_(True)
    PSpMMWeighted.apply(plan, v, xw).backward(g)
    for p in (plan, fresh):
        xp = x.clone().requires_grad_(True)
        z = PSpMM.apply(p, xp)
        z.backward(g)
        p._out = (z.detach(), xp.grad)
    assert torch.equal(plan._out[0], fresh._out[0]) and torch.equal(plan._out[1], fresh._out[1])
    plan.close(); fresh.close()


def test_set_values_before_bind_is_refused():
    A, pv, _ = problem("gemat11_k1")
    plan = planmod.build_plan(A, pv, 0, 1, 16, device=dev())
    ones = torch.ones(plan.lp.nnz(), device=dev())
    with pytest.raises(RuntimeError, match="pgcn_plan_bind_values"):
        plan.set_values(ones)
    with pytest.raises(RuntimeError, match="bind_values"):         # the op does no set-up work on its own
        PSpMMWeighted.apply(plan, ones, torch.ones((plan.m, 16), device=dev()))
    plan.close()


@pytest.mark.parametrize("f", [40, 128])
def test_sddmm_capture_before_prepare_is_refused(f):
    A, pv, _ = problem("rmat")
    n = A.shape[0]
    plan = planmod.build_plan(A, pv, 0, 1, f, device=dev())
    lib = cabi.load()
    rs = np.random.RandomState(2)
    gz = torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev())
    x = torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev())
    dv = torch.empty(plan.lp.nnz(), device=dev())
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    call = lambda: cabi.check(lib.pgcn_sddmm(plan.handle, gz.data_ptr(), x.data_ptr(), None, dv.data_ptr(), f, stream()),
                              plan.handle)
    with pytest.raises(RuntimeError, match="pgcn_plan_prepare"):
        with torch.cuda.graph(graph, stream=s):
            call()
    with torch.cuda.stream(s):                      # the capture was not invalidated: plan and stream still work
        call()
    s.synchronize()
    truth, mag = sddmm_truth(plan.lp, gz.cpu().numpy(), x.cpu().numpy())
    assert (np.abs(dv.cpu().numpy() - truth) <= 2.0 * (f + 2) * 2.0 ** -24 * mag + 1e-30).all()
    plan.close()


def global_values(lps, vals):
    """The n x n fp64 matrix whose rank-r rows hold vals[r] at the global (row, column) of each local entry."""
    rows, cols, data = [], [], []
    for lp, v in zip(lps, vals):
        gcol = np.concatenate([lp.owned, lp.halo])
        rows.append(lp.owned[np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))])
        cols.append(gcol[lp.colidx.astype(np.int64)])
        data.append(v.astype(np.float64))
    n = lps[0].n
    return sp.csr_matrix((np.concatenate(data), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


@pytest.mark.parametrize("case,f,overlap", [("gemat11_k2", 40, 1), ("gemat11_k2", 128, 0), ("rmat_k2", 128, 1),
                                            ("gemat11_k3_hp", 256, 1)])
def test_multi_rank_weighted_layers_gradients(case, f, overlap):
    """PSpMMWeighted on k > 1 ranks over the peer transport, each rank on its own stream: two layers with different
    values on one plan per rank; Z, dH (every peer's contribution summed) and dvals (halo columns from the kept halo
    rows) against fp64."""
    A, pv, k = problem(case)
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(f + k)
    Hn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Gn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    v1n = [new_values(lp, 200 + r) for r, lp in enumerate(lps)]
    v2n = [new_values(lp, 300 + r) for r, lp in enumerate(lps)]
    x = [torch.from_numpy(Hn[lp.owned]).to(dev()).requires_grad_(True) for lp in lps]
    v1 = [torch.from_numpy(v).to(dev()).requires_grad_(True) for v in v1n]
    v2 = [torch.from_numpy(v).to(dev()).requires_grad_(True) for v in v2n]
    g = [torch.from_numpy(Gn[lp.owned]).to(dev()) for lp in lps]
    z1 = run_ranks(plans, lambda r: PSpMMWeighted.apply(plans[r], v1[r], x[r]), streams)
    z2 = run_ranks(plans, lambda r: PSpMMWeighted.apply(plans[r], v2[r], z1[r]), streams)
    run_ranks(plans, lambda r: z2[r].backward(g[r]), streams)
    A1, A2 = global_values(lps, v1n), global_values(lps, v2n)
    H64, G64 = Hn.astype(np.float64), Gn.astype(np.float64)
    Z1 = A1 @ H64
    Z2 = A2 @ Z1
    G1 = A2.T @ G64
    dH = A1.T @ G1
    for r, lp in enumerate(lps):
        gcol = np.concatenate([lp.owned, lp.halo])
        rows = lp.owned[np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))]
        cols = gcol[lp.colidx.astype(np.int64)]
        dv2 = (G64[rows] * Z1[cols]).sum(1)
        dv1 = (G1[rows] * H64[cols]).sum(1)
        for got, want, what in ((z2[r], Z2[lp.owned], "Z"), (x[r].grad, dH[lp.owned], "dH"),
                                (v2[r].grad, dv2, "dvals layer 2"), (v1[r].grad, dv1, "dvals layer 1")):
            u = got.detach().cpu().numpy().astype(np.float64)
            np.testing.assert_allclose(u, want, rtol=2e-4, atol=2e-4 * (np.abs(want).max() + 1e-30),
                                       err_msg="%s f=%d overlap=%d rank %d: %s" % (case, f, overlap, r, what))
    for p in plans:
        assert p.stats["send_volume"] == 2 * p.lp.S + 2 * p.lp.h    # two forward and two backward exchanges counted
        p.close()


def test_bind_rejects_a_mismatched_transpose():
    A, pv, _ = problem("gemat11_k1")
    lp = planmod.build_local_plan(A, pv, 0, 1)
    t = lp.t_colidx.copy()
    row0 = t[lp.t_rowptr[0]:lp.t_rowptr[1]]
    t[lp.t_rowptr[0]] = (int(row0.max()) + 1) % lp.m          # an entry the forward CSR does not have
    lp.t_colidx = t
    plan = planmod.PgcnPlan(lp, 16, device=dev())
    with pytest.raises(RuntimeError, match="does not hold the forward entries"):
        plan.bind_values()
    plan.close()


def test_one_rank_capture_of_weighted_layers():
    A, pv, _ = problem("rmat")
    n, f = A.shape[0], 128
    plan = planmod.build_plan(A, pv, 0, 1, f, device=dev())
    plan.prepare(f)
    plan.bind_values()
    rs = np.random.RandomState(11)
    ins = [(torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev()),
            torch.from_numpy(rs.uniform(-1, 1, size=(n, f)).astype(np.float32)).to(dev()),
            torch.from_numpy(new_values(plan.lp, 20 + i)).to(dev()),
            torch.from_numpy(new_values(plan.lp, 40 + i)).to(dev())) for i in range(3)]
    x = torch.zeros((n, f), device=dev(), requires_grad=True)
    g = torch.zeros((n, f), device=dev())
    v1 = torch.zeros(plan.lp.nnz(), device=dev(), requires_grad=True)
    v2 = torch.zeros(plan.lp.nnz(), device=dev(), requires_grad=True)

    def step():
        z = PSpMMWeighted.apply(plan, v2, PSpMMWeighted.apply(plan, v1, x))
        z.backward(g)
        return dict(Z=z, dH=x.grad, dv1=v1.grad, dv2=v2.grad)

    def load(i):
        with torch.no_grad():
            for u, w in zip((x, g, v1, v2), ins[i]):
                u.copy_(w)

    def eager(i):
        xi, gi, a, b = ins[i]
        xe, ae, be = (u.clone().requires_grad_(True) for u in (xi, a, b))
        ze = PSpMMWeighted.apply(plan, be, PSpMMWeighted.apply(plan, ae, xe))
        ze.backward(gi)
        PSpMM.apply(plan, xi)                                      # the creation values in between
        return dict(Z=ze, dH=xe.grad, dv1=ae.grad, dv2=be.grad)

    check_one_rank_capture(plan, step, load, eager)
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f = 128
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1, bind=False)
    for p in plans:
        p.prepare(f)
        p.bind_values()
    lib = cabi.load()
    n = A.shape[0]
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(5)
    ins = [(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.uniform(-1, 1, size=(n, f)).astype(np.float32),
            [new_values(lp, 60 + 2 * i) for lp in lps], [new_values(lp, 61 + 2 * i) for lp in lps]) for i in range(3)]

    def buffers(r):
        lp = lps[r]
        m, h, nnz = lp.m, lp.h, lp.nnz()
        return dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()),
                    v1=torch.zeros(nnz, device=dev()), v2=torch.zeros(nnz, device=dev()),
                    z1=torch.zeros((m, f), device=dev()), z2=torch.zeros((m, f), device=dev()),
                    h1=torch.zeros((max(h, 1), f), device=dev()), h2=torch.zeros((max(h, 1), f), device=dev()),
                    g1=torch.zeros((m, f), device=dev()), g0=torch.zeros((m, f), device=dev()),
                    d1=torch.zeros(nnz, device=dev()), d2=torch.zeros(nnz, device=dev()))

    def step(r, b):
        p = plans[r]
        hd, st = p.handle, stream()
        chk = lambda rc: cabi.check(rc, hd)
        chk(lib.pgcn_plan_set_values(hd, b["v1"].data_ptr(), st))
        chk(lib.pgcn_forward_keep_halo(hd, b["x"].data_ptr(), b["z1"].data_ptr(), b["h1"].data_ptr(), f, st))
        chk(lib.pgcn_plan_set_values(hd, b["v2"].data_ptr(), st))
        chk(lib.pgcn_forward_keep_halo(hd, b["z1"].data_ptr(), b["z2"].data_ptr(), b["h2"].data_ptr(), f, st))
        chk(lib.pgcn_backward(hd, b["g"].data_ptr(), b["g1"].data_ptr(), f, st))
        chk(lib.pgcn_sddmm(hd, b["g"].data_ptr(), b["z1"].data_ptr(), b["h2"].data_ptr(), b["d2"].data_ptr(), f, st))
        chk(lib.pgcn_plan_set_values(hd, b["v1"].data_ptr(), st))
        chk(lib.pgcn_backward(hd, b["g1"].data_ptr(), b["g0"].data_ptr(), f, st))
        chk(lib.pgcn_sddmm(hd, b["g1"].data_ptr(), b["x"].data_ptr(), b["h1"].data_ptr(), b["d1"].data_ptr(), f, st))
        return {o: b[o] for o in ("z2", "g0", "d1", "d2")}

    def load(bufs, i):
        H, G, a, c = ins[i]
        for r, lp in enumerate(lps):
            bufs[r]["x"].copy_(torch.from_numpy(H[lp.owned])); bufs[r]["g"].copy_(torch.from_numpy(G[lp.owned]))
            bufs[r]["v1"].copy_(torch.from_numpy(a[r])); bufs[r]["v2"].copy_(torch.from_numpy(c[r]))
        torch.cuda.synchronize()

    check_two_rank_capture(plans, streams, buffers, load, step)
    assert plans[0].get_option("epoch") % 2 == 1
    for p in plans:
        p.close()
