"""GATv2 attention on the H100 path: pgcn_forward_gatv2, pgcn_backward_gatv2, op.PGATv2Attention and PGAT.py --v2.

  * alpha, Z, dxl, dxr and datt lie within a per-entry fp32 bound of the fp64 formulas (tests/gatv2_oracle.py) on
    gemat11, a hub graph (a row over 1 024 entries, empty rows, rows of one entry, split rows) and a matrix with
    duplicated entries, for f in {8, 16, 40, 128, 256}, every K that divides f and slopes 0.2 and 1.0;
  * two runs give the same bits; the ring and plain score kernels give the same bits (an operand 4 bytes into its
    buffer), and so do the 4-wide and scalar backward kernels;
  * att = 0 gives the neighbour mean of xl, and slope 1.0 gives dxr = 0 (exact identities, within the bound);
  * 2 and 3 ranks with overlap 0 and 1 match fp64 on every rank, and the returned halo rows are the owners' rows;
  * autograd in both layouts and with XL is XR; CUDA-graph capture on one and two ranks; refusals;
  * PGAT.py --v2 follows the fp64 loss curve, and PGAT.py without --v2 prints what it printed before.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import gatv2_oracle as go
import harness
from harness import (EPS, assert_follows, check_one_rank_capture, check_two_rank_capture, dev, edges, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PGATv2Attention

pytestmark = pytest.mark.gpu
PGCN_ERR_INVALID, PGCN_ERR_STATE = -1, -5


def dup_graph():
    """400 vertices, every stored entry twice or three times (the copies are separate entries)."""
    rs = np.random.RandomState(4)
    row = rs.randint(0, 400, 3000)
    col = rs.randint(0, 400, 3000)
    row = np.concatenate([row, row, row[:1000]])
    col = np.concatenate([col, col, col[:1000]])
    return sp.coo_matrix((np.ones(len(row), np.float32), (row, col)), shape=(400, 400))


def one_rank_plan(case, f):
    """The harness's one-rank plan, or one of dup_graph() (a case of this file only)."""
    if case != "dup":
        return harness.one_rank_plan(case, f)
    A = dup_graph()
    plan = planmod.build_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1, f, device=dev())
    plan.bind_values()
    return A, plan


def gatv2_run(plan, K, xl, xr, att, gZ, slope):
    """(alpha, Z, dxl, dxr, datt) of the C-ABI calls on one rank."""
    lib = cabi.load()
    lp = plan.lp
    f = xl.shape[1]
    alpha = torch.full((lp.nnz(), K), float("nan"), device=dev())
    Z = torch.full((lp.m, f), float("nan"), device=dev())
    cabi.check(lib.pgcn_forward_gatv2(plan.handle, K, xl.data_ptr(), xr.data_ptr(), att.data_ptr(), slope,
                                      alpha.data_ptr(), Z.data_ptr(), None, f, stream()), plan.handle)
    work = torch.full_like(alpha, float("nan"))
    dxl, dxr = torch.full_like(Z, float("nan")), torch.full_like(Z, float("nan"))
    datt = torch.full((K, f // K), float("nan"), device=dev())
    cabi.check(lib.pgcn_backward_gatv2(plan.handle, K, alpha.data_ptr(), gZ.data_ptr(), xl.data_ptr(), None,
                                       xr.data_ptr(), att.data_ptr(), slope, work.data_ptr(), dxl.data_ptr(),
                                       dxr.data_ptr(), datt.data_ptr(), f, stream()), plan.handle)
    torch.cuda.synchronize()
    return [u.cpu().numpy() for u in (alpha, Z, dxl, dxr, datt)]


def bounds(rows, cols, n, xl, xr, att, slope, gZ, alpha32):
    """fp64 values and per-entry fp32 bounds: the forward from the fp32 inputs, the backward from the kernel's alpha
    (so that each bound covers one call's rounding). A bound is EPS times the operation count of the longest chain
    times the same computation over absolute values."""
    K, d = att.shape
    deg = np.bincount(rows, minlength=n)
    cdeg = np.bincount(cols, minlength=n)
    Z64, a64, s64 = go.forward(rows, cols, n, xl, xr, att, slope)
    xl, xr, att, gZ = (np.asarray(x, np.float64) for x in (xl, xr, att, gZ))
    T = np.abs(xl[cols]) + np.abs(xr[rows])
    ds = EPS * (d + 8) * (T.reshape(-1, K, d) * np.abs(att)[None]).sum(2)        # score rounding, per entry and head
    dmax = np.zeros((n, K))
    np.maximum.at(dmax, rows, ds)
    smax = np.zeros((n, K))
    np.maximum.at(smax, rows, np.abs(s64))
    ta = a64 * (2 * ds + 2 * dmax[rows] + EPS * (8 * smax[rows] + 4 * deg[rows, None] + 32)) + 1e-38
    tZ = np.zeros((n, K * d))
    P = np.repeat(a64, d, 1) * np.abs(xl[cols])
    np.add.at(tZ, rows, np.repeat(ta, d, 1) * np.abs(xl[cols]) + EPS * (deg[rows, None] + 4) * P)
    a = np.asarray(alpha32, np.float64)
    dxl, dxr, datt, _, _ = go.backward(rows, cols, n, xl, xr, att, slope, a, gZ)
    Md = (np.abs(gZ[rows]) * np.abs(xl[cols])).reshape(-1, K, d).sum(2)
    Mc = np.zeros((n, K))
    np.add.at(Mc, rows, a * Md)
    Ms = np.repeat(a * (Md + Mc[rows]), d, 1)
    Mg = Ms * np.abs(att).reshape(1, -1) * np.where(xl[cols] + xr[rows] > 0, 1.0, slope)
    Mxr = np.zeros((n, K * d))
    np.add.at(Mxr, rows, Mg)
    Mxl = np.zeros((n, K * d))
    np.add.at(Mxl, cols, np.repeat(a, d, 1) * np.abs(gZ[rows]) + Mg)
    Mat = (Ms * T).sum(0).reshape(K, d)
    chain = 2 * (d + deg.max() + 32)
    tol = dict(dxr=EPS * chain * Mxr + 1e-30, dxl=EPS * 2 * (chain + cdeg.max()) * Mxl + 1e-30,
               datt=EPS * (2 * chain + 1024 + len(rows) // 256) * Mat + 1e-30)
    return dict(alpha=(a64, ta), Z=(Z64, tZ), dxl=(dxl, tol["dxl"]), dxr=(dxr, tol["dxr"]), datt=(datt, tol["datt"]))


def check(got, ref, names=("alpha", "Z", "dxl", "dxr", "datt"), what=""):
    for name, u in zip(names, got):
        want, tol = ref[name]
        err = np.abs(u.astype(np.float64) - want)
        assert np.isfinite(u).all() and (err <= tol).all(), \
            "%s%s: %d entries beyond the bound, worst %g" % (what, name, (err > tol).sum(), (err - tol).max())


def inputs(rs, n, f, K, scale=1.0):
    xl = rs.uniform(-scale, scale, (n, f)).astype(np.float32)
    xr = rs.uniform(-scale, scale, (n, f)).astype(np.float32)
    att = (rs.standard_normal((K, f // K)) / np.sqrt(f // K)).astype(np.float32)
    gZ = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    return xl, xr, att, gZ


CASES = [(f, K) for f in (8, 16, 40, 128, 256) for K in (1, 2, 4, 8) if f % K == 0]


@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
@pytest.mark.parametrize("f,K", CASES)
@pytest.mark.parametrize("slope", [0.2, 1.0])
def test_against_fp64_and_deterministic(case, f, K, slope):
    A, plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > 1024 and (deg == 0).any() and (deg == 1).any()
    rs = np.random.RandomState(f * 10 + K + int(slope * 10))
    xl, xr, att, gZ = inputs(rs, lp.m, f, K)
    runs = [gatv2_run(plan, K, t(xl), t(xr), t(att), t(gZ), slope) for _ in range(2)]
    for a, b in zip(*runs):
        assert np.array_equal(a, b, equal_nan=True), "not run-to-run identical"
    rows, cols = edges(lp)
    check(runs[0], bounds(rows, cols, lp.m, xl, xr, att, slope, gZ, runs[0][0]), what="%s f=%d K=%d: " % (case, f, K))
    deg = np.diff(lp.rowptr.astype(np.int64))
    assert np.all(runs[0][1][deg == 0] == 0)
    plan.close()


@pytest.mark.parametrize("f,K", [(128, 1), (128, 2), (128, 4), (128, 8), (256, 1), (256, 2), (256, 4), (256, 8),
                                 (16, 4), (40, 2)])
def test_ring_and_plain_scores_and_vector_widths_give_the_same_bits(f, K):
    """Shifting an operand 4 bytes sends the scores to the plain kernel and the backward to the scalar instances."""
    A, plan = one_rank_plan("hub", f)
    lp = plan.lp
    rs = np.random.RandomState(f + K)
    xl, xr, att, gZ = (t(x) for x in inputs(rs, lp.m, f, K))
    base = gatv2_run(plan, K, xl, xr, att, gZ, 0.2)
    for which in range(3):
        ops = [xl, xr, att]
        ops[which] = shifted(ops[which])
        got = gatv2_run(plan, K, ops[0], ops[1], ops[2], gZ, 0.2)
        # a shifted xl also moves pgcn_sddmm_heads (dalpha) to its plain instance, which sums in another order: the
        # backward is compared when xr or att is shifted (the backward walks then take their scalar instances)
        names = ("alpha", "Z") if which == 0 else ("alpha", "Z", "dxl", "dxr", "datt")
        for name, a, b in zip(names, base, got):
            assert np.array_equal(a, b), "operand %d shifted: %s differs" % (which, name)
    plan.close()


@pytest.mark.parametrize("f,K", [(40, 4), (128, 8), (256, 1)])
def test_exact_identities(f, K):
    A, plan = one_rank_plan("hub", f)
    lp = plan.lp
    rows, cols = edges(lp)
    rs = np.random.RandomState(7)
    xl, xr, att, gZ = inputs(rs, lp.m, f, K)
    # att = 0: every score is 0, alpha = 1 / degree and Z is the neighbour mean of xl
    zero = np.zeros_like(att)
    alpha, Z, _, _, _ = gatv2_run(plan, K, t(xl), t(xr), t(zero), t(gZ), 0.2)
    deg = np.bincount(rows, minlength=lp.m)
    mean = np.zeros((lp.m, f))
    np.add.at(mean, rows, xl[cols].astype(np.float64))
    mean /= np.maximum(deg, 1)[:, None]
    mag = np.zeros((lp.m, f))
    np.add.at(mag, rows, np.abs(xl[cols]).astype(np.float64))
    assert np.array_equal(alpha, np.repeat((np.float32(1) / deg[rows].astype(np.float32))[:, None], K, 1))
    assert (np.abs(Z - mean) <= EPS * (deg[:, None] + 8) * mag / np.maximum(deg, 1)[:, None] + 1e-30).all()
    # slope 1: the score is att . (xl + xr), whose xr part is constant over a row and cancels in the softmax, so
    # dxr = sum_row dscore * att = 0 (sum_row dscore = 0 per head)
    got = gatv2_run(plan, K, t(xl), t(xr), t(att), t(gZ), 1.0)
    ref = bounds(rows, cols, lp.m, xl, xr, att, 1.0, gZ, got[0])
    assert (np.abs(got[3]) <= ref["dxr"][1]).all(), "slope 1: dxr is not zero within the bound"
    plan.close()


def global_edges(A):
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    C = C.tocoo()
    return C.row.astype(np.int64), C.col.astype(np.int64)


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("case,f,K", [("gemat11_k2", 40, 2), ("gemat11_k2", 128, 8), ("gemat11_k3_hp", 256, 4),
                                      ("gemat11_k3_hp", 16, 1)])
def test_multi_rank(case, f, K, overlap):
    A, pv, k = problem(case)
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(f + k + K)
    xl, xr, att, gZ = inputs(rs, n, f, K)
    lib = cabi.load()
    bufs = []

    def fwd(r):
        lp = lps[r]
        b = dict(xl=t(xl[lp.owned]), xr=t(xr[lp.owned]), att=t(att), g=t(gZ[lp.owned]),
                 alpha=torch.empty((lp.nnz(), K), device=dev()), Z=torch.empty((lp.m, f), device=dev()),
                 halo=torch.full((lp.h, f), float("nan"), device=dev()))
        cabi.check(lib.pgcn_forward_gatv2(plans[r].handle, K, b["xl"].data_ptr(), b["xr"].data_ptr(),
                                          b["att"].data_ptr(), 0.2, b["alpha"].data_ptr(), b["Z"].data_ptr(),
                                          b["halo"].data_ptr(), f, stream()), plans[r].handle)
        bufs.append(b)

    def bwd(r):
        lp, b = lps[r], bufs[r]
        for name in ("work", "dxl", "dxr"):
            b[name] = torch.empty_like(b["alpha"] if name == "work" else b["Z"])
        b["datt"] = torch.empty((K, f // K), device=dev())
        cabi.check(lib.pgcn_backward_gatv2(plans[r].handle, K, b["alpha"].data_ptr(), b["g"].data_ptr(),
                                           b["xl"].data_ptr(), b["halo"].data_ptr(), b["xr"].data_ptr(),
                                           b["att"].data_ptr(), 0.2, b["work"].data_ptr(), b["dxl"].data_ptr(),
                                           b["dxr"].data_ptr(), b["datt"].data_ptr(), f, stream()), plans[r].handle)

    run_ranks(plans, fwd, streams)
    run_ranks(plans, bwd, streams)
    rows, cols = global_edges(A)
    Z64, a64, _ = go.forward(rows, cols, n, xl, xr, att, 0.2)
    ref = bounds(rows, cols, n, xl, xr, att, 0.2, gZ, a64)
    datt = sum(b["datt"].cpu().numpy().astype(np.float64) for b in bufs)
    for r, lp in enumerate(lps):
        w = "%s f=%d K=%d overlap=%d rank %d: " % (case, f, K, overlap, r)
        b = bufs[r]
        assert torch.equal(b["halo"].cpu(), torch.from_numpy(xl[lp.halo])), w + "halo rows of xl"
        for name in ("Z", "dxl", "dxr"):
            want, tol = ref[name]
            # alpha is rounded differently here than in the reference's backward: allow its bound once more
            slack = ref["Z"][1][lp.owned] if name == "Z" else 2 * tol[lp.owned] + 64 * EPS * np.abs(want[lp.owned])
            err = np.abs(b[name].cpu().numpy() - want[lp.owned])
            assert (err <= slack + (tol[lp.owned] if name == "Z" else 0) + 1e-30).all(), w + name
    want, tol = ref["datt"]
    assert (np.abs(datt - want) <= 2 * tol + 64 * EPS * np.abs(want) * k).all(), "datt summed over ranks"
    for p in plans:
        p.close()


def layer64(rows, cols, n, xl, xr, att, slope):
    return go.forward_torch(torch.from_numpy(rows), torch.from_numpy(cols), n, xl, xr, att, slope)


def close(got, want, mag, what):
    u = got.detach().cpu().numpy().astype(np.float64)
    assert (np.abs(u - want) <= 4096 * EPS * mag + 1e-30).all(), what


@pytest.mark.parametrize("layout", ["local", "global"])
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("f,K", [(16, 2), (128, 4), (256, 8)])
def test_autograd(f, K, layout, shared):
    A, plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp, n = plan.lp, A.shape[0]
    rs = np.random.RandomState(f + K)
    H = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    G = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    Wl = (rs.standard_normal((f, f)) / np.sqrt(f)).astype(np.float32)
    Wr = Wl if shared else (rs.standard_normal((f, f)) / np.sqrt(f)).astype(np.float32)
    att = (rs.standard_normal((K, f // K)) / np.sqrt(f // K)).astype(np.float32)
    Wlt, att_t = t(Wl).requires_grad_(True), t(att).requires_grad_(True)
    Wrt = Wlt if shared else t(Wr).requires_grad_(True)
    XL = t(H) @ Wlt.T
    XR = XL if shared else t(H) @ Wrt.T
    out = PGATv2Attention.apply(plan, XL, XR, att_t, 0.2)
    out.backward(t(G))
    W64l = torch.tensor(Wl, dtype=torch.float64, requires_grad=True)
    W64r = W64l if shared else torch.tensor(Wr, dtype=torch.float64, requires_grad=True)
    a64 = torch.tensor(att, dtype=torch.float64, requires_grad=True)
    H64 = torch.from_numpy(H.astype(np.float64))
    XL64 = H64 @ W64l.T
    XR64 = XL64 if shared else H64 @ W64r.T
    rows, cols = edges(lp)
    o64 = layer64(rows, cols, n, XL64, XR64, a64, 0.2)
    o64.backward(torch.from_numpy(G.astype(np.float64)))
    # magnitudes: the same computation over absolute values
    HA = torch.from_numpy(np.abs(H).astype(np.float64))
    mag_o = layer64(rows, cols, n, HA @ W64l.detach().abs().T, HA @ W64r.detach().abs().T, a64.detach().abs(), 0.2)
    mo = mag_o.numpy().max(1, keepdims=True) + np.abs(o64.detach().numpy())
    close(out, o64.detach().numpy(), mo, "out")
    # dW = dX^T H: the per-entry bounds of dxl and dxr (bounds(), which also cover cancellation inside a row) through
    # |H|, plus the rounding of the product's own sum
    XLn, XRn = (x.detach().numpy() for x in (XL64, XR64))
    a_ref = go.forward(rows, cols, n, XLn, XRn, att, 0.2)[1]
    ref = bounds(rows, cols, n, XLn, XRn, att, 0.2, G, a_ref)
    Ha = np.abs(H).astype(np.float64)
    wtol = lambda name: 4 * ref[name][1].T @ Ha + EPS * (n + 8) * (np.abs(ref[name][0]).T @ Ha) + 1e-30
    gl, gr = (w.grad.numpy() for w in (W64l, W64r))
    if shared:
        close(Wlt.grad, gl, np.abs(gl).max() + np.abs(gl), "dW")
    else:
        for got, want, name in ((Wlt.grad, gl, "dxl"), (Wrt.grad, gr, "dxr")):
            err = np.abs(got.detach().cpu().numpy() - want)
            assert (err <= wtol(name) + 64 * EPS * f * np.abs(want)).all(), "dW from " + name
    ga = a64.grad.numpy()
    close(att_t.grad, ga, np.abs(ga).max() + np.abs(ga), "datt")
    plan.close()


def step(plan, x, Wl, Wr, att, g):
    out = PGATv2Attention.apply(plan, x @ Wl.T, x @ Wr.T, att, 0.2)
    out.backward(g)
    return out


def test_one_rank_capture_and_refusals():
    A, plan = one_rank_plan("hub", 128)
    f, n, K = 128, A.shape[0], 4
    lib = cabi.load()
    # an unbound plan
    unbound = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    z = torch.zeros((n, f), device=dev())
    rc = lib.pgcn_forward_gatv2(unbound.handle, K, z.data_ptr(), z.data_ptr(), z.data_ptr(), 0.2, z.data_ptr(),
                                z.data_ptr(), None, f, stream())
    assert rc == PGCN_ERR_STATE
    unbound.close()
    for heads, ff in ((3, f), (0, f), (16, f), (8, 36)):
        assert lib.pgcn_forward_gatv2(plan.handle, heads, z.data_ptr(), z.data_ptr(), z.data_ptr(), 0.2, z.data_ptr(),
                                      z.data_ptr(), None, ff, stream()) == PGCN_ERR_INVALID
    assert lib.pgcn_forward_gatv2(plan.handle, K, z.data_ptr(), z.data_ptr(), None, 0.2, z.data_ptr(), z.data_ptr(),
                                  None, f, stream()) == PGCN_ERR_INVALID
    rs = np.random.RandomState(11)
    rnd = lambda *s: t(rs.uniform(-1, 1, size=s).astype(np.float32))
    x, g = torch.zeros((n, f), device=dev()), torch.zeros((n, f), device=dev())
    Wl = torch.zeros((f, f), device=dev(), requires_grad=True)
    Wr = torch.zeros((f, f), device=dev(), requires_grad=True)
    att = torch.zeros((K, f // K), device=dev(), requires_grad=True)
    ins = [(rnd(n, f), rnd(n, f), rnd(f, f) * 0.1, rnd(f, f) * 0.1, rnd(K, f // K)) for _ in range(3)]

    def load(i):
        with torch.no_grad():
            for u, v in zip((x, g, Wl, Wr, att), ins[i]):
                u.copy_(v)

    def eager(i):
        xi, gi, Wli, Wri, ai = ins[i]
        e = [u.clone().requires_grad_(True) for u in (Wli, Wri, ai)]
        oe = step(plan, xi, e[0], e[1], e[2], gi)
        return dict(out=oe, dWl=e[0].grad, dWr=e[1].grad, datt=e[2].grad)

    check_one_rank_capture(plan, lambda: dict(out=step(plan, x, Wl, Wr, att, g), dWl=Wl.grad, dWr=Wr.grad,
                                              datt=att.grad), load, eager, prepare=(f,), leaves=(Wl, Wr, att))
    plan.close()


def test_two_rank_capture():
    A, pv, k = problem("gemat11_k2")
    f, n, K = 128, A.shape[0], 8
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(5)
    ins = [tuple(rs.uniform(-1, 1, size=s).astype(np.float32) for s in ((n, f), (n, f), (f, f), (f, f), (K, f // K)))
           for _ in range(3)]

    def buffers(r):
        m = lps[r].m
        return dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()),
                    Wl=torch.zeros((f, f), device=dev(), requires_grad=True),
                    Wr=torch.zeros((f, f), device=dev(), requires_grad=True),
                    att=torch.zeros((K, f // K), device=dev(), requires_grad=True))

    def load(bufs, i):
        H, G, Wl, Wr, att = ins[i]
        with torch.no_grad():
            for r, lp in enumerate(lps):
                b = bufs[r]
                b["x"].copy_(torch.from_numpy(H[lp.owned])); b["g"].copy_(torch.from_numpy(G[lp.owned]))
                b["Wl"].copy_(torch.from_numpy(Wl) * 0.1); b["Wr"].copy_(torch.from_numpy(Wr) * 0.1)
                b["att"].copy_(torch.from_numpy(att))
        torch.cuda.synchronize()

    def run(r, b):
        out = step(plans[r], b["x"], b["Wl"], b["Wr"], b["att"], b["g"])
        return dict(out=out, dWl=b["Wl"].grad, dWr=b["Wr"].grad, datt=b["att"].grad)

    check_two_rank_capture(plans, streams, buffers, load, run)
    for p in plans:
        p.close()


def test_cli_v2_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", ["--v2", "--heads", "2"], 29681)
    assert_follows(lines, go.intended_training(karate(), 2, 4, 7, 1.0, heads=2))


def test_cli_without_v2_is_unchanged(tmp_path):
    import pgat_heads_oracle as ho
    lines = run_cli(tmp_path, "PGAT.py", ["--heads", "2"], 29682)
    assert_follows(lines, ho.intended_training(karate(), 2, 4, 7, 1.0, heads=2))
