"""Multi-head sparse graph attention on the H100 path: pgcn_edge_softmax_heads, pgcn_edge_softmax_backward_heads,
pgcn_forward_heads, pgcn_backward_heads, pgcn_sddmm_heads, op.PGATMultiHeadAttention and PGAT.py --heads.

  * the K-head softmax kernels lie within the fp32 bound of fp64 per head (hub rows on the CTA path, empty rows, rows of
    one entry, slopes 0.2 and 1.0, scores near +-80), are run-to-run identical, and K = 1 equals pgcn_edge_softmax(_backward);
  * with every head's alpha equal to the creation values the multi-head aggregation gives the bits of pgcn_forward /
    pgcn_backward on the register kernel; with random alpha it lies within fp32 of fp64, and an operand 4 bytes into its
    buffer gives the aligned bits;
  * pgcn_sddmm_heads against fp64 on the ring instance and the plain path, K = 1 equal to pgcn_sddmm;
  * the operator's output and gradients (Z, el, er, W, a) against fp64 on one rank in both layouts and on 2 and 3 ranks
    with overlap 0 and 1; the plan's resident values are untouched; CUDA-graph capture on one and two ranks;
  * the command line follows the fp64 loss curve with --heads 2, and --heads 1 prints what no flag prints.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import pgat_heads_oracle as ho
from harness import (EPS, assert_follows, check_one_rank_capture, check_two_rank_capture, dev, edges, karate,
                     linked_plans, one_rank_plan, problem, run_cli, run_ranks, shifted, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PGATAttention, PGATMultiHeadAttention, PSpMM

pytestmark = pytest.mark.gpu


def softmax_run(lib, plan, K, el, er, dal, slope):
    lp = plan.lp
    alpha = torch.empty((lp.nnz(), K), device=dev())
    dpre = torch.empty((lp.nnz(), K), device=dev())
    d_el = torch.full((lp.m, K), float("nan"), device=dev())
    cabi.check(lib.pgcn_edge_softmax_heads(plan.handle, K, el.data_ptr(), er.data_ptr(), None, slope, alpha.data_ptr(),
                                           stream()), plan.handle)
    cabi.check(lib.pgcn_edge_softmax_backward_heads(plan.handle, K, el.data_ptr(), er.data_ptr(), None, alpha.data_ptr(),
                                                    dal.data_ptr(), slope, dpre.data_ptr(), d_el.data_ptr(), stream()),
               plan.handle)
    return alpha, dpre, d_el


@pytest.mark.parametrize("case", ["gemat11_k1", "hub"])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("slope", [0.2, 1.0])
@pytest.mark.parametrize("scale", [1.0, 80.0])
def test_softmax_kernels_within_fp32_bound_and_deterministic(case, K, slope, scale):
    A, plan = one_rank_plan(case, 8)
    lp = plan.lp
    deg = np.diff(lp.rowptr.astype(np.int64))
    if case == "hub":
        assert deg.max() > 1024 and (deg == 0).any() and (deg == 1).any()
    rs = np.random.RandomState(int(scale) + int(10 * slope) + K)
    el = rs.uniform(-scale, scale, (lp.m, K)).astype(np.float32)
    er = rs.uniform(-scale, scale, (lp.m, K)).astype(np.float32)
    dal = rs.uniform(-1, 1, (lp.nnz(), K)).astype(np.float32)
    lib = cabi.load()
    runs = [[u.cpu().numpy() for u in softmax_run(lib, plan, K, t(el), t(er), t(dal), slope)] for _ in range(2)]
    for a, b in zip(runs[0], runs[1]):
        assert np.array_equal(a, b), "not run-to-run identical"
    if K == 1:
        ref = []
        alpha = torch.empty(lp.nnz(), device=dev())
        dpre = torch.empty(lp.nnz(), device=dev())
        d_el = torch.full((lp.m,), float("nan"), device=dev())
        e1, r1, d1 = t(el[:, 0]), t(er[:, 0]), t(dal[:, 0])
        cabi.check(lib.pgcn_edge_softmax(plan.handle, e1.data_ptr(), r1.data_ptr(), None, slope, alpha.data_ptr(),
                                         stream()), plan.handle)
        cabi.check(lib.pgcn_edge_softmax_backward(plan.handle, e1.data_ptr(), r1.data_ptr(), None, alpha.data_ptr(),
                                                  d1.data_ptr(), slope, dpre.data_ptr(), d_el.data_ptr(), stream()),
                   plan.handle)
        ref = [alpha, dpre, d_el]
        for got, want in zip(runs[0], ref):
            assert torch.equal(torch.from_numpy(got).reshape(-1), want.cpu()), "K = 1 differs from the single-head kernels"
    rows, cols = edges(lp)
    for h in range(K):
        alpha, dpre, d_el = (x[:, h].astype(np.float64) for x in runs[0])
        s = el[:, h].astype(np.float64)[rows] + er[:, h].astype(np.float64)[cols]
        s = np.where(s > 0, s, slope * s)
        mx = np.full(lp.m, -np.inf)
        np.maximum.at(mx, rows, s)
        ex = np.exp(s - mx[rows])
        a64 = ex / np.bincount(rows, ex, minlength=lp.m)[rows]
        smax = np.zeros(lp.m)
        np.maximum.at(smax, rows, np.abs(s))
        tol_a = a64 * EPS * (8 * smax[rows] + 4 * deg[rows] + 32) + 1e-38
        assert (np.abs(alpha - a64) <= tol_a).all(), "head %d: alpha beyond the bound" % h
        d64 = dal[:, h].astype(np.float64)
        c = np.bincount(rows, alpha * d64, minlength=lp.m)
        cmag = np.bincount(rows, np.abs(alpha * d64), minlength=lp.m)
        sl = np.where(s > 0, 1.0, slope)
        p64 = alpha * (d64 - c[rows]) * sl
        tol_p = sl * alpha * EPS * (4 * np.abs(d64) + 4 * np.abs(c[rows]) + 2 * (deg[rows] + 4) * cmag[rows]) + 1e-38
        assert (np.abs(dpre - p64) <= tol_p).all(), "head %d: dpre beyond the bound" % h
        e64 = np.bincount(rows, p64, minlength=lp.m)
        tol_e = np.bincount(rows, tol_p + (deg[rows] + 4) * EPS * np.abs(p64), minlength=lp.m) + 1e-38
        assert (np.abs(d_el - e64) <= tol_e).all(), "head %d: d_el beyond the bound" % h
        assert np.all(d_el[deg == 0] == 0)
    plan.close()


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("f", [40, 128])
def test_aggregation_equals_the_register_kernel_with_creation_values(K, f):
    if f % K:
        pytest.skip("f % K")
    A, plan = one_rank_plan("hub", f)
    lp = plan.lp
    plan.set_option("kernel", 4)
    rs = np.random.RandomState(f + K)
    H = t(rs.uniform(-1, 1, (lp.m, f)).astype(np.float32))
    alpha = t(np.repeat(lp.vals.astype(np.float32)[:, None], K, axis=1))
    lib = cabi.load()
    Z, Zh = torch.empty_like(H), torch.full_like(H, float("nan"))
    G, Gh = torch.empty_like(H), torch.full_like(H, float("nan"))
    cabi.check(lib.pgcn_forward(plan.handle, H.data_ptr(), Z.data_ptr(), f, stream()), plan.handle)
    cabi.check(lib.pgcn_forward_heads(plan.handle, K, alpha.data_ptr(), H.data_ptr(), Zh.data_ptr(), None, f, stream()),
               plan.handle)
    cabi.check(lib.pgcn_backward(plan.handle, H.data_ptr(), G.data_ptr(), f, stream()), plan.handle)
    cabi.check(lib.pgcn_backward_heads(plan.handle, K, alpha.data_ptr(), H.data_ptr(), Gh.data_ptr(), f, stream()),
               plan.handle)
    assert torch.equal(Z, Zh) and torch.equal(G, Gh)
    plan.close()


def heads64(rows, cols, n_out, alpha, X, K):
    """sum over entries of alpha[e, h] X[col(e), head h] into row(e) (fp64), and the bound sum of |products|."""
    d = X.shape[1] // K
    a = np.repeat(alpha.astype(np.float64), d, axis=1)
    P = a * X.astype(np.float64)[cols]
    out = np.zeros((n_out, X.shape[1]))
    mag = np.zeros((n_out, X.shape[1]))
    np.add.at(out, rows, P)
    np.add.at(mag, rows, np.abs(P))
    return out, mag


@pytest.mark.parametrize("f,K", [(16, 1), (16, 2), (16, 4), (16, 8), (40, 2), (40, 4), (40, 8), (128, 1), (128, 4),
                                 (128, 8), (256, 2), (256, 8)])
def test_aggregation_against_fp64_and_unaligned_operands(f, K):
    A, plan = one_rank_plan("hub", f)
    lp = plan.lp
    rows, cols = edges(lp)
    deg = np.diff(lp.rowptr.astype(np.int64))
    rs = np.random.RandomState(f * 10 + K)
    Hn = rs.uniform(-1, 1, (lp.m, f)).astype(np.float32)
    an = rs.uniform(0, 1, (lp.nnz(), K)).astype(np.float32)
    H, alpha = t(Hn), t(an)
    lib = cabi.load()
    Z, G = torch.empty_like(H), torch.empty_like(H)
    cabi.check(lib.pgcn_forward_heads(plan.handle, K, alpha.data_ptr(), H.data_ptr(), Z.data_ptr(), None, f, stream()),
               plan.handle)
    cabi.check(lib.pgcn_backward_heads(plan.handle, K, alpha.data_ptr(), H.data_ptr(), G.data_ptr(), f, stream()),
               plan.handle)
    z64, zmag = heads64(rows, cols, lp.m, an, Hn, K)
    g64, gmag = heads64(cols, rows, lp.m, an, Hn, K)
    cdeg = np.bincount(cols, minlength=lp.m)
    assert (np.abs(Z.cpu().numpy() - z64) <= (deg[:, None] + 2) * EPS * zmag + 1e-30).all()
    assert (np.abs(G.cpu().numpy() - g64) <= (cdeg[:, None] + 2) * EPS * gmag + 1e-30).all()
    # every operand 4 bytes into its buffer: the same bits
    Hs, As = shifted(H), shifted(alpha)
    Zs, Gs = shifted(torch.full_like(H, float("nan"))), shifted(torch.full_like(H, float("nan")))
    cabi.check(lib.pgcn_forward_heads(plan.handle, K, As.data_ptr(), Hs.data_ptr(), Zs.data_ptr(), None, f, stream()),
               plan.handle)
    cabi.check(lib.pgcn_backward_heads(plan.handle, K, As.data_ptr(), Hs.data_ptr(), Gs.data_ptr(), f, stream()),
               plan.handle)
    assert torch.equal(Zs, Z) and torch.equal(Gs, G)
    plan.close()


@pytest.mark.parametrize("f,K,shift", [(128, 1, False), (128, 2, False), (128, 4, False), (128, 8, False),
                                       (256, 2, False), (256, 4, False), (256, 8, False), (40, 1, True), (40, 2, True),
                                       (40, 4, True), (40, 8, True)])
def test_sddmm_heads_against_fp64(f, K, shift):
    A, plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    rows, cols = edges(lp)
    rs = np.random.RandomState(f + K)
    gn = rs.uniform(-1, 1, (lp.m, f)).astype(np.float32)
    Hn = rs.uniform(-1, 1, (lp.m, f)).astype(np.float32)
    g, H = t(gn), t(Hn)
    if shift:
        g, H = shifted(g), shifted(H)
    lib = cabi.load()
    out = torch.full((lp.nnz(), K), float("nan"), device=dev())
    runs = []
    for _ in range(2):
        cabi.check(lib.pgcn_sddmm_heads(plan.handle, K, g.data_ptr(), H.data_ptr(), None, out.data_ptr(), f, stream()),
                   plan.handle)
        runs.append(out.clone())
    assert torch.equal(runs[0], runs[1])
    d = f // K
    P = gn.astype(np.float64)[rows] * Hn.astype(np.float64)[cols]
    want = P.reshape(-1, K, d).sum(2)
    mag = np.abs(P).reshape(-1, K, d).sum(2)
    got = runs[0].cpu().numpy()
    assert (np.abs(got - want) <= (d + 8) * EPS * mag + 1e-30).all()
    if K == 1:
        ref = torch.empty(lp.nnz(), device=dev())
        cabi.check(lib.pgcn_sddmm(plan.handle, g.data_ptr(), H.data_ptr(), None, ref.data_ptr(), f, stream()), plan.handle)
        assert torch.equal(runs[0].reshape(-1), ref)
    plan.close()


def close(got, want, what):
    u = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else got
    np.testing.assert_allclose(u, want, rtol=2e-4, atol=2e-4 * (np.abs(want).max() + 1e-30), err_msg=what)


def layer(plan, x, W, a, K):
    Z = x @ W.T
    el, er = ho.scores(Z, a, K)
    return PGATMultiHeadAttention.apply(plan, Z, el, er, 0.2)


@pytest.mark.parametrize("layout", ["local", "global"])
@pytest.mark.parametrize("f,K", [(16, 2), (40, 4), (128, 4), (128, 8), (256, 8)])
def test_layer_gradients_one_rank(f, K, layout):
    A, plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp, n = plan.lp, A.shape[0]
    d = f // K
    rs = np.random.RandomState(f + K)
    H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    W = (rs.standard_normal((f, f)) / np.sqrt(f)).astype(np.float32)
    a = (rs.standard_normal((2 * d, K)) / np.sqrt(d)).astype(np.float32)
    Wt, at = t(W).requires_grad_(True), t(a).requires_grad_(True)
    out = layer(plan, t(H), Wt, at, K)
    out.backward(t(G))
    W64 = torch.tensor(W, dtype=torch.float64, requires_grad=True)
    a64 = torch.tensor(a, dtype=torch.float64, requires_grad=True)
    Z64 = torch.from_numpy(H.astype(np.float64)) @ W64.T
    el64, er64 = ho.scores(Z64, a64, K)
    rows, cols = edges(lp)
    o64, _ = ho.attention(torch.from_numpy(rows), torch.from_numpy(cols), n, Z64, el64, er64, 0.2, K)
    o64.backward(torch.from_numpy(G.astype(np.float64)))
    close(out, o64.detach().numpy(), "out")
    close(Wt.grad, W64.grad.numpy(), "dW")
    close(at.grad, a64.grad.numpy(), "da")
    plan.close()


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("case,f,K", [("gemat11_k2", 40, 2), ("gemat11_k2", 128, 8), ("gemat11_k3_hp", 256, 4),
                                      ("karate", 16, 4)])
def test_layer_gradients_multi_rank(case, f, K, overlap):
    A, pv, k = problem(case)
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(f + k + K)
    Zn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Gn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    eln = rs.uniform(-3, 3, (n, K)).astype(np.float32)
    ern = rs.uniform(-3, 3, (n, K)).astype(np.float32)
    own = lambda x, lp: t(x[lp.owned]).requires_grad_(True)
    Z = [own(Zn, lp) for lp in lps]
    el = [own(eln, lp) for lp in lps]
    er = [own(ern, lp) for lp in lps]
    out = run_ranks(plans, lambda r: PGATMultiHeadAttention.apply(plans[r], Z[r], el[r], er[r], 0.2), streams)
    run_ranks(plans, lambda r: out[r].backward(t(Gn[lps[r].owned])), streams)
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    C = C.tocoo()
    Zd, eld, erd = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (Zn, eln, ern))
    o64, _ = ho.attention(torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64)), n, Zd,
                          eld, erd, 0.2, K)
    o64.backward(torch.from_numpy(Gn.astype(np.float64)))
    for r, lp in enumerate(lps):
        w = "%s f=%d K=%d overlap=%d rank %d: " % (case, f, K, overlap, r)
        close(out[r], o64.detach().numpy()[lp.owned], w + "out")
        close(Z[r].grad, Zd.grad.numpy()[lp.owned], w + "dZ")
        close(el[r].grad, eld.grad.numpy()[lp.owned], w + "d_el")
        close(er[r].grad, erd.grad.numpy()[lp.owned], w + "d_er")
    for p in plans:
        assert p.stats["send_volume"] == 2 * p.lp.S + 2 * p.lp.h      # rows: er and Z forward, dZ and d_er back
        p.close()


def test_resident_values_untouched():
    A, plan = one_rank_plan("hub", 128)
    n, f = A.shape[0], 128
    rs = np.random.RandomState(3)
    x = t(rs.uniform(-1, 1, size=(n, f)).astype(np.float32))
    g = t(rs.uniform(-1, 1, size=(n, f)).astype(np.float32))

    def pspmm():
        xp = x.clone().requires_grad_(True)
        z = PSpMM.apply(plan, xp)
        z.backward(g)
        return z.detach(), xp.grad

    before = pspmm()
    e = [t(rs.uniform(-1, 1, (n, 4)).astype(np.float32)).requires_grad_(True) for _ in range(2)]
    for _ in range(2):
        PGATMultiHeadAttention.apply(plan, x.clone().requires_grad_(True), e[0], e[1], 0.2).backward(g)
    after = pspmm()
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])
    plan.close()


def step(plan, x, W, a, g, K):
    out = layer(plan, x, W, a, K)
    out.backward(g)
    return dict(out=out, dW=W.grad, da=a.grad)


def test_one_rank_capture_and_refusal_before_prepare():
    A, plan = one_rank_plan("hub", 128)
    f, n, K = 128, A.shape[0], 4
    rs = np.random.RandomState(11)
    rnd = lambda *s: t(rs.uniform(-1, 1, size=s).astype(np.float32))
    x, g = torch.zeros((n, f), device=dev()), torch.zeros((n, f), device=dev())
    W = torch.zeros((f, f), device=dev(), requires_grad=True)
    a = torch.zeros((2 * f // K, K), device=dev(), requires_grad=True)
    ins = [(rnd(n, f), rnd(n, f), rnd(f, f) * 0.1, rnd(2 * f // K, K) * 0.1) for _ in range(3)]

    def load(i):
        with torch.no_grad():
            for u, v in zip((x, g, W, a), ins[i]):
                u.copy_(v)

    def eager(i):
        xi, gi, Wi, ai = ins[i]
        return step(plan, xi, Wi.clone().requires_grad_(True), ai.clone().requires_grad_(True), gi, K)

    check_one_rank_capture(plan, lambda: step(plan, x, W, a, g, K), load, eager, prepare=(f, 4 * K), leaves=(W, a))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n, K = 128, A.shape[0], 8
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
        p.prepare(4 * K)
        p.prepare(8)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(5)
    ins = [(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.uniform(-1, 1, size=(n, f)).astype(np.float32),
            (rs.standard_normal((f, f)) * 0.1).astype(np.float32),
            (rs.standard_normal((2 * f // K, K)) * 0.1).astype(np.float32)) for _ in range(3)]

    def buffers(r):
        m = lps[r].m
        return dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()),
                    W=torch.zeros((f, f), device=dev(), requires_grad=True),
                    a=torch.zeros((2 * f // K, K), device=dev(), requires_grad=True))

    def load(bufs, i):
        H, G, Wn, an = ins[i]
        with torch.no_grad():
            for r, lp in enumerate(lps):
                b = bufs[r]
                b["x"].copy_(torch.from_numpy(H[lp.owned])); b["g"].copy_(torch.from_numpy(G[lp.owned]))
                b["W"].copy_(torch.from_numpy(Wn)); b["a"].copy_(torch.from_numpy(an))
        torch.cuda.synchronize()

    check_two_rank_capture(plans, streams, buffers, load,
                           lambda r, b: step(plans[r], b["x"], b["W"], b["a"], b["g"], K))
    for p in plans:
        p.close()


def test_cli_heads_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", ["--heads", "2"], 29671)
    assert_follows(lines, ho.intended_training(karate(), 2, 4, 7, 1.0, heads=2))


def test_cli_heads_one_prints_what_no_flag_prints(tmp_path):
    plain = run_cli(tmp_path, "PGAT.py", [], 29672)
    one = run_cli(tmp_path, "PGAT.py", ["--heads", "1"], 29673)
    assert len(plain) == 50 and one == plain
