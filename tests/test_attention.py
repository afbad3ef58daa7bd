"""Sparse graph attention on the H100 path: pgcn_edge_softmax, pgcn_edge_softmax_backward, pgcn_halo_rows,
op.PGATAttention and the PGAT command line.

  * alpha, dpre and d_el lie within an fp32 bound of fp64 and are run-to-run identical: warp rows and CTA rows (hub rows
    of more than 1024 entries), rows of one entry, empty rows, slopes 0.2 and 1.0, scores around +-80 and beyond;
  * PGATAttention's output and the gradients of Z, el, er (and through torch of W and a) against fp64, on one rank
    in both layouts and on two and three ranks of one process over the peer transport;
  * pgcn_halo_rows is bit-exact, interleaved with fused calls so that both exchange parities occur;
  * PSpMM after attention equals a fresh plan; CUDA-graph capture of the layer on one and two ranks, and its refusal
    before pgcn_plan_prepare; PGAT.py follows the fp64 loss curve of oracle/pgat_oracle.py.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from harness import (EPS, assert_follows, check_one_rank_capture, check_two_rank_capture, dev, edges, karate,
                     linked_plans, one_rank_plan, problem, run_cli, run_ranks, stream, t)
from oracle import pgat_oracle as po
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import PGATAttention, PSpMM

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", ["gemat11_k1", "karate", "hub"])
@pytest.mark.parametrize("slope", [0.2, 1.0])
@pytest.mark.parametrize("scale", [1.0, 80.0])
def test_softmax_kernels_within_fp32_bound_and_deterministic(case, slope, scale):
    A, plan = one_rank_plan(case, 4)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr)
        assert deg.max() > 1024 and (deg == 0).any() and (deg == 1).any()
    rs = np.random.RandomState(int(scale) + int(10 * slope))
    el = rs.uniform(-scale, scale, lp.m).astype(np.float32)
    er = rs.uniform(-scale, scale, lp.m).astype(np.float32)
    dal = rs.uniform(-1, 1, lp.nnz()).astype(np.float32)
    lib = cabi.load()
    el_d, er_d, dal_d = t(el), t(er), t(dal)
    runs = []
    for _ in range(2):
        alpha = torch.empty(lp.nnz(), device=dev())
        dpre = torch.empty(lp.nnz(), device=dev())
        d_el = torch.full((lp.m,), float("nan"), device=dev())
        cabi.check(lib.pgcn_edge_softmax(plan.handle, el_d.data_ptr(), er_d.data_ptr(), None, slope, alpha.data_ptr(),
                                         stream()), plan.handle)
        cabi.check(lib.pgcn_edge_softmax_backward(plan.handle, el_d.data_ptr(), er_d.data_ptr(), None, alpha.data_ptr(),
                                                  dal_d.data_ptr(), slope, dpre.data_ptr(), d_el.data_ptr(), stream()),
                   plan.handle)
        runs.append((alpha.cpu().numpy(), dpre.cpu().numpy(), d_el.cpu().numpy()))
    for a, b in zip(runs[0], runs[1]):
        assert np.array_equal(a, b), "not run-to-run identical"
    alpha, dpre, d_el = (x.astype(np.float64) for x in runs[0])
    rows, cols = edges(lp)
    deg = np.diff(lp.rowptr.astype(np.int64))
    s = el.astype(np.float64)[rows] + er.astype(np.float64)[cols]
    s = np.where(s > 0, s, slope * s)
    mx = np.full(lp.m, -np.inf)
    np.maximum.at(mx, rows, s)
    ex = np.exp(s - mx[rows])
    den = np.bincount(rows, ex, minlength=lp.m)
    a64 = ex / den[rows]
    smax = np.zeros(lp.m)
    np.maximum.at(smax, rows, np.abs(s))
    tol_a = a64 * EPS * (8 * smax[rows] + 4 * deg[rows] + 32) + 1e-38
    assert (np.abs(alpha - a64) <= tol_a).all(), "%s: %d alphas beyond the bound" % (case, int((np.abs(alpha - a64) > tol_a).sum()))
    assert np.isfinite(alpha).all()
    # backward, from the kernel's own alpha
    d64 = dal.astype(np.float64)
    c = np.bincount(rows, alpha * d64, minlength=lp.m)
    cmag = np.bincount(rows, np.abs(alpha * d64), minlength=lp.m)
    sl = np.where(s > 0, 1.0, slope)
    p64 = alpha * (d64 - c[rows]) * sl
    tol_p = sl * alpha * EPS * (4 * np.abs(d64) + 4 * np.abs(c[rows]) + 2 * (deg[rows] + 4) * cmag[rows]) + 1e-38
    assert (np.abs(dpre - p64) <= tol_p).all(), "%s: %d dpre beyond the bound" % (case, int((np.abs(dpre - p64) > tol_p).sum()))
    e64 = np.bincount(rows, p64, minlength=lp.m)
    tol_e = np.bincount(rows, tol_p + (deg[rows] + 4) * EPS * np.abs(p64), minlength=lp.m) + 1e-38
    assert (np.abs(d_el - e64) <= tol_e).all()
    assert np.all(d_el[deg == 0] == 0)
    plan.close()


def attention64(rows, cols, n, Z, el, er, slope, G):
    """fp64 out and the gradients of Z, el, er of <out, G> (oracle.pgat_oracle.attention)."""
    Z, el, er = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (Z, el, er))
    out, _ = po.attention(torch.from_numpy(rows), torch.from_numpy(cols), n, Z, el, er, slope)
    out.backward(torch.from_numpy(G.astype(np.float64)))
    return [x.detach().numpy() for x in (out, Z.grad, el.grad, er.grad)]


def close(got, want, what):
    u = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else got
    np.testing.assert_allclose(u, want, rtol=2e-4, atol=2e-4 * (np.abs(want).max() + 1e-30), err_msg=what)


@pytest.mark.parametrize("layout", ["local", "global"])
@pytest.mark.parametrize("f", [16, 40, 128, 256])
@pytest.mark.parametrize("case", ["gemat11_k1", "hub"])
def test_layer_gradients_one_rank(case, f, layout):
    A, plan = one_rank_plan(case, f)
    plan.layout = layout
    lp, n = plan.lp, A.shape[0]
    rs = np.random.RandomState(f)
    H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    W = (rs.standard_normal((f, f)) / np.sqrt(f)).astype(np.float32)
    a = (rs.standard_normal((2 * f, 1)) / np.sqrt(f)).astype(np.float32)
    x = torch.from_numpy(H).to(dev())
    Wt = torch.from_numpy(W).to(dev()).requires_grad_(True)
    at = torch.from_numpy(a).to(dev()).requires_grad_(True)
    Z = x @ Wt.T
    Z.retain_grad()
    el = (Z @ at[:f]).squeeze(1)
    er = (Z @ at[f:]).squeeze(1)
    el.retain_grad(); er.retain_grad()
    out = PGATAttention.apply(plan, Z, el, er, 0.2)
    out.backward(torch.from_numpy(G).to(dev()))
    # fp64 through the same torch graph
    W64 = torch.tensor(W, dtype=torch.float64, requires_grad=True)
    a64 = torch.tensor(a, dtype=torch.float64, requires_grad=True)
    Z64 = torch.from_numpy(H.astype(np.float64)) @ W64.T
    el64, er64 = (Z64 @ a64[:f]).squeeze(1), (Z64 @ a64[f:]).squeeze(1)
    for u in (Z64, el64, er64):
        u.retain_grad()
    rows, cols = edges(lp)
    o64, _ = po.attention(torch.from_numpy(rows), torch.from_numpy(cols), n, Z64, el64, er64, 0.2)
    o64.backward(torch.from_numpy(G.astype(np.float64)))
    close(out, o64.detach().numpy(), "out")
    close(Z.grad, Z64.grad.numpy(), "dZ")
    close(el.grad, el64.grad.numpy(), "d_el")
    close(er.grad, er64.grad.numpy(), "d_er")
    close(Wt.grad, W64.grad.numpy(), "dW")
    close(at.grad, a64.grad.numpy(), "da")
    plan.close()


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("case,f", [("gemat11_k2", 40), ("gemat11_k2", 128), ("gemat11_k3_hp", 256),
                                    ("karate", 16)])
def test_layer_gradients_multi_rank(case, f, overlap):
    A, pv, k = problem(case)
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(f + k)
    Zn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Gn = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    eln = rs.uniform(-3, 3, n).astype(np.float32)
    ern = rs.uniform(-3, 3, n).astype(np.float32)
    own = lambda x, lp: t(x[lp.owned]).requires_grad_(True)
    Z = [own(Zn, lp) for lp in lps]
    el = [own(eln, lp) for lp in lps]
    er = [own(ern, lp) for lp in lps]
    out = run_ranks(plans, lambda r: PGATAttention.apply(plans[r], Z[r], el[r], er[r], 0.2), streams)
    run_ranks(plans, lambda r: out[r].backward(torch.from_numpy(Gn[lps[r].owned]).to(dev())), streams)
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    C = C.tocoo()
    o64, gZ, gel, ger = attention64(C.row.astype(np.int64), C.col.astype(np.int64), n, Zn, eln, ern, 0.2, Gn)
    for r, lp in enumerate(lps):
        w = "%s f=%d overlap=%d rank %d: " % (case, f, overlap, r)
        close(out[r], o64[lp.owned], w + "out")
        close(Z[r].grad, gZ[lp.owned], w + "dZ")
        close(el[r].grad, gel[lp.owned], w + "d_el")
        close(er[r].grad, ger[lp.owned], w + "d_er")
    for p in plans:
        assert p.stats["send_volume"] == 2 * p.lp.S + 2 * p.lp.h      # rows: er and Z forward, dZ and d_er back
        p.close()


@pytest.mark.parametrize("w", [4, 128])
def test_halo_rows_bit_exact_across_parities(w):
    A, pv, k = problem("gemat11_k3_hp")
    n = A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 128, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    lib = cabi.load()
    rs = np.random.RandomState(w)
    for it in range(4):
        X = rs.uniform(-1, 1, size=(n, w)).astype(np.float32)
        xs = [torch.from_numpy(X[lp.owned]).to(dev()) for lp in lps]

        def one(r):
            p, lp = plans[r], lps[r]
            halo = torch.full((lp.h, w), float("nan"), device=dev())
            cabi.check(lib.pgcn_halo_rows(p.handle, xs[r].data_ptr(), halo.data_ptr(), w, stream()), p.handle)
            z = torch.empty_like(xs[r])
            # fused calls in between (epochs: halo 1, fwd 2 | halo 3, fwd 4, bwd 5 | halo 6 | halo 7, bwd 8): the
            # exchange-only call meets both parities, and so do the fused calls around it
            if it in (0, 1):
                cabi.check(lib.pgcn_forward(p.handle, xs[r].data_ptr(), z.data_ptr(), w, stream()), p.handle)
            if it in (1, 3):
                cabi.check(lib.pgcn_backward(p.handle, xs[r].data_ptr(), z.data_ptr(), w, stream()), p.handle)
            return halo
        got = run_ranks(plans, one, streams)
        for r, lp in enumerate(lps):
            assert torch.equal(got[r].cpu(), torch.from_numpy(X[lp.halo])), "iteration %d rank %d" % (it, r)
    assert {p.get_option("epoch") for p in plans} == {8}
    for p in plans:
        p.close()


def test_pspmm_after_attention_equals_fresh_plan():
    A, plan = one_rank_plan("hub", 128)
    fresh = planmod.build_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1, 128, device=dev())
    n = A.shape[0]
    rs = np.random.RandomState(3)
    x = torch.from_numpy(rs.uniform(-1, 1, size=(n, 128)).astype(np.float32)).to(dev())
    g = torch.from_numpy(rs.uniform(-1, 1, size=(n, 128)).astype(np.float32)).to(dev())
    e = [torch.from_numpy(rs.uniform(-1, 1, n).astype(np.float32)).to(dev()).requires_grad_(True) for _ in range(2)]
    PGATAttention.apply(plan, x.clone().requires_grad_(True), e[0], e[1], 0.2).backward(g)
    outs = []
    for p in (plan, fresh):
        xp = x.clone().requires_grad_(True)
        z = PSpMM.apply(p, xp)
        z.backward(g)
        outs.append((z.detach(), xp.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    plan.close(); fresh.close()


def layer_step(plan, f, x, W, a, g):
    Z = x @ W.T
    out = PGATAttention.apply(plan, Z, (Z @ a[:f]).squeeze(1), (Z @ a[f:]).squeeze(1), 0.2)
    out.backward(g)
    return out


def test_one_rank_capture_and_refusal_before_prepare():
    A, plan = one_rank_plan("hub", 128)
    f, n = 128, A.shape[0]
    rs = np.random.RandomState(11)
    rnd = lambda *s: t(rs.uniform(-1, 1, size=s).astype(np.float32))
    x, g = torch.zeros((n, f), device=dev()), torch.zeros((n, f), device=dev())
    W = torch.zeros((f, f), device=dev(), requires_grad=True)
    a = torch.zeros((2 * f, 1), device=dev(), requires_grad=True)
    ins = [(rnd(n, f), rnd(n, f), rnd(f, f) * 0.1, rnd(2 * f, 1) * 0.1) for _ in range(3)]

    def step():
        return dict(out=layer_step(plan, f, x, W, a, g), dW=W.grad, da=a.grad)

    def load(i):
        with torch.no_grad():
            for u, v in zip((x, g, W, a), ins[i]):
                u.copy_(v)

    def eager(i):
        xi, gi, Wi, ai = ins[i]
        We, ae = Wi.clone().requires_grad_(True), ai.clone().requires_grad_(True)
        oe = layer_step(plan, f, xi, We, ae, gi)
        PSpMM.apply(plan, xi)                                  # the creation values in between
        return dict(out=oe, dW=We.grad, da=ae.grad)

    check_one_rank_capture(plan, step, load, eager, prepare=(f, 4), leaves=(W, a))
    plan.close()


def test_two_rank_capture_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n = 128, A.shape[0]
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, 1)
    for p in plans:
        p.prepare(f)
        p.prepare(4)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    rs = np.random.RandomState(5)
    ins = [(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.uniform(-1, 1, size=(n, f)).astype(np.float32),
            (rs.standard_normal((f, f)) * 0.1).astype(np.float32), (rs.standard_normal((2 * f, 1)) * 0.1).astype(np.float32))
           for _ in range(3)]

    def buffers(r):
        m = lps[r].m
        return dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()),
                    W=torch.zeros((f, f), device=dev(), requires_grad=True),
                    a=torch.zeros((2 * f, 1), device=dev(), requires_grad=True))

    def load(bufs, i):
        H, G, Wn, an = ins[i]
        with torch.no_grad():
            for r, lp in enumerate(lps):
                b = bufs[r]
                b["x"].copy_(torch.from_numpy(H[lp.owned])); b["g"].copy_(torch.from_numpy(G[lp.owned]))
                b["W"].copy_(torch.from_numpy(Wn)); b["a"].copy_(torch.from_numpy(an))
        torch.cuda.synchronize()

    def step(r, b):
        return dict(out=layer_step(plans[r], f, b["x"], b["W"], b["a"], b["g"]), dW=b["W"].grad, da=b["a"].grad)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for p in plans:
        p.close()


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PGAT.py", [], 29660)
    assert_follows(lines, po.intended_training(karate(), 2, 4, 7, 1.0))
