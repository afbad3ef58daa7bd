"""Edge dropout on the H100 path: pgcn_edge_dropout (libpgcn_dropout.so), PgcnPlan.edge_pairs, op.EdgeDropout,
op.edge_dropout, the dropout argument of PGATAttention / PGATMultiHeadAttention and PGAT.py --attn-dropout.

  * every kernel instance gives the NumPy oracle's bits (K = 1, 2, 4, 8; aligned and 4-byte-shifted operands; in place
    and out of place; IEEE specials; the hub graph) and torch.profiler sees every instance of the manifest;
  * the mask depends on the global edge only: 1 rank against 3 (karate) and 2 (R-MAT) give the same bits per edge;
  * on >= 1 M entries the kept fraction, and the agreement between heads and between consecutive counters, lie within
    5 sigma of 1 - p and p^2 + (1 - p)^2;
  * both GAT operators at p = 0.5 against the fp64 oracle (one rank, both layouts; karate on 3 linked ranks, overlap 0
    and 1); p = 0, None and eval mode make exactly the calls of no dropout; a backward uses its own forward's mask;
    edge_dropout + PSpMMWeighted against fp64;
  * CUDA graphs: every replay equals the eager call at the same counter (one rank, two ranks over the peer transport);
    a capture before edge_pairs() exists is refused and enqueues nothing;
  * the command line follows the fp64 curve with --attn-dropout 0.5 (one head and two), and --attn-dropout 0 prints what
    no flag prints.
"""
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import dropout_oracle as do
from conftest import ROOT
from harness import (assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate, linked_plans,
                     one_rank_plan, problem, run_cli, run_ranks, shifted, spawn_ranks, t)
from pgcn_b200 import graphio, plan as planmod
from pgcn_b200.op import (EdgeDropout, PGATAttention, PGATMultiHeadAttention, PSpMMWeighted, edge_dropout, _mask)
from pgcn_b200.pgat import PGAT

pytestmark = pytest.mark.gpu

KEY = 0x0123456789ABCDEF


def key(name):
    """Instance name without return type, parameter list, casts and spaces, bools as 0 / 1: the manifest's and the
    profiler's spellings of one instance give the same key."""
    s = name.strip()
    for a, b in (("(int)", ""), ("(bool)", ""), ("true", "1"), ("false", "0")):
        s = s.replace(a, b)
    if s.startswith("void "):
        s = s[5:]
    return s.split("(")[0].replace(" ", "")


def profiled(fn):
    """(fn's result, the names of the CUDA kernels it launched, in order)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def state(c, k=KEY):
    return torch.tensor([k - 2 ** 64 if k >= 2 ** 63 else k, c], dtype=torch.int64, device=dev())


def specials(x):
    x = x.copy()
    flat = x.reshape(-1)
    flat[:6] = [np.nan, np.inf, -np.inf, -0.0, 1e-40, -3e38]
    return x


def same(got, want):
    """The oracle's bits, NaN for NaN (the GPU writes its canonical NaN, NumPy propagates the operand's payload)."""
    g = got.detach().cpu().numpy()
    nan = np.isnan(want)
    return np.array_equal(np.isnan(g), nan) and np.array_equal(g[~nan].view(np.uint32), want[~nan].view(np.uint32))


def run_kernel(pairs, x, y, K, p, snap):
    d = EdgeDropout(p, KEY, dev())
    _mask(pairs, snap, d, x, y)
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("p", [0.3, 0.6])
def test_instances_give_the_oracle_bits(K, shift, inplace, p):
    A, plan = one_rank_plan("hub", 8)
    pairs = plan.edge_pairs()
    lp = plan.lp
    deg = np.diff(lp.rowptr.astype(np.int64))
    assert deg.max() >= 3000 and (deg == 0).any() and (deg == 1).any()
    pn = pairs.cpu().numpy()
    rows = np.repeat(lp.owned, deg)
    assert np.array_equal(pn[:, 0], rows) and np.array_equal(pn[:, 1], lp.colidx)
    rs = np.random.RandomState(K + 10 * shift + 100 * inplace)
    xn = specials(rs.uniform(-2, 2, (lp.nnz(), K)).astype(np.float32))
    if K == 1:
        xn = xn[:, 0].copy()
    x = t(xn)
    if shift:
        x, pairs = shifted(x), shifted(pairs)
    y = x if inplace else (shifted(torch.empty_like(x)) if shift else torch.empty_like(x))
    got = run_kernel(pairs, x, y, K, p, state(5))
    assert same(got, do.apply(xn, pn[:, 0], pn[:, 1], p, KEY, 5))
    plan.close()


def _instances_worker(rank, k):
    """The keys of the edge-dropout kernels that torch.profiler sees when every instance is launched once."""
    A, plan = one_rank_plan("hub", 8)
    pairs = plan.edge_pairs()
    seen = set()

    def all_instances():
        for K in (1, 2, 4, 8):
            x = torch.ones((plan.lp.nnz(), K), device=dev())
            for pr, u in ((pairs, x), (shifted(pairs), shifted(x))):
                run_kernel(pr, u, u, K, 0.5, state(1))

    for _ in range(3):            # torch.profiler now and then loses a session's activity records
        _, names = profiled(all_instances)
        seen |= {key(n) for n in names if "edge_dropout" in n}
        if len(seen) == 8:
            break
    plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    # every torch.profiler session of this file runs in a process of its own: a session leaves the profiler attached
    # to the process, and later sessions in it (the kernel census, run after this file) then lose the records of their
    # first kernels
    with open(os.path.join(ROOT, "tests", "dropout_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


@pytest.mark.parametrize("case", ["karate", "rmat_k2"])
def test_partition_independence(case):
    A, pv, k = problem(case)
    assert k > 1
    n = A.shape[0]
    K = 8

    def per_edge(lp, plan):
        pairs = plan.edge_pairs()
        pn = pairs.cpu().numpy().astype(np.int64)
        xn = np.sin(pn[:, :1] * 0.37 + pn[:, 1:] * 1.3 + np.arange(K)).astype(np.float32)
        y = run_kernel(pairs, t(xn), torch.empty((lp.nnz(), K), device=dev()), K, 0.5, state(3))
        return dict(zip((pn[:, 0] * n + pn[:, 1]).tolist(), bits(y)))

    p1 = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, 8, device=dev())
    ref = per_edge(p1.lp, p1)
    seen = 0
    for r in range(k):
        p = planmod.build_plan(A, pv, r, k, 8, device=dev())
        got = per_edge(p.lp, p)
        for e, b in got.items():
            assert np.array_equal(b, ref[e]), "rank %d edge %d" % (r, e)
        seen += len(got)
        p.close()
    assert seen == len(ref)
    p1.close()


def test_statistics_on_a_million_entries():
    n = 1 << 17
    A = graphio.synthetic_graph(n, 1_600_000, seed=9)
    plan = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, 8, device=dev())
    nnz = plan.lp.nnz()
    assert nnz >= 1_000_000
    pairs = plan.edge_pairs()
    K = 8
    ones = torch.ones((nnz, K), device=dev())
    for p in (0.1, 0.5, 0.9):
        drop = EdgeDropout(p, 1000 + int(10 * p), dev())
        k1 = edge_dropout(plan, ones, drop) != 0
        k2 = edge_dropout(plan, ones, drop) != 0
        assert int(drop.state[1]) == 2
        N = k1.numel()
        frac = float(k1.float().mean())
        assert abs(frac - (1 - p)) <= 5 * np.sqrt(p * (1 - p) / N), (p, frac)
        q = p * p + (1 - p) * (1 - p)
        heads = float((k1[:, 0::2] == k1[:, 1::2]).float().mean())        # disjoint head pairs
        assert abs(heads - q) <= 5 * np.sqrt(q * (1 - q) / (nnz * K // 2)), (p, heads)
        calls = float((k1 == k2).float().mean())
        assert abs(calls - q) <= 5 * np.sqrt(q * (1 - q) / N), (p, calls)
        if p == 0.5:                  # the grid-stride loop goes round several times here: still the oracle's bits
            pn = pairs.cpu().numpy()
            assert np.array_equal(k1.cpu().numpy(), do.keep(pn[:, 0], pn[:, 1], K, p, drop_key(drop), 1))
    plan.close()


def drop_key(drop):
    return int(drop.state[0]) % 2 ** 64


def close(got, want, what):
    u = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else got
    np.testing.assert_allclose(u, want, rtol=2e-4, atol=2e-4 * (np.abs(want).max() + 1e-30), err_msg=what)


def apply_op(plan, Z, el, er, K, drop):
    if K == 0:
        return PGATAttention.apply(plan, Z, el, er, 0.2, drop)
    return PGATMultiHeadAttention.apply(plan, Z, el, er, 0.2, drop)


def oracle(A, Zn, eln, ern, G, K, p, counter):
    """fp64 out and gradients of Z, el, er on the global graph, mask at `counter`."""
    C = sp.csr_matrix(A)
    C.sum_duplicates()
    C = C.tocoo()
    n = A.shape[0]
    H = max(K, 1)
    Zd, eld, erd = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (Zn, eln, ern))
    mask = do.weights(C.row, C.col, H, p, KEY, counter)
    o, _ = do.attention(torch.from_numpy(C.row.astype(np.int64)), torch.from_numpy(C.col.astype(np.int64)), n, Zd,
                        eld, erd, 0.2, mask, H)
    o.backward(torch.from_numpy(G.astype(np.float64)))
    return o.detach().numpy(), Zd.grad.numpy(), eld.grad.numpy(), erd.grad.numpy()


def inputs(n, f, K, seed):
    rs = np.random.RandomState(seed)
    sc = (n,) if K == 0 else (n, K)
    return (rs.uniform(-1, 1, (n, f)).astype(np.float32), rs.uniform(-3, 3, sc).astype(np.float32),
            rs.uniform(-3, 3, sc).astype(np.float32), rs.uniform(-1, 1, (n, f)).astype(np.float32))


@pytest.mark.parametrize("layout", ["local", "global"])
@pytest.mark.parametrize("K", [0, 1, 4, 8])          # 0: PGATAttention, else PGATMultiHeadAttention
def test_operators_against_fp64_one_rank(K, layout):
    f = 64
    A, plan = one_rank_plan("hub", f)
    plan.layout = layout
    n = A.shape[0]
    Zn, eln, ern, Gn = inputs(n, f, K, 10 + K)
    Z, el, er = (t(x).requires_grad_(True) for x in (Zn, eln, ern))
    drop = EdgeDropout(0.5, KEY, dev())
    out = apply_op(plan, Z, el, er, K, drop)
    out.backward(t(Gn))
    o64, dZ, dl, dr = oracle(A, Zn, eln, ern, Gn, K, 0.5, 1)
    close(out, o64, "out")
    close(Z.grad, dZ, "dZ")
    close(el.grad, dl, "d_el")
    close(er.grad, dr, "d_er")
    plan.close()


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("K", [0, 2])
def test_operators_against_fp64_three_ranks(K, overlap):
    A, pv, k = problem("karate")
    n, f = A.shape[0], 16
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, f, overlap)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    Zn, eln, ern, Gn = inputs(n, f, K, 20 + K)
    own = lambda x, lp: t(x[lp.owned]).requires_grad_(True)
    Z, el, er = ([own(x, lp) for lp in lps] for x in (Zn, eln, ern))
    drops = [EdgeDropout(0.5, KEY, dev()) for _ in plans]
    out = run_ranks(plans, lambda r: apply_op(plans[r], Z[r], el[r], er[r], K, drops[r]), streams)
    run_ranks(plans, lambda r: out[r].backward(t(Gn[lps[r].owned])), streams)
    o64, dZ, dl, dr = oracle(A, Zn, eln, ern, Gn, K, 0.5, 1)
    for r, lp in enumerate(lps):
        w = "K=%d overlap=%d rank %d: " % (K, overlap, r)
        close(out[r], o64[lp.owned], w + "out")
        close(Z[r].grad, dZ[lp.owned], w + "dZ")
        close(el[r].grad, dl[lp.owned], w + "d_el")
        close(er[r].grad, dr[lp.owned], w + "d_er")
    for p in plans:
        p.close()


def _no_dropout_worker(rank, k, K):
    """Asserts that p = 0, None and eval mode make exactly the calls, and give the bits, of no dropout. Returns True."""
    f = 64
    A, plan = one_rank_plan("hub", f)
    n = A.shape[0]
    Zn, eln, ern, Gn = inputs(n, f, K, 30 + K)
    plan.edge_pairs()
    zero = EdgeDropout(0.0, KEY, dev())

    def step(*extra):
        Z, el, er = (t(x).requires_grad_(True) for x in (Zn, eln, ern))
        f_ = PGATAttention if K == 0 else PGATMultiHeadAttention
        out = f_.apply(plan, Z, el, er, 0.2, *extra)
        out.backward(t(Gn))
        return [out.detach(), Z.grad, el.grad, er.grad]

    def observe(*extra):
        for _ in range(3):        # torch.profiler now and then loses a session's activity records
            before, stats = plan.launch_count(), dict(plan.stats)
            res, names = profiled(lambda: step(*extra))
            names = [s for s in names if "pgcn::" in s]          # the operator's kernels, not the test's copies
            if any("softmax" in s for s in names):
                return res, names, plan.launch_count() - before, {k_: plan.stats[k_] - stats[k_] for k_ in stats}
        raise AssertionError("torch.profiler recorded no softmax kernel")

    step()                        # first-call set-up out of the way
    base = observe()
    assert not any("edge_dropout" in s for s in base[1])
    for extra in ((None,), (zero,)):
        got = observe(*extra)
        for u, w in zip(got[0], base[0]):
            assert np.array_equal(bits(u), bits(w))
        assert got[1] == base[1], "kernels %s, without dropout %s" % (got[1], base[1])
        assert got[2:] == base[2:]
    assert int(zero.state[1]) == 0
    # a PGAT module in eval mode runs without its dropout
    torch.manual_seed(3)
    m = PGAT(plan, f, f, 0.2, max(K, 1), EdgeDropout(0.5, KEY, dev())).to(dev())
    H = t(Zn)
    m.train()
    trained = m(H).detach()
    assert int(m.attn_dropout.state[1]) == 1
    m.eval()
    ev = m(H).detach()
    m.attn_dropout = None
    m.train()
    assert np.array_equal(bits(ev), bits(m(H).detach())) and not torch.equal(ev, trained)
    plan.close()
    return True


@pytest.mark.parametrize("K", [0, 4])
def test_no_dropout_makes_exactly_the_calls_without_it(K):
    # in a process of its own, for the reason test_profiler_sees_every_instance_of_the_manifest gives
    assert spawn_ranks(_no_dropout_worker, 1, (K,)) == {0: True}


@pytest.mark.parametrize("K", [0, 4])
def test_backward_uses_its_own_forwards_mask(K):
    f = 64
    A, plan = one_rank_plan("hub", f)
    n = A.shape[0]
    Zn, eln, ern, Gn = inputs(n, f, K, 40 + K)

    def forward(drop):
        Z, el, er = (t(x).requires_grad_(True) for x in (Zn, eln, ern))
        return apply_op(plan, Z, el, er, K, drop), (Z, el, er)

    drop = EdgeDropout(0.5, KEY, dev())
    out1, leaves1 = forward(drop)
    out2, _ = forward(drop)                      # counter 2 in between
    out1.backward(t(Gn))
    ref = EdgeDropout(0.5, KEY, dev())
    out0, leaves0 = forward(ref)
    out0.backward(t(Gn))
    assert np.array_equal(bits(out1), bits(out0)) and not torch.equal(out1, out2)
    for a, b in zip(leaves1, leaves0):
        assert np.array_equal(bits(a.grad), bits(b.grad))
    plan.close()


@pytest.mark.parametrize("K", [1, 4])
def test_edge_dropout_with_weighted_aggregation_against_fp64(K):
    f = 32
    A, plan = one_rank_plan("gemat11_k1", f)
    lp, n = plan.lp, A.shape[0]
    rs = np.random.RandomState(K)
    pn = plan.edge_pairs().cpu().numpy()
    if K == 1:
        vn, Hn, Gn = (rs.uniform(-1, 1, s).astype(np.float32) for s in ((lp.nnz(),), (n, f), (n, f)))
        vals, H = t(vn).requires_grad_(True), t(Hn).requires_grad_(True)
        drop = EdgeDropout(0.4, KEY, dev())
        out = PSpMMWeighted.apply(plan, edge_dropout(plan, vals, drop), H)
        out.backward(t(Gn))
        w = do.weights(pn[:, 0], pn[:, 1], 1, 0.4, KEY, 1)[:, 0]
        v64 = torch.tensor(vn, dtype=torch.float64, requires_grad=True)
        H64 = torch.tensor(Hn, dtype=torch.float64, requires_grad=True)
        rows = torch.from_numpy(pn[:, 0].astype(np.int64))
        cols = torch.from_numpy(pn[:, 1].astype(np.int64))
        o64 = torch.zeros((n, f), dtype=torch.float64).index_add(0, rows, (v64 * w)[:, None] * H64[cols])
        o64.backward(torch.from_numpy(Gn.astype(np.float64)))
        close(out, o64.detach().numpy(), "out")
        close(vals.grad, v64.grad.numpy(), "dvals")
        close(H.grad, H64.grad.numpy(), "dH")
    else:
        xn, gn = (rs.uniform(-1, 1, (lp.nnz(), K)).astype(np.float32) for _ in range(2))
        x = t(xn).requires_grad_(True)
        drop = EdgeDropout(0.4, KEY, dev())
        y = edge_dropout(plan, x, drop)
        y.backward(t(gn))
        assert np.array_equal(bits(y), do.apply(xn, pn[:, 0], pn[:, 1], 0.4, KEY, 1).view(np.uint32))
        assert np.array_equal(bits(x.grad), do.apply(gn, pn[:, 0], pn[:, 1], 0.4, KEY, 1).view(np.uint32))
    plan.close()


def layer_step(plan, x, W, a, g, K, drop):
    Z = x @ W.T
    if K == 0:
        f = Z.shape[1]
        el, er = (Z @ a[:f]).squeeze(1), (Z @ a[f:]).squeeze(1)
    else:
        d = Z.shape[1] // K
        Zh = Z.view(Z.shape[0], K, d)
        el, er = torch.einsum("nhd,dh->nh", Zh, a[:d]), torch.einsum("nhd,dh->nh", Zh, a[d:])
    out = apply_op(plan, Z, el, er, K, drop)
    out.backward(g)
    return dict(out=out, dW=W.grad, da=a.grad)


def a_shape(f, K):
    return (2 * f, 1) if K == 0 else (2 * f // K, K)


def follower(drop):
    """A second EdgeDropout whose next use draws with the counter `drop` used last."""
    ref = EdgeDropout(drop.p, KEY, dev())
    ref.state.copy_(drop.state)
    ref.state[1:].sub_(1)
    return ref


@pytest.mark.parametrize("K", [0, 4])
def test_one_rank_capture_and_refusal_before_edge_pairs(K):
    A, plan = one_rank_plan("hub", 128)
    f, n = 128, A.shape[0]
    for w in (f, 4 * max(K, 1)):
        plan.prepare(w)
    rs = np.random.RandomState(11)
    rnd = lambda *s: t(rs.uniform(-1, 1, size=s).astype(np.float32))
    x, g = torch.zeros((n, f), device=dev()), torch.zeros((n, f), device=dev())
    W = torch.zeros((f, f), device=dev(), requires_grad=True)
    a = torch.zeros(a_shape(f, K), device=dev(), requires_grad=True)
    ins = [(rnd(n, f), rnd(n, f), rnd(f, f) * 0.1, rnd(*a_shape(f, K)) * 0.1) for _ in range(3)]
    drop = EdgeDropout(0.5, KEY, dev())
    w = torch.ones((8, 8), device=dev(), requires_grad=True)     # cuBLAS handles of this thread and of the autograd
    (w @ w).sum().backward()                                    # thread, which a capture cannot create

    def load(i):
        with torch.no_grad():
            for u, v in zip((x, g, W, a), ins[i]):
                u.copy_(v)

    # before edge_pairs() exists: refused, nothing enqueued
    Zn, eln, ern, _ = inputs(n, f, K, 50)
    Z, el, er = t(Zn), t(eln), t(ern)
    torch.cuda.synchronize()
    before = plan.launch_count()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with pytest.raises(RuntimeError, match="edge_pairs"):
            with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=torch.cuda.Stream()):
                apply_op(plan, Z, el, er, K, drop)
    assert plan.launch_count() == before and int(drop.state[1]) == 0
    assert any("CUDA Graph is empty" in str(w_.message) for w_ in caught)
    plan.edge_pairs()

    def eager(i):
        xi, gi, Wi, ai = ins[i]
        return layer_step(plan, xi, Wi.clone().requires_grad_(True), ai.clone().requires_grad_(True), gi, K,
                          follower(drop))

    check_one_rank_capture(plan, lambda: layer_step(plan, x, W, a, g, K, drop), load, eager)
    assert int(drop.state[1]) == 4                # one draw per replay, none at capture
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
        p.edge_pairs()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    w = torch.ones((8, 8), device=dev(), requires_grad=True)     # cuBLAS handles of this thread and of the autograd
    (w @ w).sum().backward()                                    # thread, which a capture cannot create
    rs = np.random.RandomState(5)
    ins = [(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.uniform(-1, 1, size=(n, f)).astype(np.float32),
            (rs.standard_normal((f, f)) * 0.1).astype(np.float32),
            (rs.standard_normal((2 * f // K, K)) * 0.1).astype(np.float32)) for _ in range(3)]
    made = []

    def buffers(r):
        m = lps[r].m
        b = dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()),
                 W=torch.zeros((f, f), device=dev(), requires_grad=True),
                 a=torch.zeros((2 * f // K, K), device=dev(), requires_grad=True), drop=EdgeDropout(0.5, KEY, dev()))
        made.append(b)
        return b

    def load(bufs, i):
        H, G, Wn, an = ins[i]
        with torch.no_grad():
            for r, lp in enumerate(lps):
                b = bufs[r]
                b["x"].copy_(torch.from_numpy(H[lp.owned])); b["g"].copy_(torch.from_numpy(G[lp.owned]))
                b["W"].copy_(torch.from_numpy(Wn)); b["a"].copy_(torch.from_numpy(an))
                if b is not made[r]:              # eager buffers draw with the counter the replay just used
                    b["drop"] = follower(made[r]["drop"])
        torch.cuda.synchronize()

    check_two_rank_capture(plans, streams, buffers, load,
                           lambda r, b: layer_step(plans[r], b["x"], b["W"], b["a"], b["g"], K, b["drop"]))
    for r in range(k):
        assert int(made[r]["drop"].state[1]) == 4
    for p in plans:
        p.close()


@pytest.mark.parametrize("heads,port", [(1, 29681), (2, 29682)])
def test_cli_attn_dropout_follows_the_fp64_loss_curve(tmp_path, heads, port):
    extra = ["--attn-dropout", "0.5"] + (["--heads", str(heads)] if heads > 1 else [])
    lines = run_cli(tmp_path, "PGAT.py", extra, port)
    assert_follows(lines, do.intended_training(karate(), 2, 4, 7, 1.0, 0.5, heads=heads))


def test_cli_attn_dropout_zero_prints_what_no_flag_prints(tmp_path):
    plain = run_cli(tmp_path, "PGAT.py", [], 29683)
    zero = run_cli(tmp_path, "PGAT.py", ["--attn-dropout", "0"], 29684)
    assert len(plain) == 50 and zero == plain
