"""Parity of the sm_90a path (called through the C-ABI, libpgcn_b200.so) against
  * the golden outputs of the unmodified reference (tests/golden, k = 1, 2, 3 ranks),
  * the fp64 truth within the fp32 bound of SURVEY.md §8a:  |Z - Z64| <= 2 d 2^-24 (|A||H|),
  * the CPU oracle on seeded R-MAT inputs with hubs, empty rows, duplicates, odd feature widths,
and, at the benchmark's full size, through size-independent properties (column-sum checksum,
adjointness <A H, G> == <H, A^T G>, linearity).

Every rank's plan lives on one GPU here: the kernels, the compact layout and the
pack / unpack kernels are exercised per rank, with the wire step replaced by a device copy in
wire order. The real transports (NCCL, peer memory) are covered by tests/test_multigpu.py.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import golden_cases
from harness import dev, t
from helpers import Golden, assert_close_fp32, fp32_tol
from oracle import build_oracle, pgcn_oracle as orc
from pgcn_b200 import graphio, plan as planmod

pytestmark = pytest.mark.gpu


def build_plans(A, partvec, k, f_max):
    from pgcn_b200 import op  # noqa: F401  (import checks the extension loads)
    return [planmod.build_plan(A, partvec, r, k, f_max, device=dev()) for r in range(k)]


def forward_all(plans, H, **opts):
    """Per-rank forward through pack -> (device copy in wire order) -> SpMM. Returns list of Z_own."""
    from pgcn_b200 import op
    k = len(plans)
    slabs = [op.pack_rows(p, t(H[p.lp.owned])) for p in plans]
    out = []
    for r, p in enumerate(plans):
        lp = p.lp
        for name, v in opts.items():
            p.set_option(name, v)
        parts = []
        for q in range(k):
            if q == r:
                continue
            lq = plans[q].lp
            parts.append(slabs[q][lq.send_off[r]:lq.send_off[r + 1]])
        halo = torch.cat(parts, 0) if parts and lp.h else torch.zeros((0, H.shape[1]), device=dev())
        assert halo.shape[0] == lp.h
        out.append(op.spmm_local(p, t(H[lp.owned]), halo if lp.h else None))
    return out


def backward_all(plans, G):
    """Per-rank backward: A^T g -> halo partials routed in wire order -> fixed-order scatter-add."""
    from pgcn_b200 import op
    k = len(plans)
    own, part = [], []
    for p in plans:
        g_own, g_halo = op.spmm_local(p, t(G[p.lp.owned]), transpose=True)
        own.append(g_own); part.append(g_halo)
    out = []
    for r, p in enumerate(plans):
        lp = p.lp
        recv = torch.zeros((lp.S, G.shape[1]), device=dev())
        for q in range(k):
            if q == r:
                continue
            lq = plans[q].lp
            recv[lp.send_off[q]:lp.send_off[q + 1]] = part[q][lq.recv_off[r]:lq.recv_off[r + 1]]
        out.append(op.unpack_add(p, recv, own[r].clone()))
    return out


@pytest.mark.parametrize("case", golden_cases())
def test_golden_forward_backward(case):
    g = Golden(case)
    plans = build_plans(g.A, g.partvec, g.k, g.f)
    Z = forward_all(plans, g.H)
    Gd = backward_all(plans, g.G)
    Z64 = orc.truth_forward(g.A, g.H)
    G64 = orc.truth_backward(g.A, g.G)
    tolZ = fp32_tol(g.A, g.H, int(orc.row_degree(g.A).max()))
    tolG = fp32_tol(g.A.T, g.G, int(orc.row_degree(g.A.T).max()))
    for r in range(g.k):
        own = g.owned(r)
        z = Z[r].cpu().numpy(); gd = Gd[r].cpu().numpy()
        assert_close_fp32(z, Z64[own], tolZ[own], "%s fwd r%d" % (case, r))
        assert_close_fp32(gd, G64[own], tolG[own], "%s bwd r%d" % (case, r))
        # the reference itself (PSpMM.forward under Q0; backward where Q3 does not bite)
        np.testing.assert_allclose(z, g.get(r, "Z1_own"), rtol=2e-5, atol=2e-6 * max(1.0, np.abs(Z64).max()))
        send, _ = g.maps(r)
        cnt = np.zeros(g.n, dtype=np.int64)
        for p_ in send:
            cnt[send[p_]] += 1
        single = cnt[own] < 2
        np.testing.assert_allclose(gd[single], g.get(r, "Hgrad_own")[single], rtol=2e-5,
                                   atol=2e-6 * max(1.0, np.abs(G64).max()))
    for p in plans:
        p.close()


def skewed_graph(n, nnz, seed):
    """R-MAT (unpermuted: hub rows up front) + a few empty rows + duplicate entries."""
    lo, hi = graphio.rmat_edges(n, nnz // 2, seed=seed, permute=False)
    A = graphio.gcn_normalise(graphio.symmetric_pattern(n, lo, hi)).tocoo()
    rng = np.random.RandomState(seed)
    dead = rng.choice(n, size=max(1, n // 50), replace=False)
    keep = ~np.isin(A.row, dead)
    row, col, val = A.row[keep], A.col[keep], A.data[keep]
    dup = rng.choice(row.shape[0], size=row.shape[0] // 20, replace=False)       # duplicates are summed
    row = np.concatenate([row, row[dup]]); col = np.concatenate([col, col[dup]]); val = np.concatenate([val, val[dup]])
    return sp.coo_matrix((val, (row, col)), shape=(n, n))


@pytest.mark.parametrize("f", [1, 3, 16, 20, 32, 64, 100, 128, 130, 256, 512, 640])
def test_feature_widths_vs_oracle(f):
    n = 3000
    A = skewed_graph(n, 60000, seed=7)
    rng = np.random.RandomState(f)
    H = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    pv = graphio.random_partvec(n, 2, seed=5)
    plans = build_plans(A, pv, 2, f)
    Z = forward_all(plans, H)
    Gd = backward_all(plans, G)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
    for r, p in enumerate(plans):
        lp = p.lp
        assert_close_fp32(Z[r].cpu().numpy(), Z64[lp.owned], tolZ[lp.owned], "fwd f=%d r%d" % (f, r))
        assert_close_fp32(Gd[r].cpu().numpy(), G64[lp.owned], tolG[lp.owned], "bwd f=%d r%d" % (f, r))
        # the C restatement of the GraphBLAS aggregation on the same rank data
        Hcat = np.concatenate([H[lp.owned], H[lp.halo]], 0)
        Zc = build_oracle.grb_aggregate(lp.rowptr, lp.colidx, lp.vals, Hcat, lp.recv_off, lp.m)
        np.testing.assert_allclose(Z[r].cpu().numpy(), Zc, rtol=3e-5, atol=3e-6)
        p.close()


@pytest.mark.parametrize("opts", [
    dict(edges_per_block=8), dict(edges_per_block=64, long_row=64), dict(edges_per_block=512),
    dict(edges_per_block=256, tile_floats=32), dict(edges_per_block=128, tile_floats=16),
    dict(edges_per_block=256, tile_floats=64), dict(edges_per_block=33), dict(edges_per_block=128, long_row=100000),
])
def test_schedule_options_do_not_change_results(opts):
    """Hubs split into segments, sub-warp feature tiles, unroll depths: same answer (and the split-row
    reduction is in a fixed order, so two runs are bit-identical)."""
    n, f = 4000, 128
    A = skewed_graph(n, 120000, seed=11)
    H = np.random.RandomState(1).uniform(-1, 1, size=(n, f)).astype(np.float32)
    plans = build_plans(A, np.zeros(n, dtype=np.int64), 1, f)
    Z64 = orc.truth_forward(A, H)
    tol = fp32_tol(A, H, int(orc.row_degree(A).max()))
    opts = dict(opts, kernel=4)                  # the register-pipeline kernel (the ring kernel has its own test)
    z1 = forward_all(plans, H, **opts)[0]
    z2 = forward_all(plans, H, **opts)[0]
    assert torch.equal(z1, z2)
    assert_close_fp32(z1.cpu().numpy(), Z64, tol, str(opts))
    if "long_row" in opts and opts["long_row"] <= 64:
        assert plans[0].get_option("long_rows_fwd") > 0
    plans[0].close()


@pytest.mark.parametrize("f", [128, 256, 384, 512])
@pytest.mark.parametrize("opts", [
    dict(kernel=5), dict(kernel=6), dict(kernel=5, ring_slots=16, ring_edges_per_block=64),
    dict(kernel=5, ring_slots=32, ring_edges_per_block=100, ring_long_row=150),
    dict(kernel=5, persistent=1, ring_edges_per_block=256), dict(kernel=6, persistent=1, ring_slots=16, ring_edges_per_block=77),
    dict(kernel=6, ring_slots=32, ring_edges_per_block=4096),
    dict(kernel=7), dict(kernel=7, ring_slots=16, ring_edges_per_block=90, persistent=0),
    dict(kernel=7, ring_slots=32, ring_edges_per_block=200), dict(kernel=7, ring_slots=64, ring_edges_per_block=300),
    dict(kernel=7, ring_slots=64, ring_groups=4, ring_edges_per_block=64, ring_long_row=100), dict(kernel=5, ring_slots=32, persistent=0),
])
def test_ring_kernel_matches_truth_and_register_kernel(f, opts):
    """The shared-memory ring SpMM (TMA bulk copies / cp.async into per-warp row slots): every ring depth,
    block size (blocks that start and end anywhere inside a 32-entry index piece, hub rows split into
    segments), persistent CTAs with dynamic block fetch, 2-rank plans with a halo slab, forward and
    transposed — same numbers as the fp64 truth within the fp32 bound, bit-identical run to run, and equal
    to the register-pipeline kernel within fp32 reassociation."""
    n = 4000
    A = skewed_graph(n, 120000, seed=11)
    rng = np.random.RandomState(f)
    H = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
    for k in (1, 2):
        pv = np.zeros(n, dtype=np.int64) if k == 1 else graphio.random_partvec(n, 2, seed=5)
        plans = build_plans(A, pv, k, f)
        z1 = forward_all(plans, H, **opts)
        z2 = forward_all(plans, H, **opts)
        gd = backward_all(plans, G)
        zr = forward_all(plans, H, kernel=4)
        for r, p in enumerate(plans):
            own = p.lp.owned
            assert torch.equal(z1[r], z2[r])
            assert_close_fp32(z1[r].cpu().numpy(), Z64[own], tolZ[own], "ring fwd %s f=%d k=%d r%d" % (opts, f, k, r))
            assert_close_fp32(gd[r].cpu().numpy(), G64[own], tolG[own], "ring bwd %s f=%d k=%d r%d" % (opts, f, k, r))
            torch.testing.assert_close(z1[r], zr[r], rtol=1e-4, atol=1e-5)
            if k == 1 and opts.get("ring_edges_per_block", 1024) <= 100:
                assert p.get_option("ring_long_rows_fwd") > 0
            p.close()


def test_empty_rank_and_tiny_graphs():
    row = np.array([0, 0, 0, 1, 2, 3, 4, 1]); col = np.array([1, 1, 3, 0, 4, 3, 0, 2])
    A = sp.coo_matrix((np.arange(1, 9, dtype=np.float64), (row, col)), shape=(6, 6))
    pv = np.array([0, 1, 0, 1, 0, 1])
    H = np.arange(24, dtype=np.float32).reshape(6, 4)
    plans = build_plans(A, pv, 3, 4)                      # rank 2 owns nothing
    Z = forward_all(plans, H)
    Gd = backward_all(plans, H)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, H)
    for r, p in enumerate(plans):
        np.testing.assert_allclose(Z[r].cpu().numpy(), Z64[p.lp.owned], rtol=1e-6)
        np.testing.assert_allclose(Gd[r].cpu().numpy(), G64[p.lp.owned], rtol=1e-6)
        assert Z[r].shape == (p.lp.m, 4)
        p.close()


def test_autograd_op_single_rank_matches_torch_sparse():
    """PSpMM.apply(A, H) on one rank vs the reference's own arithmetic torch.sparse.mm (GPU/PGCN.py:127,132)."""
    from pgcn_b200.op import PSpMM
    n, f = 2500, 48
    A = skewed_graph(n, 40000, seed=3)
    p = build_plans(A, np.zeros(n, dtype=np.int64), 1, f)[0]
    H = torch.randn(n, f, device=dev(), requires_grad=True)
    Z = PSpMM.apply(p, H)
    gz = torch.randn(n, f, device=dev())
    Z.backward(gz)
    At = torch.sparse_coo_tensor(torch.from_numpy(np.vstack([A.row, A.col]).astype(np.int64)),
                                 torch.from_numpy(A.data.astype(np.float32)), A.shape).to(dev())
    Hr = H.detach().clone().requires_grad_(True)
    Zr = torch.sparse.mm(At, Hr)
    Zr.backward(gz)
    torch.testing.assert_close(Z, Zr, rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(H.grad, Hr.grad, rtol=2e-5, atol=2e-5)
    # global layout: same call shape and output shape as the reference operator
    p.layout = "global"
    Zg = PSpMM.apply(p, H.detach())
    assert Zg.shape == (n, f)
    torch.testing.assert_close(Zg, Zr.detach(), rtol=2e-5, atol=2e-5)
    p.close()


def test_full_size_properties_config_C2():
    """BASELINE.json configs[1] (R-MAT 1 M / 16 M, f = 128) through size-independent checks."""
    from pgcn_b200 import op
    n, nnz, f = 1_000_000, 16_000_000, 128
    A = graphio.synthetic_graph(n, nnz, seed=1)
    p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    assert p.lp.nnz() == nnz + n
    gen = torch.Generator(device=dev()).manual_seed(1)
    H = torch.rand((n, f), device=dev(), generator=gen) * 2 - 1
    G = torch.rand((n, f), device=dev(), generator=gen) * 2 - 1
    Z = op.aggregate_forward(p, H)
    # (1) checksum: 1^T Z == (A^T 1)^T H, column sums of A from the plan arrays in fp64
    colsum = torch.from_numpy(np.bincount(p.lp.colidx, weights=p.lp.vals.astype(np.float64), minlength=n)).to(dev())
    lhs = Z.double().sum(0)
    rhs = colsum @ H.double()
    torch.testing.assert_close(lhs, rhs, rtol=1e-6, atol=1e-3)
    # (2) adjointness ties backward to forward: <A H, G> == <H, A^T G>
    GT = op.aggregate_backward(p, G)
    a = (Z.double() * G.double()).sum(); b = (H.double() * GT.double()).sum()
    assert abs(a - b) <= 1e-7 * max(abs(a), abs(b)) + 1e-2
    # (3) linearity: A (2 H + G) == 2 A H + A G
    ZG = op.aggregate_forward(p, G)
    Z3 = op.aggregate_forward(p, 2 * H + G)
    torch.testing.assert_close(Z3, 2 * Z + ZG, rtol=1e-4, atol=1e-4)
    # (4) a sample of rows against the fp64 truth (hub rows included)
    csr = sp.csr_matrix((p.lp.vals.astype(np.float64), p.lp.colidx, p.lp.rowptr), shape=(n, n))
    deg = np.diff(p.lp.rowptr)
    rows = np.concatenate([np.argsort(deg)[-64:], np.random.RandomState(0).choice(n, 4096, replace=False)])
    Hc = H.cpu().numpy()
    Zs64 = csr[rows] @ Hc.astype(np.float64)
    bound = abs(csr[rows]) @ np.abs(Hc.astype(np.float64))
    tol = 2.0 * (deg[rows, None] + 2) * 2.0 ** -24 * bound + 1e-30
    assert_close_fp32(Z[torch.from_numpy(rows).to(dev())].cpu().numpy(), Zs64, tol, "C2 sampled rows")
    # (5) idempotent scheduling: a different tiling gives the same numbers within fp32 reassociation
    p.set_option("tile_floats", 32); p.set_option("edges_per_block", 128)
    Zt = op.aggregate_forward(p, H)
    torch.testing.assert_close(Zt, Z, rtol=1e-4, atol=1e-5)
    p.close()


@pytest.mark.parametrize("case", ["gemat11_k2", "gemat11_k3_hp", "gemat11_k3_rp", "karate_k3_hp"])
def test_overlap_halves_equal_single_pass(case):
    """The own-columns / halo-columns kernels of the overlapped forward (what runs on > 1 GPU) on one GPU."""
    from pgcn_b200 import op
    g = Golden(case)
    plans = build_plans(g.A, g.partvec, g.k, g.f)
    Z = forward_all(plans, g.H)
    Z64 = orc.truth_forward(g.A, g.H)
    tol = fp32_tol(g.A, g.H, int(orc.row_degree(g.A).max()))
    for r, p in enumerate(plans):
        lp = p.lp
        if lp.h == 0:
            continue
        zs = op.spmm_split(p, t(g.H[lp.owned]), t(g.H[lp.halo]))
        assert_close_fp32(zs.cpu().numpy(), Z64[lp.owned], tol[lp.owned], "%s split r%d" % (case, r))
        np.testing.assert_allclose(zs.cpu().numpy(), g.get(r, "Z1_own"), rtol=2e-5, atol=2e-6 * max(1.0, np.abs(Z64).max()))
        torch.testing.assert_close(zs, Z[r], rtol=1e-4, atol=1e-5)
    for p in plans:
        p.close()


def test_autotune_keeps_results():
    n, f = 6000, 128
    A = skewed_graph(n, 150000, seed=13)
    H = np.random.RandomState(4).uniform(-1, 1, size=(n, f)).astype(np.float32)
    p = build_plans(A, np.zeros(n, dtype=np.int64), 1, f)[0]
    z0 = forward_all([p], H)[0]
    chosen = p.autotune(f)                       # f = 128: the ring kernel's block size is what gets tuned
    assert chosen in (256, 512, 1024) and p.get_option("ring_edges_per_block") == chosen
    assert p.get_option("ring_slots") in (16, 32)
    z1 = forward_all([p], H)[0]
    assert_close_fp32(z1.cpu().numpy(), orc.truth_forward(A, H), fp32_tol(A, H, int(orc.row_degree(A).max())), "autotuned")
    torch.testing.assert_close(z0, z1, rtol=1e-4, atol=1e-5)
    p.close()


def test_forward_host_entry_point():
    """pgcn_forward_host: the call a C host binds (host buffers in, host buffers out)."""
    import ctypes as C
    from pgcn_b200 import cabi
    n, f = 5000, 64
    A = skewed_graph(n, 80000, seed=5)
    p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    H = np.random.RandomState(2).uniform(-1, 1, size=(n, f)).astype(np.float32)
    Z = np.empty_like(H)
    cabi.check(cabi.load().pgcn_forward_host(p.handle, H.ctypes.data_as(C.c_void_p), Z.ctypes.data_as(C.c_void_p), f), p.handle)
    Z64 = orc.truth_forward(A, H)
    assert_close_fp32(Z, Z64, fp32_tol(A, H, int(orc.row_degree(A).max())), "forward_host")
    assert p.launch_count() >= 1
    b = p.algorithmic_bytes(f)
    assert b["nnz"] == p.lp.nnz() and b["spmm_fwd"] == 8 * b["nnz"] + 4 * (n + 1) + 4 * f * b["cols_ref"] + 4 * f * n
    p.close()


def test_forward_host_async_pipeline():
    """pgcn_forward_host_async / _wait: several steps in flight through the two device slots, each with its own
    input — every result must be the aggregation of ITS input (slot re-use hazards), equal to the serial call."""
    import ctypes as C
    from pgcn_b200 import cabi
    n, f = 8000, 128
    A = skewed_graph(n, 160000, seed=6)
    p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    lib = cabi.load()
    steps = 7
    Hs = [torch.from_numpy(np.random.RandomState(10 + i).uniform(-1, 1, size=(n, f)).astype(np.float32)).pin_memory()
          for i in range(steps)]
    Zs = [torch.empty((n, f), dtype=torch.float32).pin_memory() for _ in range(steps)]
    for i in range(steps):
        cabi.check(lib.pgcn_forward_host_async(p.handle, Hs[i].data_ptr(), Zs[i].data_ptr(), f), p.handle)
    cabi.check(lib.pgcn_forward_host_wait(p.handle), p.handle)
    tol = None
    for i in (0, 3, 6):
        Z64 = orc.truth_forward(A, Hs[i].numpy())
        tol = fp32_tol(A, Hs[i].numpy(), int(orc.row_degree(A).max()))
        assert_close_fp32(Zs[i].numpy(), Z64, tol, "async step %d" % i)
    Zser = torch.empty((n, f), dtype=torch.float32).pin_memory()
    for i in (1, 2, 4, 5):
        cabi.check(lib.pgcn_forward_host(p.handle, Hs[i].data_ptr(), Zser.data_ptr(), f), p.handle)
        assert torch.equal(Zser, Zs[i])
    p.close()
