"""Kernel census: every kernel instance in lib/libpgcn_b200.so is launched through a public entry point and its output is
checked against an fp64 reference.

  * tests/kernel_instances.txt lists the library's kernels (tools/list_kernels.py); the host test here rebuilds the list
    from the current library and compares, so an added or removed instance fails the CPU suite until the manifest and
    the route table below are updated;
  * ROUTES is the route table: one row per call shape (entry point, one or two ranks, f, heads, options, operands 4 bytes
    into their buffer) with the instances the host dispatch in csrc/pgcn_b200.cu must pick for it, derived from its
    rules (choose_tile, choose_tile_heads, vec_width, use_ring, launch_spmm's row tile and ring shape,
    sddmm_use_ring, sddmm_heads_use_ring, gatv2_use_ring, attn_vec). A CPU test checks that the rows name every
    instance of the manifest;
  * each row runs under torch.profiler and must launch the instances it names; its outputs are checked against fp64
    (sums within (d + 2) 2^-24 |A||H|, dot products within (f + 8) 2^-24 sum |g||h|, max values and arguments
    exactly, pack / unpack / halo copies exactly), and against the bits of the paired instances where the kernels
    promise identical bits (vector width 1 vs 4, ring row tiles 64 / 128 / 256, ring vs plain GATv2 scores);
  * the cold-column pass repeats one row per kernel family that decodes the cold flag with every column cold
    (PGCN_HOT_MB=0 at plan creation) and asserts the same bits, since the flag is only a cache hint;
  * the last test asserts that the instances seen across the file are exactly the manifest.

The inputs are an R-MAT graph with a hub row of 1 500 entries (long-row CTAs, rows split on both schedules), empty
rows, rows of one entry and duplicated entries, on one rank and on two ranks over the peer transport (both ranks on
this GPU, every two-rank call made twice so that both halves of the double-buffered halo slab are read).
"""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import sage_oracle as so
from conftest import ROOT
from harness import EPS, dev, edges, shifted, stream, t
from pgcn_b200 import cabi, graphio, plan as planmod

F_MAX = 512
SLOPE = 0.2
MANIFEST = os.path.join(ROOT, "tests", "kernel_instances.txt")


# ---- kernel names ----------------------------------------------------------------------------------------------------

def key(name):
    """Instance name without return type, parameter list, casts and spaces, bools as 0 / 1: the manifest's and the
    profiler's spellings of one instance give the same key."""
    s = name.strip()
    for a, b in (("(int)", ""), ("(bool)", ""), ("true", "1"), ("false", "0")):
        s = s.replace(a, b)
    if s.startswith("void "):
        s = s[5:]
    return s.split("(")[0].replace(" ", "")


def manifest():
    with open(MANIFEST) as fh:
        return [ln.rstrip("\n") for ln in fh if ln.strip()]


# Instances the census does not launch, each with its reason. Empty: every instance is reached.
EXCLUDED = {}


# ---- the dispatch rules, mirrored ------------------------------------------------------------------------------------

def pow2ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def lanes(nvec):
    return max(4, min(32, pow2ceil(nvec)))


def rowblock(f, vw, halo):
    """choose_tile without a tile_floats option."""
    tv = min(f // vw, 128)
    lpe = lanes(tv)
    vpl = -(-tv // lpe)
    vpl = 1 if vpl <= 1 else (2 if vpl <= 2 else 4)
    return "pgcn::spmm_rowblock_kernel<%d,%d,%d,%d>" % (lpe, vpl, vw, int(halo))


def heads_vw(f, K, shift):
    return 1 if (f // K) % 4 or shift else 4


def heads_inst(f, K, shift, halo):
    vw = heads_vw(f, K, shift)
    return "pgcn::spmm_heads_kernel<%d,%d,%d,%d>" % (lanes(f // vw), vw, int(halo), K)


def gatv2_insts(f, K, shift_xr, halo):
    vw = heads_vw(f, K, shift_xr)
    lpe = lanes(f // vw)
    return {"pgcn::gatv2_row_backward_kernel<%d,%d,%d,%d>" % (lpe, vw, int(halo), K),
            "pgcn::gatv2_col_backward_kernel<%d,%d,%d>" % (lpe, vw, K)}


def max_vw(f, shift):
    return 1 if f % 4 or shift else 4


def max_inst(f, shift, halo):
    vw = max_vw(f, shift)
    return "pgcn::spmm_max_kernel<%d,%d,%d>" % (lanes(f // vw), vw, int(halo))


def max_bwd_inst(f, shift):
    vw = max_vw(f, shift)
    return "pgcn::spmm_max_backward_kernel<%d,%d>" % (lanes(f // vw), vw)


RING_SHAPES = {(16, 2): (8, 2), (32, 2): (16, 2), (64, 2): (32, 2), (64, 4): (16, 4)}


def ring_inst(kernel, tf, slots, groups, halo):
    """launch_spmm's ring instance at f = 256 for the options kernel / ring_tile_floats / ring_slots / ring_groups."""
    if kernel == 6:
        return "pgcn::spmm_ring_kernel<%d,8,2,1,%d>" % (tf, int(halo))
    g, ng = RING_SHAPES[(slots, groups)]
    if kernel == 5:
        g, ng = (16, 2) if slots > 16 else (8, 2)
        return "pgcn::spmm_ring_kernel<%d,%d,%d,0,%d>" % (tf, g, ng, int(halo))
    return "pgcn::spmm_ring_tm_kernel<%d,%d,%d,%d>" % (tf, g, ng, int(halo))


def walk_extras(vw):
    """The empty-row zero-fill and split-row fixup of launch_walk (the census graph has both)."""
    return {"pgcn::zero_rows_kernel<%d>" % vw, "pgcn::spmm_fixup_kernel<%d>" % vw}


# ---- the route table -------------------------------------------------------------------------------------------------

class Route:
    def __init__(self, family, expect, **kw):
        self.family, self.expect, self.kw = family, set(expect), kw
        self.id = family + "-" + "-".join("%s%s" % (k, int(v) if isinstance(v, bool) else v) for k, v in kw.items())


def build_routes():
    R = []
    # register SpMM (kernel = 4): both vector widths at each f (the scalar one from a shifted H), both transposes
    for ranks in (1, 2):
        halo = ranks == 2
        for f in (16, 32, 64, 128, 256, 512):
            R.append(Route("spmm", {rowblock(f, 4, halo), rowblock(f, 1, halo)} | walk_extras(4) | walk_extras(1),
                           ranks=ranks, f=f, tr=0, pair=True))
        for f in (3, 7):
            R.append(Route("spmm", {rowblock(f, 1, halo)} | walk_extras(1), ranks=ranks, f=f, tr=0, pair=False))
        R.append(Route("spmm", {rowblock(32, 4, False), rowblock(32, 1, False)}, ranks=ranks, f=32, tr=1, pair=True))
    # ring SpMM at f = 256: every row tile, ring shape and fill, with and without the halo operand
    for ranks in (1, 2):
        halo = ranks == 2
        for (slots, groups) in RING_SHAPES:
            R.append(Route("ring", {ring_inst(0, tf, slots, groups, halo) for tf in (64, 128, 256)},
                           ranks=ranks, kernel=0, slots=slots, groups=groups))
        for slots in (16, 32):
            R.append(Route("ring", {ring_inst(5, tf, slots, 2, halo) for tf in (64, 128, 256)},
                           ranks=ranks, kernel=5, slots=slots, groups=2))
        R.append(Route("ring", {ring_inst(6, tf, 16, 2, halo) for tf in (128, 256)}, ranks=ranks, kernel=6, slots=16,
                       groups=2))
    R.append(Route("ring_tr", {ring_inst(0, 256, 16, 2, False)}))
    # pack / unpack, the fused forward and backward over the peer transport (puts, waits, epochs, halo copies)
    # (the peer transport carries whole 4-float rows; the forward puts gather from the caller's H, whose alignment
    # picks the put's vector width)
    for f in (16, 15):
        vw = 4 if f % 4 == 0 else 1
        R.append(Route("pack", {"pgcn::pack_rows_kernel<%d>" % vw, "pgcn::unpack_add_kernel<%d>" % vw}, f=f))
    for shift in (False, True):
        for overlap in (0, 1):
            R.append(Route("fused", {"pgcn::put_rows_kernel<%d>" % (1 if shift else 4), "pgcn::p2p_wait_kernel",
                                     "pgcn::epoch_advance_kernel", "pgcn::copy_halo_kernel"}, f=16, overlap=overlap,
                           shift=shift))
    R.append(Route("pack", {"pgcn::pack_rows_kernel<1>", "pgcn::unpack_add_kernel<1>"}, f=16, shift=True))
    R.append(Route("values", {"pgcn::set_values_kernel"}))
    # SDDMM: the ring instance of each f / 128 and the plain kernel, one and two ranks
    for f in (128, 256, 384, 512):
        R.append(Route("sddmm", {"pgcn::sddmm_ring_kernel<%d>" % (f // 128)}, ranks=1, f=f, shift=False))
    R.append(Route("sddmm", {"pgcn::sddmm_ring_kernel<1>"}, ranks=2, f=128, shift=False))
    R.append(Route("sddmm", {"pgcn::sddmm_plain_kernel"}, ranks=1, f=128, shift=True))
    R.append(Route("sddmm", {"pgcn::sddmm_plain_kernel"}, ranks=2, f=40, shift=False))
    for f in (128, 256, 512):
        for K in (2, 4, 8):
            R.append(Route("sddmm_heads", {"pgcn::sddmm_heads_ring_kernel<%d,%d>" % (f // 128, K)}, f=f, K=K,
                           shift=False))
    R.append(Route("sddmm_heads", {"pgcn::sddmm_plain_heads_kernel"}, f=128, K=4, shift=True))
    R.append(Route("sddmm_heads", {"pgcn::sddmm_plain_heads_kernel"}, f=40, K=2, shift=False))
    # edge softmax, single and multi-head, vector and scalar loads of the K values
    R.append(Route("softmax", {"pgcn::edge_softmax_kernel<1,0>", "pgcn::edge_softmax_backward_kernel<1,0>"}, K=1,
                   shift=False))
    for K in (2, 4, 8):
        for shift in (False, True):
            v = int(not shift)
            R.append(Route("softmax", {"pgcn::edge_softmax_kernel<%d,%d>" % (K, v),
                                       "pgcn::edge_softmax_backward_kernel<%d,%d>" % (K, v)}, K=K, shift=shift))
    # multi-head aggregation and max aggregation: every lane count and vector width, with and without the halo
    for ranks in (1, 2):
        halo = ranks == 2
        for f in (4, 8, 16, 32, 64, 128):
            for K in (1, 2, 4, 8):
                if f % K:
                    continue
                for shift in (False, True):
                    R.append(Route("heads", {heads_inst(f, K, shift, halo)} | ({heads_inst(f, K, shift, False)}
                                                                                if not halo else set()),
                                   ranks=ranks, f=f, K=K, shift=shift))
            for shift in (False, True):
                e = {max_inst(f, shift, halo), "pgcn::max_empty_rows_kernel<%d>" % max_vw(f, shift),
                     "pgcn::spmm_max_fixup_kernel<%d>" % max_vw(f, shift)}
                R.append(Route("max", e | ({max_bwd_inst(f, shift)} if not halo else set()), ranks=ranks, f=f,
                               shift=shift))
    # GATv2: scores (ring at f = 128 / 256 with aligned operands, else plain), the raw softmax, both backward walks
    for ranks in (1, 2):
        halo = ranks == 2
        for f in (4, 8, 16, 32, 64, 128):
            for K in (1, 2, 4, 8):
                if f % K:
                    continue
                for shift in (False, True):
                    e = gatv2_insts(f, K, shift, halo) | {"pgcn::gatv2_datt_kernel"}
                    if f == 128 and not shift:
                        e.add("pgcn::gatv2_score_ring_kernel<1,%d>" % K)
                    else:
                        e.add("pgcn::gatv2_score_plain_kernel")
                    v = int(K > 1)
                    e |= {"pgcn::edge_softmax_raw_kernel<%d,%d>" % (K, v),
                          "pgcn::edge_softmax_raw_backward_kernel<%d,%d>" % (K, v)}
                    R.append(Route("gatv2", e, ranks=ranks, f=f, K=K, shift=shift, shift_alpha=False))
    for K in (1, 2, 4, 8):
        R.append(Route("gatv2", {"pgcn::gatv2_score_ring_kernel<2,%d>" % K}, ranks=1, f=256, K=K, shift=False,
                       shift_alpha=False))
        if K > 1:
            R.append(Route("gatv2", {"pgcn::edge_softmax_raw_kernel<%d,0>" % K,
                                     "pgcn::edge_softmax_raw_backward_kernel<%d,0>" % K},
                           ranks=1, f=16, K=K, shift=False, shift_alpha=True))
    R.append(Route("autotune", {"fill_hash_kernel"}))
    return R


ROUTES = build_routes()


def test_route_table_names_every_instance_of_the_manifest():
    named = set().union(*(r.expect for r in ROUTES))
    want = {key(n) for n in manifest()} - set(EXCLUDED)
    assert not (named - {key(n) for n in manifest()}), "routes name instances the library lacks: %s" % sorted(
        named - {key(n) for n in manifest()})
    assert not (want - named), "instances no route reaches: %s" % sorted(want - named)


def test_manifest_matches_the_library():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import list_kernels
    finally:
        sys.path.pop(0)
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not found")
    from pgcn_b200 import build
    build.build()                                      # rebuilds a missing or stale library
    got = list_kernels.list_kernels()
    want = manifest()
    assert got == want, ("the library's kernels differ from tests/kernel_instances.txt (python tools/list_kernels.py "
                         "--write, and add a route for each new instance): added %s, removed %s"
                         % (sorted(set(got) - set(want)), sorted(set(want) - set(got))))


# ---- GPU fixtures ----------------------------------------------------------------------------------------------------

def nan_like(x, shift=False):
    y = torch.full_like(x, float("nan")) if x.dtype.is_floating_point else torch.full_like(x, -7)
    return shifted(y) if shift else y


def ptr(x):
    return None if x is None else x.data_ptr()


def census_graph():
    """R-MAT (2 500 vertices), row 0 a hub of 1 500 entries, rows 10..19 empty, rows 20..29 of one entry, 500 entries
    stored twice (summed into one entry of value 2 by the plan), values in [0.5, 1.5)."""
    A = sp.coo_matrix(graphio.synthetic_graph(2500, 25000, seed=17))
    keep = (A.row >= 30)
    rs = np.random.RandomState(3)
    row = np.concatenate([A.row[keep], np.zeros(1500, np.int64), np.arange(20, 30)])
    col = np.concatenate([A.col[keep], np.arange(1500), np.arange(20, 30) + 700])
    dup = rs.choice(len(row), 500, replace=False)
    row, col = np.concatenate([row, row[dup]]), np.concatenate([col, col[dup]])
    val = np.ones(len(row), np.float32)
    B = sp.csr_matrix((val, (row, col)), shape=A.shape)
    B.sum_duplicates()
    B.data = (B.data * rs.uniform(0.5, 1.5, B.nnz)).astype(np.float32)
    return B.tocoo()


class Problem:
    def __init__(self, hot_mb=None):
        d = dev()
        self.A = census_graph()
        n = self.A.shape[0]
        self.n = n
        self.pv = graphio.random_partvec(n, 2, seed=5)
        self.p1 = planmod.build_plan(self.A, np.zeros(n, dtype=np.int64), 0, 1, F_MAX, device=d)
        self.p1.bind_values()
        lps = [planmod.build_local_plan(self.A, self.pv, r, 2) for r in range(2)]
        self.p2 = [planmod.PgcnPlan(lp, F_MAX, device=d) for lp in lps]
        planmod.link_local_plans(self.p2)
        for p in self.p2:
            p.bind_values()
        self.streams = [torch.cuda.Stream(device=d) for _ in self.p2]
        lp = self.p1.lp
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > 1024 and (deg == 0).any() and (deg == 1).any() and lp.vals.max() > 1.5
        assert all(p.lp.h > 0 for p in self.p2)

    def close(self):
        for p in [self.p1] + self.p2:
            p.close()


@pytest.fixture(scope="module")
def prob():
    P = Problem()
    yield P
    P.close()


SEEN = set()


def launched(fn):
    """Run fn under torch.profiler; (fn's result, the keys of the kernels it launched)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


def run_ranks(P, fn):
    """fn(r) for both ranks, each on its own stream, every rank's work enqueued before the synchronisation."""
    torch.cuda.synchronize()
    out = [None, None]
    for r, s in enumerate(P.streams):
        with torch.cuda.stream(s):
            out[r] = fn(r)
    torch.cuda.synchronize()
    return out


def set_opts(plans, **opts):
    for p in plans:
        for k, v in opts.items():
            p.set_option(k, v)


DEFAULTS = dict(kernel=0, ring_slots=16, ring_groups=2, ring_tile_floats=0, overlap=1)


def reset(P):
    for p in [P.p1] + P.p2:
        for k, v in DEFAULTS.items():
            if p.get_option(k) != v:
                p.set_option(k, v)


# ---- fp64 references -------------------------------------------------------------------------------------------------

def local_csr(lp):
    return sp.csr_matrix((lp.vals.astype(np.float64), lp.colidx, lp.rowptr), shape=(lp.m, lp.m + lp.h))


def cat(lp, X):
    return X[np.concatenate([lp.owned, lp.halo])] if lp.k > 1 else X


def assert_sum(got, M, X, what):
    """got ~ M @ X: |err| <= (d + 2) 2^-24 (|M| |X|) with d the row's entry count."""
    M = sp.csr_matrix(M)
    want = np.asarray(M @ X.astype(np.float64))
    mag = np.asarray(abs(M) @ np.abs(X.astype(np.float64)))
    deg = np.diff(M.indptr)[:, None]
    err = np.abs(got.astype(np.float64) - want)
    tol = (deg + 2) * EPS * mag + 1e-30
    assert np.isfinite(got).all() and (err <= tol).all(), "%s: %d entries beyond the fp32 bound, worst %.3e" % (
        what, int((err > tol).sum()), float((err - tol).max()))


def assert_bits(a, b, what):
    assert torch.equal(a, b), "%s: the bits differ" % what


def feats(seed, rows, f):
    return np.random.RandomState(seed).uniform(-1, 1, (rows, f)).astype(np.float32)


# ---- the rows --------------------------------------------------------------------------------------------------------

def run_spmm(P, ranks, f, tr, pair):
    lib = cabi.load()
    plans = [P.p1] if ranks == 1 else P.p2[:1]
    set_opts(plans, kernel=4)
    p = plans[0]
    lp = p.lp
    X = feats(f, P.n, f)
    Hown, Hhalo = t(X[lp.owned] if ranks > 1 else X), (t(X[lp.halo]) if ranks > 1 else None)
    outs = []
    for shift in ([False, True] if pair else [False]):
        h0 = shifted(Hown) if shift else Hown
        Z = nan_like(Hown, shift)
        Zh = torch.full((max(lp.h, 1), f), float("nan"), device=dev())
        if tr:
            cabi.check(lib.pgcn_spmm(p.handle, 1, h0.data_ptr(), None, Z.data_ptr(), Zh.data_ptr() if lp.h else None,
                                     f, stream()), p.handle)
        else:
            cabi.check(lib.pgcn_spmm(p.handle, 0, h0.data_ptr(), ptr(Hhalo), Z.data_ptr(), None, f, stream()),
                       p.handle)
        outs.append((Z.clone(), Zh[:lp.h].clone()))
    M = local_csr(lp)
    if tr:
        Xo = X[lp.owned] if ranks > 1 else X
        G = outs[0][0].cpu().numpy()
        assert_sum(G, M.T.tocsr()[:lp.m], Xo, "A^T g, own rows")
        if lp.h:
            assert_sum(outs[0][1].cpu().numpy(), M.T.tocsr()[lp.m:], Xo, "A^T g, halo partials")
    else:
        assert_sum(outs[0][0].cpu().numpy(), M, cat(lp, X), "A H")
    if pair:
        assert_bits(outs[0][0], outs[1][0], "vector width 4 vs 1")
        if tr:
            assert_bits(outs[0][1], outs[1][1], "vector width 4 vs 1, halo partials")


def run_ring(P, ranks, kernel, slots, groups):
    lib = cabi.load()
    f = 256
    p = P.p1 if ranks == 1 else P.p2[0]
    lp = p.lp
    X = feats(7, P.n, f)
    Hown, Hhalo = t(X[lp.owned] if ranks > 1 else X), (t(X[lp.halo]) if ranks > 1 else None)
    set_opts([p], kernel=kernel, ring_slots=slots, ring_groups=groups)
    outs = []
    for tf in ((128, 256) if kernel == 6 else (64, 128, 256)):
        p.set_option("ring_tile_floats", tf)
        Z = nan_like(Hown)
        cabi.check(lib.pgcn_spmm(p.handle, 0, Hown.data_ptr(), ptr(Hhalo), Z.data_ptr(), None, f, stream()), p.handle)
        outs.append(Z)
    assert_sum(outs[0].cpu().numpy(), local_csr(lp), cat(lp, X), "ring A H")
    for Z in outs[1:]:
        assert_bits(outs[0], Z, "ring row tiles")


def run_ring_tr(P):
    lib = cabi.load()
    f = 256
    lp = P.p1.lp
    X = feats(8, P.n, f)
    H = t(X)
    G = nan_like(H)
    cabi.check(lib.pgcn_spmm(P.p1.handle, 1, H.data_ptr(), None, G.data_ptr(), None, f, stream()), P.p1.handle)
    assert_sum(G.cpu().numpy(), local_csr(lp).T.tocsr(), X, "ring A^T g")


def run_pack(P, f, shift=False):
    p = P.p2[0]
    lp = p.lp
    lib = cabi.load()
    X = feats(f, lp.m, f)
    H = shifted(t(X)) if shift else t(X)
    slab = nan_like(torch.empty((lp.S, f), device=dev()), shift)
    cabi.check(lib.pgcn_pack(p.handle, H.data_ptr(), slab.data_ptr(), f, stream()), p.handle)
    assert np.array_equal(slab.cpu().numpy(), X[lp.send_idx]), "pack is not the send rows"
    recv = feats(f + 1, lp.S, f)
    G0 = feats(f + 2, lp.m, f)
    G = shifted(t(G0)) if shift else t(G0)
    R = shifted(t(recv)) if shift else t(recv)
    cabi.check(lib.pgcn_unpack_add(p.handle, R.data_ptr(), G.data_ptr(), f, stream()), p.handle)
    want = G0.copy()
    np.add.at(want, lp.send_idx, recv)        # fp32, one add per element (distinct rows per peer on two ranks)
    assert np.array_equal(G.cpu().numpy(), want), "unpack_add is not the fp32 sum"


def run_fused(P, f, overlap, shift):
    lib = cabi.load()
    set_opts(P.p2, overlap=overlap, kernel=4)
    X, Y = feats(11, P.n, f), feats(12, P.n, f)
    for _ in range(2):                       # both parities of the halo slab
        Hs = [shifted(t(X[p.lp.owned])) if shift else t(X[p.lp.owned]) for p in P.p2]
        Gs = [t(Y[p.lp.owned]) for p in P.p2]
        Z = [nan_like(h) for h in Hs]
        Hh = [torch.full((p.lp.h, f), float("nan"), device=dev()) for p in P.p2]
        B = [nan_like(g) for g in Gs]
        run_ranks(P, lambda r: cabi.check(lib.pgcn_forward_keep_halo(P.p2[r].handle, Hs[r].data_ptr(), Z[r].data_ptr(),
                                                                     Hh[r].data_ptr(), f, stream()), P.p2[r].handle))
        run_ranks(P, lambda r: cabi.check(lib.pgcn_backward(P.p2[r].handle, Gs[r].data_ptr(), B[r].data_ptr(), f,
                                                            stream()), P.p2[r].handle))
        A = P.A.tocsr()
        for r, p in enumerate(P.p2):
            own = p.lp.owned
            assert_sum(Z[r].cpu().numpy(), A[own], X, "fused forward, rank %d" % r)
            assert_sum(B[r].cpu().numpy(), A.T.tocsr()[own], Y, "fused backward, rank %d" % r)
            assert np.array_equal(Hh[r].cpu().numpy(), X[p.lp.halo]), "kept halo rows"


def run_values(P):
    lib = cabi.load()
    p = P.p1
    lp = p.lp
    f = 32
    vals = np.random.RandomState(9).uniform(-1, 1, lp.nnz()).astype(np.float32)
    X = feats(13, P.n, f)
    H = t(X)
    Z = nan_like(H)
    try:
        p.set_values(t(vals))
        cabi.check(lib.pgcn_forward(p.handle, H.data_ptr(), Z.data_ptr(), f, stream()), p.handle)
    finally:
        p.set_values(None)
    M = sp.csr_matrix((vals.astype(np.float64), lp.colidx, lp.rowptr), shape=(lp.m, lp.m))
    assert_sum(Z.cpu().numpy(), M, X, "A(vals) H")


def dots(rows, cols, g, h, K):
    d = g.shape[1] // K
    P = g.astype(np.float64)[rows] * h.astype(np.float64)[cols]
    return P.reshape(-1, K, d).sum(2), np.abs(P).reshape(-1, K, d).sum(2), d


def run_sddmm(P, ranks, f, shift):
    lib = cabi.load()
    p = P.p1 if ranks == 1 else P.p2[0]
    lp = p.lp
    g, X = feats(f + 3, lp.m, f), feats(f + 4, P.n, f)
    gd, Hown = t(g), t(X[lp.owned] if ranks > 1 else X)
    Hhalo = t(X[lp.halo]) if ranks > 1 else None
    if shift:
        gd, Hown = shifted(gd), shifted(Hown)
    out = torch.full((lp.nnz(),), float("nan"), device=dev())
    cabi.check(lib.pgcn_sddmm(p.handle, gd.data_ptr(), Hown.data_ptr(), ptr(Hhalo), out.data_ptr(), f, stream()),
               p.handle)
    rows, cols = edges(lp)
    want, mag, d = dots(rows, cols, g, cat(lp, X), 1)
    err = np.abs(out.cpu().numpy().astype(np.float64)[:, None] - want)
    assert (err <= (d + 8) * EPS * mag + 1e-30).all(), "sddmm beyond the bound"


def run_sddmm_heads(P, f, K, shift):
    lib = cabi.load()
    p = P.p1
    lp = p.lp
    g, X = feats(f + 5, lp.m, f), feats(f + 6, lp.m, f)
    gd, H = t(g), t(X)
    if shift:
        gd, H = shifted(gd), shifted(H)
    out = torch.full((lp.nnz(), K), float("nan"), device=dev())
    cabi.check(lib.pgcn_sddmm_heads(p.handle, K, gd.data_ptr(), H.data_ptr(), None, out.data_ptr(), f, stream()),
               p.handle)
    rows, cols = edges(lp)
    want, mag, d = dots(rows, cols, g, X, K)
    err = np.abs(out.cpu().numpy().astype(np.float64) - want)
    assert (err <= (d + 8) * EPS * mag + 1e-30).all(), "sddmm_heads beyond the bound"


def run_softmax(P, K, shift):
    lib = cabi.load()
    p = P.p1
    lp = p.lp
    rs = np.random.RandomState(K + 20 * shift)
    el, er = rs.uniform(-4, 4, (lp.m, K)).astype(np.float32), rs.uniform(-4, 4, (lp.m, K)).astype(np.float32)
    dal = rs.uniform(-1, 1, (lp.nnz(), K)).astype(np.float32)
    e, r_, da = t(el), t(er), t(dal)
    if shift:
        e = shifted(e)
    alpha = torch.full((lp.nnz(), K), float("nan"), device=dev())
    dpre = torch.full_like(alpha, float("nan"))
    d_el = torch.full((lp.m, K), float("nan"), device=dev())
    if K == 1:
        cabi.check(lib.pgcn_edge_softmax(p.handle, e.data_ptr(), r_.data_ptr(), None, SLOPE, alpha.data_ptr(),
                                         stream()), p.handle)
        cabi.check(lib.pgcn_edge_softmax_backward(p.handle, e.data_ptr(), r_.data_ptr(), None, alpha.data_ptr(),
                                                  da.data_ptr(), SLOPE, dpre.data_ptr(), d_el.data_ptr(), stream()),
                   p.handle)
    else:
        cabi.check(lib.pgcn_edge_softmax_heads(p.handle, K, e.data_ptr(), r_.data_ptr(), None, SLOPE, alpha.data_ptr(),
                                               stream()), p.handle)
        cabi.check(lib.pgcn_edge_softmax_backward_heads(p.handle, K, e.data_ptr(), r_.data_ptr(), None,
                                                        alpha.data_ptr(), da.data_ptr(), SLOPE, dpre.data_ptr(),
                                                        d_el.data_ptr(), stream()), p.handle)
    check_softmax(lp, el, er, dal, [u.cpu().numpy() for u in (alpha, dpre, d_el)], K)


def check_softmax(lp, el, er, dal, got, K):
    """The bounds of test_multihead_attention's softmax test."""
    rows, cols = edges(lp)
    deg = np.diff(lp.rowptr.astype(np.int64))
    for h in range(K):
        alpha, dpre, d_el = (x[:, h].astype(np.float64) for x in got)
        s = el[:, h].astype(np.float64)[rows] + er[:, h].astype(np.float64)[cols]
        s = np.where(s > 0, s, SLOPE * s)
        mx = np.full(lp.m, -np.inf)
        np.maximum.at(mx, rows, s)
        ex = np.exp(s - mx[rows])
        a64 = ex / np.bincount(rows, ex, minlength=lp.m)[rows]
        smax = np.zeros(lp.m)
        np.maximum.at(smax, rows, np.abs(s))
        assert (np.abs(alpha - a64) <= a64 * EPS * (8 * smax[rows] + 4 * deg[rows] + 32) + 1e-38).all(), \
            "head %d: alpha beyond the bound" % h
        d64 = dal[:, h].astype(np.float64)
        c = np.bincount(rows, alpha * d64, minlength=lp.m)
        cmag = np.bincount(rows, np.abs(alpha * d64), minlength=lp.m)
        sl = np.where(s > 0, 1.0, SLOPE)
        p64 = alpha * (d64 - c[rows]) * sl
        tol_p = sl * alpha * EPS * (4 * np.abs(d64) + 4 * np.abs(c[rows]) + 2 * (deg[rows] + 4) * cmag[rows]) + 1e-38
        assert (np.abs(dpre - p64) <= tol_p).all(), "head %d: dpre beyond the bound" % h
        e64 = np.bincount(rows, p64, minlength=lp.m)
        tol_e = np.bincount(rows, tol_p + (deg[rows] + 4) * EPS * np.abs(p64), minlength=lp.m) + 1e-38
        assert (np.abs(d_el - e64) <= tol_e).all(), "head %d: d_el beyond the bound" % h


def heads_ref(M, alpha, X, K):
    """Per head h: A(alpha[:, h]) X[:, head h] as sparse matrices sharing M's pattern (forward CSR order)."""
    d = X.shape[1] // K
    return [(sp.csr_matrix((alpha[:, h].astype(np.float64), M.indices, M.indptr), shape=M.shape),
             X[:, h * d:(h + 1) * d]) for h in range(K)]


def assert_heads(got, M, alpha, X, K, what):
    d = X.shape[1] // K
    for h, (Mh, Xh) in enumerate(heads_ref(M, alpha, X, K)):
        assert_sum(got[:, h * d:(h + 1) * d], Mh, Xh, "%s, head %d" % (what, h))


def run_heads(P, ranks, f, K, shift):
    lib = cabi.load()
    X, Y = feats(f * 8 + K, P.n, f), feats(f * 8 + K + 1, P.n, f)
    if ranks == 1:
        p = P.p1
        lp = p.lp
        alpha = np.random.RandomState(K).uniform(0, 1, (lp.nnz(), K)).astype(np.float32)
        outs = []
        for sh in ([False, True] if not shift else [True]):
            H, G, a = t(X), t(Y), t(alpha)
            if sh:
                H, G, a = shifted(H), shifted(G), shifted(a)
            Z, B = nan_like(H, sh), nan_like(H, sh)
            cabi.check(lib.pgcn_forward_heads(p.handle, K, a.data_ptr(), H.data_ptr(), Z.data_ptr(), None, f,
                                              stream()), p.handle)
            cabi.check(lib.pgcn_backward_heads(p.handle, K, a.data_ptr(), G.data_ptr(), B.data_ptr(), f, stream()),
                       p.handle)
            outs.append((Z, B))
        M = local_csr(lp)
        assert_heads(outs[0][0].cpu().numpy(), M, alpha, X, K, "heads forward")
        assert_heads(outs[0][1].cpu().numpy(), M.T.tocsr(), alpha[local_csr_t_order(lp)], Y, K, "heads backward")
        if len(outs) == 2:
            assert_bits(outs[0][0], outs[1][0], "heads forward, aligned vs shifted")
            assert_bits(outs[0][1], outs[1][1], "heads backward, aligned vs shifted")
        return
    alphas = [np.random.RandomState(K + r).uniform(0, 1, (p.lp.nnz(), K)).astype(np.float32)
              for r, p in enumerate(P.p2)]
    for _ in range(2):
        Hs = [t(X[p.lp.owned]) for p in P.p2]
        As = [t(a) for a in alphas]
        if shift:
            Hs = [shifted(h) for h in Hs]
        Z = [nan_like(h, shift) for h in Hs]
        Hh = [torch.full((p.lp.h, f), float("nan"), device=dev()) for p in P.p2]
        run_ranks(P, lambda r: cabi.check(lib.pgcn_forward_heads(P.p2[r].handle, K, As[r].data_ptr(), Hs[r].data_ptr(),
                                                                 Z[r].data_ptr(), Hh[r].data_ptr(), f, stream()),
                                          P.p2[r].handle))
        for r, p in enumerate(P.p2):
            assert_heads(Z[r].cpu().numpy(), local_csr(p.lp), alphas[r], cat(p.lp, X), K, "heads forward rank %d" % r)
            assert np.array_equal(Hh[r].cpu().numpy(), X[p.lp.halo]), "heads: kept halo rows"


def local_csr_t_order(lp):
    """For each entry of the transposed records (CSC of the forward matrix, rows sorted), its forward entry."""
    rows, cols = edges(lp)
    order = np.lexsort((rows, cols))
    return order


def run_max(P, ranks, f, shift):
    lib = cabi.load()
    X, Y = feats(f * 3 + 1, P.n, f), feats(f * 3 + 2, P.n, f)
    if ranks == 1:
        p = P.p1
        lp = p.lp
        outs = []
        for sh in ([False, True] if not shift else [True]):
            H, G = t(X), t(Y)
            if sh:
                H, G = shifted(H), shifted(G)
            Z = nan_like(H, sh)
            arg = nan_like(torch.empty((lp.m, f), dtype=torch.int32, device=dev()), sh)
            cabi.check(lib.pgcn_forward_max(p.handle, H.data_ptr(), Z.data_ptr(), arg.data_ptr(), f, stream()),
                       p.handle)
            B = nan_like(H, sh)
            cabi.check(lib.pgcn_backward_max(p.handle, arg.data_ptr(), G.data_ptr(), B.data_ptr(), f, stream()),
                       p.handle)
            outs.append((Z, arg, B))
        Zw, argw = so.max_aggregate(lp.rowptr, lp.colidx, X)
        assert np.array_equal(outs[0][0].cpu().numpy(), Zw) and np.array_equal(outs[0][1].cpu().numpy(), argw), \
            "max values / arguments differ from the oracle"
        check_max_backward(outs[0][2].cpu().numpy(), lp.colidx, argw, Y, lp.m)
        if len(outs) == 2:
            for a, b, w in zip(outs[0], outs[1], ("Z", "arg", "G")):
                assert_bits(a, b, "max %s, aligned vs shifted" % w)
        return
    for _ in range(2):
        Hs = [t(X[p.lp.owned]) for p in P.p2]
        if shift:
            Hs = [shifted(h) for h in Hs]
        Z = [nan_like(h, shift) for h in Hs]
        args = [nan_like(torch.empty((p.lp.m, f), dtype=torch.int32, device=dev()), shift) for p in P.p2]
        run_ranks(P, lambda r: cabi.check(lib.pgcn_forward_max(P.p2[r].handle, Hs[r].data_ptr(), Z[r].data_ptr(),
                                                               args[r].data_ptr(), f, stream()), P.p2[r].handle))
        for r, p in enumerate(P.p2):
            Zw, argw = so.max_aggregate(p.lp.rowptr, p.lp.colidx, cat(p.lp, X))
            assert np.array_equal(Z[r].cpu().numpy(), Zw) and np.array_equal(args[r].cpu().numpy(), argw), \
                "rank %d: max values / arguments differ from the oracle" % r


def check_max_backward(G, colidx, arg, gZ, ncols):
    want = so.max_backward(colidx, arg, gZ, ncols)
    i, c = np.nonzero(arg >= 0)
    mag = np.zeros_like(want)
    cnt = np.zeros_like(want)
    np.add.at(mag, (np.asarray(colidx)[arg[i, c]], c), np.abs(gZ[i, c]).astype(np.float64))
    np.add.at(cnt, (np.asarray(colidx)[arg[i, c]], c), 1.0)
    assert (np.abs(G.astype(np.float64) - want) <= (cnt + 2) * EPS * mag + 1e-30).all(), "max backward beyond bound"


def gatv2_inputs(f, K, n, seed):
    rs = np.random.RandomState(seed)
    xl = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    xr = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    att = (rs.standard_normal((K, f // K)) / np.sqrt(f // K)).astype(np.float32)
    gZ = rs.uniform(-1, 1, (n, f)).astype(np.float32)
    return xl, xr, att, gZ


def gatv2_fwd(p, K, xl, xr, att, xl_halo_out, shift_alpha):
    lib = cabi.load()
    lp = p.lp
    f = xl.shape[1]
    alpha = nan_like(torch.empty((lp.nnz(), K), device=dev()), shift_alpha)
    Z = nan_like(torch.empty((lp.m, f), device=dev()))
    cabi.check(lib.pgcn_forward_gatv2(p.handle, K, xl.data_ptr(), xr.data_ptr(), att.data_ptr(), SLOPE,
                                      alpha.data_ptr(), Z.data_ptr(), ptr(xl_halo_out), f, stream()), p.handle)
    return alpha, Z


def gatv2_bwd(p, K, alpha, Z, xl, xr, att, gZ, xl_halo, shift_alpha):
    lib = cabi.load()
    f = xl.shape[1]
    work = nan_like(alpha, shift_alpha)
    dxl, dxr = nan_like(Z), nan_like(Z)
    datt = torch.full((K, f // K), float("nan"), device=dev())
    cabi.check(lib.pgcn_backward_gatv2(p.handle, K, alpha.data_ptr(), gZ.data_ptr(), xl.data_ptr(), ptr(xl_halo),
                                       xr.data_ptr(), att.data_ptr(), SLOPE, work.data_ptr(), dxl.data_ptr(),
                                       dxr.data_ptr(), datt.data_ptr(), f, stream()), p.handle)
    return alpha, Z, dxl, dxr, datt


def gatv2_call(p, K, xl, xr, att, gZ, shift_alpha=False):
    """Forward then backward of one rank on one rank's plan; (alpha, Z, dxl, dxr, datt)."""
    alpha, Z = gatv2_fwd(p, K, xl, xr, att, None, shift_alpha)
    return gatv2_bwd(p, K, alpha, Z, xl, xr, att, gZ, None, shift_alpha)


def run_gatv2(P, ranks, f, K, shift, shift_alpha):
    from test_gatv2 import bounds, check
    xl, xr, att, gZ = gatv2_inputs(f, K, P.n, f * 10 + K)
    if ranks == 1:
        p = P.p1
        lp = p.lp
        outs = []
        for sh in ([False, True] if shift else [False]):
            xrd = shifted(t(xr)) if sh else t(xr)
            outs.append([u.clone() for u in gatv2_call(p, K, t(xl), xrd, t(att), t(gZ), shift_alpha)])
        rows, cols = edges(lp)
        got = [u.cpu().numpy() for u in outs[0]]
        check(got, bounds(rows, cols, lp.m, xl, xr, att, SLOPE, gZ, got[0]), what="f=%d K=%d: " % (f, K))
        if shift:
            for name, a, b in zip(("alpha", "Z", "dxl", "dxr", "datt"), outs[0], outs[1]):
                assert_bits(a, b, "GATv2 %s, aligned vs shifted xr (ring vs plain scores, VW 4 vs 1)" % name)
        return
    # two ranks: the global problem's fp64 values and bounds, alpha mapped to global entry order
    A = P.A.tocsr()
    grows = np.repeat(np.arange(P.n), np.diff(A.indptr))
    gcols = A.indices.astype(np.int64)
    gkeys = grows * P.n + gcols
    for _ in range(2):
        ops = []
        for p in P.p2:
            own = p.lp.owned
            xrd = shifted(t(xr[own])) if shift else t(xr[own])
            ops.append((t(xl[own]), xrd, t(att), t(gZ[own]), torch.empty((p.lp.h, f), device=dev())))
        fw = run_ranks(P, lambda r: gatv2_fwd(P.p2[r], K, ops[r][0], ops[r][1], ops[r][2], ops[r][4], False))
        res = run_ranks(P, lambda r: gatv2_bwd(P.p2[r], K, fw[r][0], fw[r][1], ops[r][0], ops[r][1], ops[r][2],
                                               ops[r][3], ops[r][4], False))
        for r, p in enumerate(P.p2):
            assert np.array_equal(ops[r][4].cpu().numpy(), xl[p.lp.halo]), "GATv2: kept halo rows"
        alpha_g = np.zeros((len(gkeys), K), np.float32)
        for r, p in enumerate(P.p2):
            rows, cols = edges(p.lp)
            gc = cat(p.lp, np.arange(P.n))
            idx = np.searchsorted(gkeys, p.lp.owned[rows] * P.n + gc[cols])
            alpha_g[idx] = res[r][0].cpu().numpy()
        ref = bounds(grows, gcols, P.n, xl, xr, att, SLOPE, gZ, alpha_g)
        check([alpha_g], ref, names=("alpha",), what="2 ranks f=%d K=%d: " % (f, K))
        for r, p in enumerate(P.p2):
            own = p.lp.owned
            sub = {k: (v[0][own], v[1][own]) for k, v in ref.items() if k in ("Z", "dxl", "dxr")}
            check([res[r][i].cpu().numpy() for i in (1, 2, 3)], sub, names=("Z", "dxl", "dxr"),
                  what="rank %d f=%d K=%d: " % (r, f, K))
        datt = res[0][4].cpu().numpy().astype(np.float64) + res[1][4].cpu().numpy()
        want, tol = ref["datt"]
        assert (np.abs(datt - want) <= 2 * tol).all(), "2 ranks: datt beyond the bound"


def run_autotune(P):
    """autotune (the hashed fill of its timing operands), then SDDMM, GATv2 and max calls on the tuned schedules."""
    d = dev()
    p = planmod.build_plan(P.A, np.zeros(P.n, dtype=np.int64), 0, 1, F_MAX, device=d)
    try:
        p.bind_values()
        p.autotune(256)
        P2 = type("P", (), {})()
        P2.p1, P2.n, P2.A = p, P.n, P.A
        run_sddmm(P2, 1, 256, False)
        run_gatv2(P2, 1, 256, 2, False, False)
        run_max(P2, 1, 32, False)
    finally:
        p.close()


RUNNERS = {
    "spmm": run_spmm, "ring": run_ring, "ring_tr": run_ring_tr, "pack": run_pack, "fused": run_fused,
    "values": run_values, "sddmm": run_sddmm, "sddmm_heads": run_sddmm_heads, "softmax": run_softmax,
    "heads": run_heads, "max": run_max, "gatv2": run_gatv2, "autotune": run_autotune,
}


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES, ids=[r.id for r in ROUTES])
def test_route(prob, route):
    # torch.profiler now and then loses the activity records of a session (none at all, or only a copy): the row, whose
    # checks pass each time, is run again; a dispatch that picks another instance misses it every time
    names = set()
    for _ in range(3):
        try:
            _, got = launched(lambda: RUNNERS[route.family](prob, **route.kw))
        finally:
            reset(prob)
        names |= got
        if route.expect <= names:
            break
    assert names, "torch.profiler recorded no CUDA kernel"
    SEEN.update(names)
    missing = route.expect - names
    assert not missing, "%s no longer launches %s (it launched %s)" % (route.id, sorted(missing), sorted(names))


# ---- cold columns ----------------------------------------------------------------------------------------------------

def cold_rows(P):
    """One call per kernel family that decodes the cold flag of a column or a piece's cold masks; their outputs."""
    lib = cabi.load()
    outs = {}
    p, lp = P.p1, P.p1.lp

    def spmm(kernel, f):
        X = t(feats(f, P.n, f))
        set_opts([p], kernel=kernel)
        Z = nan_like(X)
        cabi.check(lib.pgcn_spmm(p.handle, 0, X.data_ptr(), None, Z.data_ptr(), None, f, stream()), p.handle)
        G = nan_like(X)
        cabi.check(lib.pgcn_spmm(p.handle, 1, X.data_ptr(), None, G.data_ptr(), None, f, stream()), p.handle)
        set_opts([p], kernel=0)
        return Z, G
    outs["register"] = spmm(4, 32)
    outs["ring256"] = spmm(0, 256)
    outs["ring128"] = spmm(0, 128)
    for f, K in ((32, 2), (128, 8)):
        X = t(feats(f, P.n, f))
        a = t(np.random.RandomState(K).uniform(0, 1, (lp.nnz(), K)).astype(np.float32))
        Z, B = nan_like(X), nan_like(X)
        cabi.check(lib.pgcn_forward_heads(p.handle, K, a.data_ptr(), X.data_ptr(), Z.data_ptr(), None, f, stream()),
                   p.handle)
        cabi.check(lib.pgcn_backward_heads(p.handle, K, a.data_ptr(), X.data_ptr(), B.data_ptr(), f, stream()),
                   p.handle)
        outs["heads%d" % f] = (Z, B)
    for f in (33, 128):
        X = t(feats(f, P.n, f))
        Z = nan_like(X)
        arg = torch.full((lp.m, f), -7, dtype=torch.int32, device=dev())
        cabi.check(lib.pgcn_forward_max(p.handle, X.data_ptr(), Z.data_ptr(), arg.data_ptr(), f, stream()), p.handle)
        B = nan_like(X)
        cabi.check(lib.pgcn_backward_max(p.handle, arg.data_ptr(), X.data_ptr(), B.data_ptr(), f, stream()), p.handle)
        outs["max%d" % f] = (Z, arg, B)
    for f, K in ((128, 2), (40, 4)):
        xl, xr, att, gZ = (t(x) for x in gatv2_inputs(f, K, P.n, 99))
        outs["gatv2_%d" % f] = gatv2_call(p, K, xl, xr, att, gZ)
    for f, sh in ((256, False), (40, True)):
        g, X = t(feats(f + 1, P.n, f)), t(feats(f + 2, P.n, f))
        if sh:
            g, X = shifted(g), shifted(X)
        out = torch.full((lp.nnz(),), float("nan"), device=dev())
        cabi.check(lib.pgcn_sddmm(p.handle, g.data_ptr(), X.data_ptr(), None, out.data_ptr(), f, stream()), p.handle)
        out4 = torch.full((lp.nnz(), 4), float("nan"), device=dev())
        cabi.check(lib.pgcn_sddmm_heads(p.handle, 4, g.data_ptr(), X.data_ptr(), None, out4.data_ptr(), f, stream()),
                   p.handle)
        outs["sddmm%d" % f] = (out, out4)
    torch.cuda.synchronize()
    return outs


@pytest.mark.gpu
def test_cold_columns_give_the_same_bits(prob, monkeypatch):
    hot = cold_rows(prob)
    monkeypatch.setenv("PGCN_HOT_MB", "0")
    cold = type("P", (), {})()
    cold.n, cold.A = prob.n, prob.A
    cold.p1 = planmod.build_plan(prob.A, np.zeros(prob.n, dtype=np.int64), 0, 1, F_MAX, device=dev())
    try:
        cold.p1.bind_values()
        got = cold_rows(cold)
    finally:
        cold.p1.close()
    for name in hot:
        for i, (a, b) in enumerate(zip(hot[name], got[name])):
            assert_bits(a, b, "%s output %d, every column cold vs the default hot set" % (name, i))


# ---- completeness ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_every_instance_was_launched_and_checked():
    """Runs last in this file: the instances the rows above launched are exactly the library's."""
    want = {key(n) for n in manifest()}
    seen = SEEN & want
    routed = sum(1 for r in ROUTES)
    if not SEEN:
        pytest.fail("no route ran before this test (run the whole file)")
    missing = want - seen - set(EXCLUDED)
    assert not missing, "%d instances never launched: %s" % (len(missing), sorted(missing))
    print("\n%d/%d kernels launched and checked (%d routes, %d excluded)" % (len(seen), len(want), routed,
                                                                            len(EXCLUDED)))
