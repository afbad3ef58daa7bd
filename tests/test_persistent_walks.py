"""Persistent ring walks at many work items per warp.

Every ring kernel is a persistent walk: a warp takes a work item (a row block of one row tile) from the plan's counter,
walks it and takes the next, and the grid is capped at the CTAs the device holds at once. State that lives from one item
to the next (the group-barrier phase bits, the index-piece FIFO counters, the accumulators, the row tile, the halo
slab's parity) is only read on a warp's second and later items, which the census's small graphs rarely reach. Here
every launch has at least 4 items per warp the device could hold:

    items >= 4 * SMs * W,   W = min(64, floor(233 472 / (16 * TF * 4)))

233 472 B is an SM's shared memory and every ring warp holds at least 16 row slots of TF floats (TF: the row tile, 64 /
128 / 256 for the SpMM, 128 NV for the edge rings), so W bounds the resident warps whatever occupancy the library
picks; items = blocks * (f / TF). The rows use ring_edges_per_block = 64 (the ring's minimum) and ring_long_row = 96,
so the hub rows split into many segments; each row asserts and prints its item count against the bound.

  * ROUTES is a route table in the census's style: one row per call shape naming the instances it must launch, run
    under torch.profiler. Its oracles, beside an fp64 bound and run-to-run bits in every row:
      - ring SpMM, one rank, forward and transposed, every kernel / slot / group / row tile: the bits of the same call
        with persistent = 0 (the same instance and schedule, one item per warp). Every output element sums the same
        products in the same order whichever warp walks its block, and split rows are reduced in a fixed order;
      - the HALO instances, two ranks, overlap = 0: pgcn_spmm with a halo operand, and the fused forward and backward,
        each called twice so that both halves of the double-buffered slabs are read: the bits of persistent = 0;
      - persistent_multi = 1 with overlap = 1: the fused forward (relu = 1) and backward, each called twice (own part
        and per-peer halo blocks, reading H_odd / tm_odd): the bits of persistent_multi = 0;
      - the SDDMM, multi-head SDDMM and GATv2 score rings: the bits of a few-item schedule (a block size that leaves
        fewer blocks than SMs). sddmm_heads_ring_walk computes an edge's value from its slot in its aligned 8-entry
        group, its gZ / xr row and its H / xl row only: a block's bounds only mask other edges' partials, which the
        butterfly reduces in other positions, so the block cut cannot change a bit. GATv2 scores also keep the bits
        of gatv2_score_plain_kernel (xr 4 bytes into its buffer);
  * a plan made with PGCN_HOT_MB=1 (a few hundred hot rows at full width, a few thousand in 64-float slices, the rest
    cold) repeats one many-item row per ring family with the default plan's bits;
  * CUDA-graph capture and replay at many items (one rank: forward + backward; two ranks: persistent_multi), every
    replay resetting the counter;
  * the grid-capped copies (put_rows_kernel at 4 CTAs per SM, pack_rows_kernel, copy_halo_kernel and
    set_values_kernel at 32) run at least 4 grid strides and are checked exactly;
  * a host test asserts that the route table names every ring instance of the manifest, and the last GPU test that
    each was launched by a row whose precondition held.

The graph is test_gpu_parity's skewed R-MAT at 200 000 vertices (2.6 M stored entries: hub rows up front, empty rows,
summed duplicates) with planted one-entry rows, on one rank and on two ranks over the peer transport. The fp64
references are computed once, at f = 512, by plain float64 gathers, products and index_add_ on the device (the CPU
helpers of the census take seconds per call at this size); a narrower width reads their first f columns.
"""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from harness import EPS, check_one_rank_capture, check_two_rank_capture, dev, edges, linked_plans, run_ranks, shifted, \
    stream
from test_gpu_parity import skewed_graph
from test_kernel_census import SLOPE, Route, gatv2_fwd, gatv2_inputs, key, launched, manifest, ring_inst
from pgcn_b200 import cabi, graphio, plan as planmod

F_MAX = 512
N = 200_000
SMEM = 233_472                # bytes of shared memory per H100 SM
EPB, LONG = 64, 96            # the many-item schedule: the ring's smallest block, hub rows split into segments
FEW = 1 << 16                 # the few-item schedule of the edge rings: fewer blocks than SMs
CHUNK = 1 << 16               # entries per step of the fp64 references
NAN = float("nan")
SPMM_SHAPES = [(7, 16, 2), (7, 32, 2), (7, 64, 2), (7, 64, 4), (5, 16, 2), (5, 32, 2), (6, 16, 2)]   # kernel, slots, groups


# ---- the route table -------------------------------------------------------------------------------------------------

def row_tiles(kernel, f):
    """The ring row tiles launch_spmm runs at width f: those that divide f, 128 and up with the cp.async fill."""
    return [tf for tf in (64, 128, 256) if f % tf == 0 and not (kernel == 6 and tf < 128)]


def spmm_insts(kernel, slots, groups, f, halo):
    return {ring_inst(0 if kernel == 7 else kernel, tf, slots, groups, halo) for tf in row_tiles(kernel, f)}


def build_routes():
    R = []
    for (kernel, slots, groups) in SPMM_SHAPES:
        for f in (128, 256, 384, 512):
            R.append(Route("ring", spmm_insts(kernel, slots, groups, f, False), kernel=kernel, slots=slots,
                           groups=groups, f=f))
    for (kernel, slots, groups) in SPMM_SHAPES:
        R.append(Route("ring_halo", spmm_insts(kernel, slots, groups, 256, True)
                       | spmm_insts(kernel, slots, groups, 256, False), kernel=kernel, slots=slots, groups=groups, f=256))
        R.append(Route("ring_multi", spmm_insts(kernel, slots, groups, 256, False), kernel=kernel, slots=slots,
                       groups=groups, f=256))
    for ranks in (1, 2):
        for f in (128, 256, 384, 512):
            R.append(Route("sddmm", {"pgcn::sddmm_ring_kernel<%d>" % (f // 128)}, ranks=ranks, f=f))
    for f in (128, 256, 512):
        for K in (2, 4, 8):
            R.append(Route("sddmm_heads", {"pgcn::sddmm_heads_ring_kernel<%d,%d>" % (f // 128, K)}, f=f, K=K))
    for ranks in (1, 2):
        for f in (128, 256):
            for K in (1, 2, 4, 8):
                R.append(Route("gatv2", {"pgcn::gatv2_score_ring_kernel<%d,%d>" % (f // 128, K),
                                         "pgcn::gatv2_score_plain_kernel"}, ranks=ranks, f=f, K=K))
    return R


ROUTES = build_routes()


def ring_manifest():
    return {key(n) for n in manifest() if "_ring_" in n}


def test_route_table_names_every_persistent_instance():
    named = set().union(*(r.expect for r in ROUTES))
    want = ring_manifest()
    assert not (named - {key(n) for n in manifest()}), "routes name instances the library lacks: %s" % sorted(
        named - {key(n) for n in manifest()})
    assert not (want - named), "ring instances without a many-item row: %s" % sorted(want - named)


# ---- the problem -----------------------------------------------------------------------------------------------------

def graph():
    """skewed_graph at 200 000 vertices, with 16 of its empty rows planted with one entry each (to a hub column)."""
    A = skewed_graph(N, 2_500_000, seed=11)
    empty = np.flatnonzero(np.bincount(A.row, minlength=N) == 0)[:16]
    rs = np.random.RandomState(4)
    row = np.concatenate([A.row, empty])
    col = np.concatenate([A.col, rs.randint(0, 64, empty.size)])
    val = np.concatenate([A.data, rs.uniform(0.5, 1.5, empty.size)]).astype(np.float32)
    return sp.coo_matrix((val, (row, col)), shape=A.shape)


def spmm_ref(rows, cols, vals, X, nrows):
    """(M X in fp64, its fp32 bound (d + 2) 2^-24 |M||X| rounded up to fp32) for the entries (rows, cols, vals)."""
    want = torch.zeros((nrows, X.shape[1]), dtype=torch.float64, device=dev())
    mag = torch.zeros_like(want)
    for s in range(0, rows.numel(), CHUNK):
        P = vals[s:s + CHUNK, None] * X[cols[s:s + CHUNK]].double()
        want.index_add_(0, rows[s:s + CHUNK], P)
        mag.index_add_(0, rows[s:s + CHUNK], P.abs_())
    deg = torch.bincount(rows, minlength=nrows).double()[:, None]
    tol = ((deg + 2) * EPS * mag + 1e-30).float()
    del mag
    return want, torch.nextafter(tol, torch.full_like(tol, float("inf")))


def edge_ref(rows, cols, G, H, K):
    """Per entry and head: sum over the head's d features of G[row] H[col] in fp64, and the bound (d + 8) 2^-24 sum |.|."""
    f = G.shape[1]
    d = f // K
    want = torch.empty((rows.numel(), K), dtype=torch.float64, device=dev())
    mag = torch.empty_like(want)
    for s in range(0, rows.numel(), CHUNK):
        P = (G[rows[s:s + CHUNK]].double() * H[cols[s:s + CHUNK]].double()).view(-1, K, d)
        want[s:s + CHUNK] = P.sum(2)
        mag[s:s + CHUNK] = P.abs_().sum(2)
    return want, (d + 8) * EPS * mag + 1e-30


def alpha_ref(rows, grows, gcols, nrows, xl, xr, att):
    """GATv2 attention (nnz x K) in fp64 over the entries of an nrows-row matrix (rows: their rows, the softmax
    groups; grows / gcols: the rows of xr and xl they read), with test_gatv2.bounds' per-entry fp32 bound."""
    K, d = att.shape
    a64 = att.double()
    s = torch.empty((rows.numel(), K), dtype=torch.float64, device=dev())
    ds = torch.empty_like(s)
    for c in range(0, rows.numel(), CHUNK):
        L, R = xl[gcols[c:c + CHUNK]].double(), xr[grows[c:c + CHUNK]].double()
        tt = L + R
        s[c:c + CHUNK] = (torch.where(tt > 0, tt, SLOPE * tt).view(-1, K, d) * a64[None]).sum(2)
        ds[c:c + CHUNK] = EPS * (d + 8) * ((L.abs_() + R.abs_()).view(-1, K, d) * a64.abs()[None]).sum(2)
    idx = rows[:, None].expand(-1, K)
    mx = torch.full((nrows, K), -float("inf"), dtype=torch.float64, device=dev()).scatter_reduce(0, idx, s, "amax")
    ex = torch.exp(s - mx[rows])
    den = torch.zeros((nrows, K), dtype=torch.float64, device=dev()).index_add_(0, rows, ex)
    a = ex / den[rows]
    zero = torch.zeros((nrows, K), dtype=torch.float64, device=dev())
    dmax = zero.scatter_reduce(0, idx, ds, "amax")
    smax = zero.scatter_reduce(0, idx, s.abs(), "amax")
    deg = torch.bincount(rows, minlength=nrows).double()[:, None]
    return a, a * (2 * ds + 2 * dmax[rows] + EPS * (8 * smax[rows] + 4 * deg[rows] + 32)) + 1e-38


def check_close(got, want, tol, what):
    err = (got.double() - want).abs_()
    bad = ~(err <= tol)
    nbad = int(bad.sum())
    assert nbad == 0, "%s: %d entries beyond the fp32 bound (worst excess %.3e)" % (
        what, nbad, float((err - tol).nan_to_num(float("inf")).max()))


def assert_bits(a, b, what):
    assert torch.equal(a, b) and torch.equal(a.view(torch.int32), b.view(torch.int32)), "%s: the bits differ" % what


def sched_blocks(counts, epb=EPB, long_row=LONG):
    """Ring blocks of a matrix whose rows hold `counts` entries (empty rows squeezed out, as the plan uploads it)."""
    c = np.asarray(counts, np.int64)
    rp = np.ascontiguousarray(np.concatenate([[0], np.cumsum(c[c > 0])]).astype(np.int32))
    n = cabi.load().pgcn_debug_schedule(rp.ctypes.data_as(C.c_void_p), len(rp) - 1, epb, long_row, None, 0, None, None)
    return cabi.check(int(n))


def part_counts(lp):
    """Row entry counts of the matrices a two-rank plan launches: forward, transposed, own-column part, the peer's
    halo block, and the transposed own rows and peer rows of the pipelined backward."""
    rows, cols = edges(lp)
    q = 1 - lp.rank
    lo, hi = lp.m + lp.recv_off[q], lp.m + lp.recv_off[q + 1]
    return dict(fwd=np.diff(lp.rowptr), tr=np.diff(lp.t_rowptr),
                own=np.bincount(rows[cols < lp.m], minlength=lp.m),
                halo=np.bincount(rows[(cols >= lo) & (cols < hi)], minlength=lp.m),
                tr_own=np.diff(lp.t_rowptr[:lp.m + 1]), tr_halo=np.diff(lp.t_rowptr[lo:hi + 1]))


RATIOS = []


def many_items(what, blocks, f, tf):
    """Assert the many-item precondition of a launch of `blocks` row blocks at width f and row tile tf: at least 4
    items per warp the device could hold."""
    sms = torch.cuda.get_device_properties(dev()).multi_processor_count
    warps = sms * min(64, SMEM // (16 * tf * 4))
    items = blocks * (f // tf)
    print("  %s: %d items, %.2f per resident warp (bound %d)" % (what, items, items / warps, warps))
    assert items >= 4 * warps, "%s: %d items, fewer than 4 per resident warp (%d warps)" % (what, items, warps)
    RATIOS.append(items / warps)


def set_opts(plans, **opts):
    for p in plans:
        for k, v in opts.items():
            p.set_option(k, v)


BASE = dict(kernel=0, ring_slots=16, ring_groups=2, ring_tile_floats=0, ring_edges_per_block=EPB, ring_long_row=LONG,
            persistent=1, persistent_multi=0, relu=0)


def many(plans, **opts):
    """The many-item options, then `opts`."""
    set_opts(plans, **dict(BASE, **opts))


class Problem:
    def __init__(self):
        d = dev()
        A = graph()
        self.p1 = planmod.build_plan(A, np.zeros(N, dtype=np.int64), 0, 1, F_MAX, device=d)
        self.p1.bind_values()
        lp = self.p1.lp
        pv = graphio.random_partvec(N, 2, seed=5)
        self.lps = [planmod.build_local_plan(A, pv, r, 2) for r in range(2)]
        self.p2 = linked_plans(self.lps, F_MAX, 1)
        self.streams = [torch.cuda.Stream(device=d) for _ in self.p2]
        rs = np.random.RandomState(21)
        self.X = torch.from_numpy(rs.uniform(-1, 1, (N, F_MAX)).astype(np.float32)).to(d)
        self.Y = torch.from_numpy(rs.uniform(-1, 1, (N, F_MAX)).astype(np.float32)).to(d)
        rows, cols = edges(lp)
        self.rows, self.cols = torch.from_numpy(rows).to(d), torch.from_numpy(cols).to(d)
        vals = torch.from_numpy(lp.vals.astype(np.float64)).to(d)
        self.AX = spmm_ref(self.rows, self.cols, vals, self.X, N)            # forward
        self.ATY = spmm_ref(self.cols, self.rows, vals, self.Y, N)           # transposed
        self.own = [torch.from_numpy(l.owned).to(d) for l in self.lps]
        # global row and column of every entry of each rank's local matrix
        self.grows, self.gcols = [], []
        for l in self.lps:
            r, c = edges(l)
            self.grows.append(torch.from_numpy(l.owned[r]).to(d))
            self.gcols.append(torch.from_numpy(np.concatenate([l.owned, l.halo])[c]).to(d))
        self.counts1 = dict(fwd=np.diff(lp.rowptr), tr=np.diff(lp.t_rowptr))
        self.counts2 = [part_counts(l) for l in self.lps]
        deg = np.diff(lp.rowptr)
        assert deg.max() > 64 * 100 and (deg == 0).any() and (deg == 1).sum() > 16 and lp.nnz() > 2_400_000

    def ref(self, which, f, rows=None, relu=False):
        want, tol = getattr(self, which)
        want, tol = want[:, :f], tol[:, :f]
        if rows is not None:
            want, tol = want[rows], tol[rows]
        return (want.clamp(min=0) if relu else want), tol

    def close(self):
        for p in [self.p1] + self.p2:
            p.close()


@pytest.fixture(scope="module")
def prob():
    free, _ = torch.cuda.mem_get_info(dev())
    if free < 12 * 2 ** 30:
        pytest.skip("needs 12 GiB of free device memory, %.1f GiB free (the GPU is shared)" % (free / 2 ** 30))
    P = Problem()
    yield P
    P.close()


def spmm(p, tr, H, Hh, f, Zh=None):
    Z = torch.full((p.lp.m, f), NAN, device=dev())
    cabi.check(cabi.load().pgcn_spmm(p.handle, tr, H.data_ptr(), None if Hh is None else Hh.data_ptr(), Z.data_ptr(),
                                     None if Zh is None else Zh.data_ptr(), f, stream()), p.handle)
    return Z


def fused(P, f, calls, X_in, Y_in):
    """`calls` fused forwards on both ranks, then as many backwards: [(Z per rank)], [(G per rank)]. Each call moves
    the exchange epoch on by one, so consecutive calls read the two halves of the double-buffered slabs."""
    lib = cabi.load()
    Hs = [X_in[o, :f].contiguous() for o in P.own]
    Gs = [Y_in[o, :f].contiguous() for o in P.own]
    Zs, Bs = [], []
    for _ in range(calls):
        Z = [torch.full_like(h, NAN) for h in Hs]
        run_ranks(P.p2, lambda r: cabi.check(lib.pgcn_forward(P.p2[r].handle, Hs[r].data_ptr(), Z[r].data_ptr(), f,
                                                              stream()), P.p2[r].handle), P.streams)
        Zs.append(Z)
    for _ in range(calls):
        B = [torch.full_like(g, NAN) for g in Gs]
        run_ranks(P.p2, lambda r: cabi.check(lib.pgcn_backward(P.p2[r].handle, Gs[r].data_ptr(), B[r].data_ptr(), f,
                                                               stream()), P.p2[r].handle), P.streams)
        Bs.append(B)
    return Zs, Bs


# ---- the rows --------------------------------------------------------------------------------------------------------

def run_ring(P, kernel, slots, groups, f):
    p = P.p1
    many([p], kernel=kernel, ring_slots=slots, ring_groups=groups)
    tr_blocks = sched_blocks(P.counts1["tr"])
    first = {}
    for tf in row_tiles(kernel, f):
        p.set_option("ring_tile_floats", tf)
        for tr, X, which in ((0, P.X, "AX"), (1, P.Y, "ATY")):
            H = X[:, :f].contiguous()
            outs = []
            for pers in (1, 1, 0):
                p.set_option("persistent", pers)
                outs.append(spmm(p, tr, H, None, f))
            p.set_option("persistent", 1)
            blocks = tr_blocks if tr else p.get_option("ring_blocks_fwd")
            if not tr:
                assert blocks == sched_blocks(P.counts1["fwd"]), "the host mirror of the schedule is off"
            what = "%s f=%d tf=%d" % ("A^T g" if tr else "A H", f, tf)
            many_items(what, blocks, f, tf)
            check_close(outs[0], *P.ref(which, f), what=what)
            assert_bits(outs[0], outs[1], what + ", run to run")
            assert_bits(outs[0], outs[2], what + ", persistent vs one item per warp")
            if tr in first:
                assert_bits(first[tr], outs[0], what + " vs the first row tile")
            first.setdefault(tr, outs[0])


def run_ring_halo(P, kernel, slots, groups, f):
    """Two ranks, overlap = 0 (persistent HALO launches): pgcn_spmm with a halo operand on rank 0, and the fused forward
    and backward of both ranks."""
    p = P.p2[0]
    lp = p.lp
    many(P.p2, kernel=kernel, ring_slots=slots, ring_groups=groups, overlap=0)
    H = P.X[P.own[0], :f].contiguous()
    Hh = P.X[torch.from_numpy(lp.halo).to(dev()), :f].contiguous()
    try:
        for tf in row_tiles(kernel, f):
            set_opts(P.p2, ring_tile_floats=tf)
            outs = []
            for pers in (1, 1, 0):
                p.set_option("persistent", pers)
                outs.append(spmm(p, 0, H, Hh, f))
            p.set_option("persistent", 1)
            what = "rank 0 A [H | halo] f=%d tf=%d" % (f, tf)
            many_items(what, p.get_option("ring_blocks_fwd"), f, tf)
            check_close(outs[0], *P.ref("AX", f, P.own[0]), what=what)
            assert_bits(outs[0], outs[1], what + ", run to run")
            assert_bits(outs[0], outs[2], what + ", persistent vs one item per warp")
            res = {}
            for pers in (1, 0):
                set_opts(P.p2, persistent=pers)
                res[pers] = fused(P, f, 2, P.X, P.Y)
            set_opts(P.p2, persistent=1)
            for r in range(2):
                many_items("rank %d fused A^T g tf=%d" % (r, tf), sched_blocks(P.counts2[r]["tr"]), f, tf)
                for i in range(2):
                    w = "rank %d fused call %d tf=%d" % (r, i, tf)
                    check_close(res[1][0][i][r], *P.ref("AX", f, P.own[r]), what=w + ", forward")
                    check_close(res[1][1][i][r], *P.ref("ATY", f, P.own[r]), what=w + ", backward")
                    for j in range(2):
                        assert_bits(res[1][j][0][r], res[1][j][i][r], w + ", both slab parities")
                        assert_bits(res[1][j][i][r], res[0][j][i][r], w + ", persistent vs one item per warp")
    finally:
        set_opts(P.p2, overlap=1, persistent=1)


def run_ring_multi(P, kernel, slots, groups, f):
    """Two ranks, overlap = 1: persistent_multi = 1 makes the own-part and per-peer halo-block launches (and the
    pipelined backward's row ranges) persistent; the forward has the ReLU epilogue."""
    many(P.p2, kernel=kernel, ring_slots=slots, ring_groups=groups, overlap=1, relu=1)
    try:
        for tf in row_tiles(kernel, f):
            set_opts(P.p2, ring_tile_floats=tf)
            for r in range(2):
                for part in ("own", "halo", "tr_own", "tr_halo"):
                    many_items("rank %d %s tf=%d" % (r, part, tf), sched_blocks(P.counts2[r][part]), f, tf)
            res = {}
            for pm in (1, 0):
                set_opts(P.p2, persistent_multi=pm)
                res[pm] = fused(P, f, 2, P.X, P.Y)
            for r in range(2):
                for i in range(2):
                    w = "rank %d call %d tf=%d" % (r, i, tf)
                    check_close(res[1][0][i][r], *P.ref("AX", f, P.own[r], relu=True), what=w + ", relu forward")
                    check_close(res[1][1][i][r], *P.ref("ATY", f, P.own[r]), what=w + ", backward")
                    for j, name in ((0, "Z"), (1, "G")):
                        assert_bits(res[1][j][0][r], res[1][j][i][r], w + ", %s, both slab parities" % name)
                        assert_bits(res[1][j][i][r], res[0][j][i][r], w + ", %s, persistent_multi 1 vs 0" % name)
    finally:
        set_opts(P.p2, relu=0, persistent_multi=0)


def few_items(p):
    """Switch p's edge rings to the few-item schedule (asserted: fewer blocks than SMs, once a call has built it)."""
    p.set_option("ring_edges_per_block", FEW)
    p.set_option("ring_long_row", 0)


def assert_few(p):
    sms = torch.cuda.get_device_properties(dev()).multi_processor_count
    assert p.get_option("ring_blocks_fwd") < sms, "the few-item schedule has %d blocks" % p.get_option("ring_blocks_fwd")


def edge_call(fn, p, K, g, H, Hh, f):
    out = torch.full((p.lp.nnz(), K), NAN, device=dev())
    cabi.check(fn(p, g, H, Hh, out), p.handle)
    return out


def run_edges(P, p, K, f, g, H, Hh, grows, gcols, call, what):
    """Many-item calls (twice), then the few-item one: same bits, and the first within the fp64 bound."""
    outs = []
    for few in (False, False, True):
        if few:
            few_items(p)
        outs.append(edge_call(call, p, K, g, H, Hh, f))
        if not few:
            many_items(what, p.get_option("ring_blocks_fwd"), f, f)
    assert_few(p)
    many([p])
    want, tol = edge_ref(grows, gcols, P.Y[:, :f], P.X[:, :f], K)
    check_close(outs[0].view(-1, K), want, tol, what)
    assert_bits(outs[0], outs[1], what + ", run to run")
    assert_bits(outs[0], outs[2], what + ", many items vs a few")


def run_sddmm(P, ranks, f):
    lib = cabi.load()

    def call(p, g, H, Hh, out):
        return lib.pgcn_sddmm(p.handle, g.data_ptr(), H.data_ptr(), None if Hh is None else Hh.data_ptr(),
                              out.data_ptr(), f, stream())
    if ranks == 1:
        p = P.p1
        many([p])
        run_edges(P, p, 1, f, P.Y[:, :f].contiguous(), P.X[:, :f].contiguous(), None, P.rows, P.cols, call,
                  "sddmm f=%d" % f)
        return
    # the kept halo rows of a fused forward are the SDDMM's halo operand
    many(P.p2)
    Hs = [P.X[o, :f].contiguous() for o in P.own]
    Hh = [torch.full((l.h, f), NAN, device=dev()) for l in P.lps]
    Z = [torch.full_like(h, NAN) for h in Hs]
    run_ranks(P.p2, lambda r: cabi.check(lib.pgcn_forward_keep_halo(P.p2[r].handle, Hs[r].data_ptr(), Z[r].data_ptr(),
                                                                    Hh[r].data_ptr(), f, stream()), P.p2[r].handle),
              P.streams)
    for r, l in enumerate(P.lps):
        assert_bits(Hh[r], P.X[torch.from_numpy(l.halo).to(dev()), :f], "rank %d kept halo rows" % r)
    run_edges(P, P.p2[0], 1, f, P.Y[P.own[0], :f].contiguous(), Hs[0], Hh[0], P.grows[0], P.gcols[0], call,
              "rank 0 sddmm f=%d" % f)


def run_sddmm_heads(P, f, K):
    lib = cabi.load()

    def call(p, g, H, Hh, out):
        return lib.pgcn_sddmm_heads(p.handle, K, g.data_ptr(), H.data_ptr(), None, out.data_ptr(), f, stream())
    many([P.p1])
    run_edges(P, P.p1, K, f, P.Y[:, :f].contiguous(), P.X[:, :f].contiguous(), None, P.rows, P.cols, call,
              "sddmm_heads f=%d K=%d" % (f, K))


def run_gatv2(P, ranks, f, K):
    """Forward scores + softmax + aggregation: the ring scores at many items (twice; on two ranks each call reads the
    other slab half), the plain scores (xr 4 bytes into its buffer) and the ring at a few items give the same bits."""
    xl, xr, att, _ = (torch.from_numpy(x).to(dev()) for x in gatv2_inputs(f, K, N, f * 10 + K))
    plans = [P.p1] if ranks == 1 else P.p2

    def ready():
        # the schedules of new options are built up front: a set-up that frees device memory inside a fused call
        # would wait for this process's other rank, whose rows are enqueued after it
        if ranks == 2:
            for p in plans:
                p.prepare(f)
    many(plans)
    ready()
    res = {}
    for mode in ("ring", "plain", "few"):
        if mode == "few":
            for p in plans:
                few_items(p)
            ready()
        outs = []
        for _ in range(2):
            if ranks == 1:
                xrd = shifted(xr) if mode == "plain" else xr
                outs.append([gatv2_fwd(P.p1, K, xl, xrd, att, None, False)])
            else:
                ins = [(xl[o].contiguous(), xr[o].contiguous()) for o in P.own]
                if mode == "plain":
                    ins = [(a, shifted(b)) for a, b in ins]
                outs.append(run_ranks(P.p2, lambda r: gatv2_fwd(P.p2[r], K, ins[r][0], ins[r][1], att, None, False),
                                      P.streams))
        res[mode] = outs
        if mode == "ring":
            for r, p in enumerate(plans):
                many_items("rank %d gatv2 scores f=%d K=%d" % (r, f, K), p.get_option("ring_blocks_fwd"), f, f)
    for p in plans:
        assert_few(p)
    many(plans)
    ready()
    for r, p in enumerate(plans):
        what = "rank %d of %d: gatv2 f=%d K=%d" % (r, ranks, f, K)
        grows, gcols = (P.rows, P.cols) if ranks == 1 else (P.grows[r], P.gcols[r])
        lrows = P.rows if ranks == 1 else torch.from_numpy(edges(p.lp)[0]).to(dev())
        want, tol = alpha_ref(lrows, grows, gcols, p.lp.m, xl, xr, att)
        check_close(res["ring"][0][r][0], want, tol, what + ", alpha")
        for i in range(2):
            for mode in ("ring", "plain", "few"):
                for j, name in ((0, "alpha"), (1, "Z")):
                    assert_bits(res["ring"][0][r][j], res[mode][i][r][j], "%s, %s: ring call 1 vs %s call %d" % (
                        what, name, mode, i + 1))


def settle():
    x = torch.zeros(1024, device=dev())
    for _ in range(16):
        x.add_(1)
    torch.cuda.synchronize()
    time.sleep(0.05)


RUNNERS = {"ring": run_ring, "ring_halo": run_ring_halo, "ring_multi": run_ring_multi, "sddmm": run_sddmm,
           "sddmm_heads": run_sddmm_heads, "gatv2": run_gatv2}
SEEN = set()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES, ids=[r.id for r in ROUTES])
def test_route(prob, route):
    # torch.profiler now and then loses a session's first kernel records (as in the census; more often after a long
    # run of profiled sessions in one process): a few throw-away kernels open each session, and the row, whose checks
    # pass each time, is run again; a dispatch that picks another instance misses it every time
    names = set()
    for _ in range(6):
        try:
            _, got = launched(lambda: (settle(), RUNNERS[route.family](prob, **route.kw)))
        finally:
            many([prob.p1] + prob.p2)
        names |= got
        if route.expect <= names:
            break
    assert names, "torch.profiler recorded no CUDA kernel"
    missing = route.expect - names
    assert not missing, "%s no longer launches %s (it launched %s)" % (route.id, sorted(missing), sorted(names))
    SEEN.update(names)


# ---- mixed hot and cold columns --------------------------------------------------------------------------------------

def family_rows(P, p):
    """One many-item call per ring family on plan p (one rank): SpMM at full-width and 64-float tiles, forward and
    transposed, the SDDMM, the multi-head SDDMM and the GATv2 scores."""
    lib = cabi.load()
    f = 256
    many([p])
    H, G = P.X[:, :f].contiguous(), P.Y[:, :f].contiguous()
    outs = {}
    for tf in (64, 256):
        p.set_option("ring_tile_floats", tf)
        outs["spmm tf=%d" % tf] = (spmm(p, 0, H, None, f), spmm(p, 1, G, None, f))
        many_items("hot/cold A H tf=%d" % tf, p.get_option("ring_blocks_fwd"), f, tf)
    p.set_option("ring_tile_floats", 0)
    out = torch.full((p.lp.nnz(), 1), NAN, device=dev())
    cabi.check(lib.pgcn_sddmm(p.handle, G.data_ptr(), H.data_ptr(), None, out.data_ptr(), f, stream()), p.handle)
    out4 = torch.full((p.lp.nnz(), 4), NAN, device=dev())
    cabi.check(lib.pgcn_sddmm_heads(p.handle, 4, G.data_ptr(), H.data_ptr(), None, out4.data_ptr(), f, stream()),
               p.handle)
    outs["sddmm"] = (out, out4)
    xl, xr, att, _ = (torch.from_numpy(x).to(dev()) for x in gatv2_inputs(128, 2, N, 5))
    outs["gatv2"] = gatv2_fwd(p, 2, xl, xr, att, None, False)
    many_items("hot/cold edge rings f=256", p.get_option("ring_blocks_fwd"), f, f)
    torch.cuda.synchronize()
    return outs


@pytest.mark.gpu
def test_mixed_hot_and_cold_columns_give_the_same_bits(prob, monkeypatch):
    hot = family_rows(prob, prob.p1)
    monkeypatch.setenv("PGCN_HOT_MB", "1")
    mixed = planmod.PgcnPlan(prob.p1.lp, F_MAX, device=dev())
    try:
        assert mixed.get_option("hot_mb") == 1
        mixed.bind_values()
        got = family_rows(prob, mixed)
    finally:
        mixed.close()
    for name in hot:
        for i, (a, b) in enumerate(zip(hot[name], got[name])):
            assert_bits(a, b, "%s output %d, hot and cold columns vs the default hot set" % (name, i))


# ---- capture and replay ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_one_rank_capture_replays_many_items(prob):
    lib = cabi.load()
    p, f = prob.p1, 256
    many([p])
    rs = np.random.RandomState(8)
    ins = [tuple(torch.from_numpy(rs.uniform(-1, 1, (N, f)).astype(np.float32)).to(dev()) for _ in range(2))
           for _ in range(3)]
    x, g = torch.zeros((N, f), device=dev()), torch.zeros((N, f), device=dev())

    def step(x, g):
        z, b = torch.empty_like(x), torch.empty_like(g)
        cabi.check(lib.pgcn_forward(p.handle, x.data_ptr(), z.data_ptr(), f, stream()), p.handle)
        cabi.check(lib.pgcn_backward(p.handle, g.data_ptr(), b.data_ptr(), f, stream()), p.handle)
        return dict(z=z, b=b)

    def load(i):
        x.copy_(ins[i][0])
        g.copy_(ins[i][1])

    p.prepare(f)
    many_items("capture A H", p.get_option("ring_blocks_fwd"), f, 256)
    many_items("capture A^T g", sched_blocks(prob.counts1["tr"]), f, 256)
    check_one_rank_capture(p, lambda: step(x, g), load, lambda i: step(*ins[i]))


@pytest.mark.gpu
def test_two_rank_capture_replays_persistent_multi(prob):
    lib = cabi.load()
    plans, f = prob.p2, 256
    many(plans, overlap=1, persistent_multi=1)
    try:
        for r in range(2):
            for part in ("own", "halo", "tr_own", "tr_halo"):
                many_items("capture rank %d %s" % (r, part), sched_blocks(prob.counts2[r][part]), f, 256)
        for p in plans:
            p.prepare(f)
        rs = np.random.RandomState(9)
        ins = [tuple(rs.uniform(-1, 1, (N, f)).astype(np.float32) for _ in range(2)) for _ in range(3)]

        def buffers(r):
            m = prob.lps[r].m
            return dict(x=torch.zeros((m, f), device=dev()), g=torch.zeros((m, f), device=dev()))

        def load(bufs, i):
            for r, l in enumerate(prob.lps):
                bufs[r]["x"].copy_(torch.from_numpy(ins[i][0][l.owned]))
                bufs[r]["g"].copy_(torch.from_numpy(ins[i][1][l.owned]))
            torch.cuda.synchronize()

        def step(r, b):
            z, gr = torch.empty_like(b["x"]), torch.empty_like(b["g"])
            cabi.check(lib.pgcn_forward(plans[r].handle, b["x"].data_ptr(), z.data_ptr(), f, stream()), plans[r].handle)
            cabi.check(lib.pgcn_backward(plans[r].handle, b["g"].data_ptr(), gr.data_ptr(), f, stream()),
                       plans[r].handle)
            return dict(z=z, gr=gr)

        check_two_rank_capture(plans, prob.streams, buffers, load, step)
    finally:
        set_opts(plans, persistent_multi=0)


# ---- grid-capped copies ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_grid_capped_copies_over_many_strides(prob):
    """put_rows_kernel (4 CTAs per SM), pack_rows_kernel, copy_halo_kernel and set_values_kernel (32 per SM) at work of
    at least 4 grid strides, checked exactly (set_values through the ring SpMM over the rewritten records)."""
    lib = cabi.load()
    sms = torch.cuda.get_device_properties(dev()).multi_processor_count
    f = 512
    many([prob.p1] + prob.p2)
    for r, (p, l) in enumerate(zip(prob.p2, prob.lps)):
        assert l.S * f // 4 >= 4 * 4 * sms * 256, "put_rows: %d vectors" % (l.S * f // 4)
        assert l.S * f // 4 >= 4 * 32 * sms * 256, "pack_rows: %d vectors" % (l.S * f // 4)
        assert l.h * f >= 4 * 32 * sms * 256, "copy_halo: %d floats" % (l.h * f)
        H = prob.X[prob.own[r], :f].contiguous()
        slab = torch.full((l.S, f), NAN, device=dev())
        cabi.check(lib.pgcn_pack(p.handle, H.data_ptr(), slab.data_ptr(), f, stream()), p.handle)
        assert_bits(slab, H[torch.from_numpy(l.send_idx.astype(np.int64)).to(dev())], "rank %d pack" % r)
    Hs = [prob.X[o, :f].contiguous() for o in prob.own]
    for call in ("halo_rows", "keep_halo", "halo_rows"):             # the exchange epoch alternates its parity
        Hh = [torch.full((l.h, f), NAN, device=dev()) for l in prob.lps]
        if call == "halo_rows":
            run_ranks(prob.p2, lambda r: cabi.check(lib.pgcn_halo_rows(prob.p2[r].handle, Hs[r].data_ptr(),
                                                                       Hh[r].data_ptr(), f, stream()),
                                                    prob.p2[r].handle), prob.streams)
        else:
            Z = [torch.full_like(h, NAN) for h in Hs]
            run_ranks(prob.p2, lambda r: cabi.check(lib.pgcn_forward_keep_halo(
                prob.p2[r].handle, Hs[r].data_ptr(), Z[r].data_ptr(), Hh[r].data_ptr(), f, stream()),
                prob.p2[r].handle), prob.streams)
        for r, l in enumerate(prob.lps):
            assert_bits(Hh[r], prob.X[torch.from_numpy(l.halo).to(dev()), :f], "rank %d %s rows" % (r, call))
    # set_values: one rank's forward and transposed record sets (2 nnz entries)
    p, lp = prob.p1, prob.p1.lp
    assert 2 * lp.nnz() >= 4 * 32 * sms * 256, "set_values: %d entries" % (2 * lp.nnz())
    vals = torch.from_numpy(np.random.RandomState(9).uniform(-1, 1, lp.nnz()).astype(np.float32)).to(dev())
    fv = 256
    try:
        p.set_values(vals)
        Z = spmm(p, 0, prob.X[:, :fv].contiguous(), None, fv)
        G = spmm(p, 1, prob.Y[:, :fv].contiguous(), None, fv)
    finally:
        p.set_values(None)
    v64 = vals.double()
    check_close(Z, *spmm_ref(prob.rows, prob.cols, v64, prob.X[:, :fv], N), what="A(vals) H")
    check_close(G, *spmm_ref(prob.cols, prob.rows, v64, prob.Y[:, :fv], N), what="A(vals)^T g")
    assert_bits(spmm(p, 0, prob.X[:, :fv].contiguous(), None, fv), spmm(p, 0, prob.X[:, :fv].contiguous(), None, fv),
                "creation values restored, run to run")
    check_close(spmm(p, 0, prob.X[:, :fv].contiguous(), None, fv), *prob.ref("AX", fv), what="creation values restored")


# ---- completeness ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_every_ring_instance_ran_at_many_items():
    """Runs last in this file: every ring instance of the library was launched by a row whose precondition held."""
    want = ring_manifest()
    if not SEEN:
        pytest.fail("no route ran before this test (run the whole file)")
    missing = want - SEEN
    assert not missing, "%d ring instances never launched at many items: %s" % (len(missing), sorted(missing))
    print("\n%d/%d ring instances launched at many items per warp; fewest items per resident warp %.2f over %d "
          "launches" % (len(want & SEEN), len(want), min(RATIOS), len(RATIOS)))
