"""Operands at the edges the rest of the suite does not reach: rows that are not 16-byte aligned, IEEE special values,
and feature matrices larger than 4 GiB.

  * Unaligned operands. Every pointer argument of the aggregation path (pgcn_spmm in all four transposes, pgcn_pack,
    pgcn_unpack_add, the fused forward / backward on 1, 2 and 3 ranks over the peer transport, forward_keep_halo,
    halo_rows, the SDDMM, the edge softmax, set_values) and the autograd ops are fed contiguous views that start 4, 8
    or 12 bytes into their buffer (shift 0 is the control). Such a call takes the register kernel with scalar accesses,
    whose schedule and per-element summation order do not depend on the vector width: SpMM results are bit-identical to
    the same call on aligned copies with option kernel=4, copies are exact. Each view is guarded by sentinel floats on
    both sides that must be bit-unchanged after the call, and every output starts as NaN, so a row that is never
    written cannot hide behind stale memory.
  * IEEE special values. +-Inf and NaN in features, scores and edge values must land exactly where the fp64 product
    puts them (hub rows split into segments, ordinary rows, halo rows, rows nothing references); the fused ReLU keeps
    NaN like torch.relu; subnormal products are neither flushed nor approximated.
  * Operands over 4 GiB: rows past byte offset 2^32 of H and Z, forward on the ring and register kernels, backward and
    the SDDMM, checked on a sample of rows and edges against fp64.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from harness import EPS, bits, dev, hub_graph, stream
from helpers import assert_close_fp32, fp32_tol
from oracle import pgcn_oracle as orc
from pgcn_b200 import cabi, graphio, op, plan as planmod
from pgcn_b200.op import PGATAttention, PSpMM, PSpMMRelu, PSpMMWeighted
from test_gpu_parity import skewed_graph

pytestmark = pytest.mark.gpu
SENTINEL = 0x7FBADBAD                    # a NaN payload no kernel produces: any write to a guard float changes it
N, NNZ, F_MAX = 3000, 60000, 640


def ptr(x):
    return None if x is None else x.data_ptr()


def call(name, plan, *args):
    cabi.check(getattr(cabi.load(), name)(plan.handle, *args), plan.handle)


# ---- guarded, deliberately misaligned operands ---------------------------------------------------------------------

_GUARDED = []


@pytest.fixture(autouse=True)
def _guards():
    _GUARDED.clear()
    yield
    check_guards()


def offset_view(shape, shift_floats, fill=None):
    """A contiguous fp32 view whose first float lies `shift_floats` floats past a 16-byte boundary, with at least 4
    sentinel floats on each side. Filled with `fill` (array or tensor), else with NaN."""
    shape = tuple(int(s) for s in shape)
    numel = int(np.prod(shape))
    buf = torch.empty(numel + 8 + shift_floats, dtype=torch.float32, device=dev())
    buf.view(torch.int32).fill_(SENTINEL)
    v = buf[4 + shift_floats:4 + shift_floats + numel].view(shape)
    assert v.is_contiguous() and (numel == 0 or v.data_ptr() % 16 == 4 * shift_floats)
    if fill is None:
        v.fill_(float("nan"))
    else:
        v.copy_(torch.as_tensor(np.ascontiguousarray(fill)) if isinstance(fill, np.ndarray) else fill)
    _GUARDED.append((buf, 4 + shift_floats, 4 + shift_floats + numel))
    return v


def check_guards():
    torch.cuda.synchronize()
    for buf, lo, hi in _GUARDED:
        b = buf.view(torch.int32)
        assert bool((b[:lo] == SENTINEL).all()) and bool((b[hi:] == SENTINEL).all()), "write outside the operand"


def assert_bits(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape and np.array_equal(g, w), "%s: %d elements differ in their bits" % (what, int((g != w).sum()))


def random_plans(A, k, f_max=F_MAX, link=True, seed=5):
    pv = graphio.random_partvec(A.shape[0], k, seed=seed)
    plans = [planmod.build_plan(A, pv, r, k, f_max, device=dev()) for r in range(k)]
    if k > 1 and link:
        planmod.link_local_plans(plans)
    return plans


def set_opts(plans, **opts):
    for p in plans:
        for name, v in opts.items():
            p.set_option(name, v)


def run_ranks(calls):
    """One call per rank, each on its own stream (the peer transport's waits are on the device), then synchronise."""
    streams = [torch.cuda.Stream(device=dev()) for _ in calls]
    torch.cuda.synchronize()
    for c, s in zip(calls, streams):
        with torch.cuda.stream(s):
            c()
    torch.cuda.synchronize()


def local_csr(lp, vals=None):
    """The rank's A_local over [own | halo] columns in fp64, entries as stored (duplicates and explicit zeros kept)."""
    v = lp.vals if vals is None else vals
    return sp.csr_matrix((np.asarray(v, np.float64), lp.colidx, lp.rowptr), shape=(lp.m, lp.m + lp.h))


def dmax(A):
    return int(np.diff(sp.csr_matrix(A).indptr).max())


# ---- A. unaligned operands -----------------------------------------------------------------------------------------

# operands of each transpose of pgcn_spmm
SPMM_OPERANDS = {0: ("H_own", "H_halo", "Z"), 1: ("H_own", "Z", "Z_halo"), 2: ("H_own", "Z"), 3: ("H_halo", "Z")}


def spmm_call(p, tr, f, Hown, Hhalo, Zin, shifts):
    lp = p.lp
    s = lambda name: shifts.get(name, 0)
    ho = offset_view((lp.m, f), s("H_own"), Hown) if tr != 3 else None
    hh = offset_view((lp.h, f), s("H_halo"), Hhalo) if tr in (0, 3) else None
    z = offset_view((lp.m, f), s("Z"), Zin)
    zh = offset_view((lp.h, f), s("Z_halo")) if tr == 1 else None
    call("pgcn_spmm", p, tr, ptr(ho), ptr(hh), z.data_ptr(), ptr(zh), f, stream())
    check_guards()
    return z.clone(), (zh.clone() if zh is not None else None)


@pytest.mark.parametrize("f", [3, 4, 12, 128, 256, 384, 640])
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_spmm_pack_unpack_unaligned(f, shift):
    """pgcn_spmm (transposes 0-3), pgcn_pack and pgcn_unpack_add with each operand misaligned on its own and all at
    once: bit-identical to aligned copies on the register kernel (shift 0: to the same aligned call), within the fp32
    bound of fp64, exact copies for the pack. Hub rows are split (edges_per_block 16), so the fixup writes into the
    unaligned Z; empty rows are zero-filled there."""
    A = skewed_graph(N, NNZ, seed=7)
    plans = random_plans(A, 2, link=False)
    rs = np.random.RandomState(f)
    H = rs.uniform(-1, 1, size=(N, f)).astype(np.float32)
    G = rs.uniform(-1, 1, size=(N, f)).astype(np.float32)
    set_opts(plans, edges_per_block=16, ring_edges_per_block=64)
    for r, p in enumerate(plans):
        lp = p.lp
        Hown, Hhalo, Gown = H[lp.owned], H[lp.halo], G[lp.owned]
        csr = local_csr(lp)
        d = dmax(csr)
        Hcat = np.concatenate([Hown, Hhalo], 0)
        Z64, tolZ = csr @ Hcat.astype(np.float64), fp32_tol(csr, Hcat, d)
        own = csr[:, :lp.m]
        Zo64, tolZo = own @ Hown.astype(np.float64), fp32_tol(own, Hown, d)
        Gt64, tolG = csr.T @ Gown.astype(np.float64), fp32_tol(csr.T, Gown, dmax(csr.T))
        p.set_option("kernel", 4 if shift else 0)
        ref = {0: spmm_call(p, 0, f, Hown, Hhalo, None, {}), 1: spmm_call(p, 1, f, Gown, None, None, {}),
               2: spmm_call(p, 2, f, Hown, None, None, {})}
        ref[3] = spmm_call(p, 3, f, None, Hhalo, ref[2][0], {})
        p.set_option("kernel", 0)
        assert p.get_option("long_rows_fwd") + p.get_option("ring_long_rows_fwd") > 0
        for tr, names in SPMM_OPERANDS.items():
            for which in names + ("all",):
                sh = {nm: shift for nm in names if which in (nm, "all")}
                z, zh = spmm_call(p, tr, f, Gown if tr == 1 else Hown, Hhalo, ref[2][0] if tr == 3 else None, sh)
                what = "f=%d shift=%d r%d transpose %d %s" % (f, shift, r, tr, which)
                assert_bits(z, ref[tr][0], what)
                if tr == 1:
                    assert_bits(zh, ref[1][1], what + " Z_halo")
                    assert_close_fp32(z.cpu().numpy(), Gt64[:lp.m], tolG[:lp.m], what)
                    assert_close_fp32(zh.cpu().numpy(), Gt64[lp.m:], tolG[lp.m:], what + " Z_halo")
                elif tr == 2:
                    assert_close_fp32(z.cpu().numpy(), Zo64, tolZo, what)
                else:
                    assert_close_fp32(z.cpu().numpy(), Z64, tolZ, what)
        # pack: an exact gather of the send rows
        want = torch.from_numpy(Hown[lp.send_idx]).to(dev())
        for which in ("H", "slab", "all"):
            h = offset_view((lp.m, f), shift if which in ("H", "all") else 0, Hown)
            slab = offset_view((lp.S, f), shift if which in ("slab", "all") else 0)
            call("pgcn_pack", p, h.data_ptr(), slab.data_ptr(), f, stream())
            assert_bits(slab, want, "pack f=%d shift=%d %s" % (f, shift, which))
        # unpack_add: in-place fixed-order sum, bit-identical to the aligned call
        recv = rs.uniform(-1, 1, size=(lp.S, f)).astype(np.float32)
        g0 = offset_view((lp.m, f), 0, Gown)
        call("pgcn_unpack_add", p, offset_view((lp.S, f), 0, recv).data_ptr(), g0.data_ptr(), f, stream())
        want64, mag = Gown.astype(np.float64), np.abs(Gown.astype(np.float64))
        np.add.at(want64, lp.send_idx, recv.astype(np.float64))
        np.add.at(mag, lp.send_idx, np.abs(recv.astype(np.float64)))
        cnt = np.bincount(lp.send_idx, minlength=lp.m)[:, None]
        assert_close_fp32(g0.cpu().numpy(), want64, 2.0 * (cnt + 2) * EPS * mag + 1e-30, "unpack aligned")
        for which in ("recv", "G", "all"):
            rv = offset_view((lp.S, f), shift if which in ("recv", "all") else 0, recv)
            g = offset_view((lp.m, f), shift if which in ("G", "all") else 0, Gown)
            call("pgcn_unpack_add", p, rv.data_ptr(), g.data_ptr(), f, stream())
            assert_bits(g, g0, "unpack f=%d shift=%d %s" % (f, shift, which))
    for p in plans:
        p.close()


def rank_shifts(k, s):
    """s = 0: every rank aligned (the control); else a different non-zero shift on each rank (k <= 3)."""
    return [0] * k if s == 0 else [1 + (s - 1 + r) % 3 for r in range(k)]


@pytest.mark.parametrize("k,f", [(1, 3), (1, 12), (1, 128), (2, 4), (2, 128), (3, 12), (3, 384), (3, 640)])
@pytest.mark.parametrize("s", [0, 1, 2, 3])
def test_fused_forward_backward_unaligned(k, f, s):
    """pgcn_forward / pgcn_backward on 1 rank and on 2 and 3 ranks of this process over the peer transport, overlap 0
    and 1, relu 0 and 1, split rows, a different shift on every rank (the transport must not depend on alignment: all
    ranks have to agree), the input, the output or both misaligned: bit-identical to aligned copies on the register
    kernel, within the fp32 bound of fp64."""
    A = skewed_graph(N, NNZ, seed=9)
    plans = random_plans(A, k)
    rs = np.random.RandomState(10 * k + f)
    H = rs.uniform(-1, 1, size=(N, f)).astype(np.float32)
    G = rs.uniform(-1, 1, size=(N, f)).astype(np.float32)
    pre64 = orc.truth_forward(A, H)
    tolZ = fp32_tol(A, H, dmax(A))
    G64, tolG = orc.truth_backward(A, G), fp32_tol(A.T, G, dmax(A.T))
    shifts = rank_shifts(k, s)
    set_opts(plans, edges_per_block=16, ring_edges_per_block=64)
    if k > 1:
        for p in plans:
            assert p.get_option("p2p") == 1

    def fused(name, X, sh_in, sh_out):
        ins = [offset_view((p.lp.m, f), sh_in[r], X[p.lp.owned]) for r, p in enumerate(plans)]
        outs = [offset_view((p.lp.m, f), sh_out[r]) for r, p in enumerate(plans)]
        run_ranks([lambda p=p, x=x, y=y: call(name, p, x.data_ptr(), y.data_ptr(), f, stream())
                   for p, x, y in zip(plans, ins, outs)])
        check_guards()
        return [y.clone() for y in outs]

    zero = [0] * k
    for overlap in ((0, 1) if k > 1 else (1,)):
        for relu in (0, 1):
            set_opts(plans, overlap=overlap, relu=relu, kernel=4 if s else 0)
            zref, gref = fused("pgcn_forward", H, zero, zero), fused("pgcn_backward", G, zero, zero)
            set_opts(plans, kernel=0)
            for which in ("in", "out", "both"):
                sh_in = shifts if which in ("in", "both") else zero
                sh_out = shifts if which in ("out", "both") else zero
                z, g = fused("pgcn_forward", H, sh_in, sh_out), fused("pgcn_backward", G, sh_in, sh_out)
                # an aligned Z with an unaligned H_own: the launches of the peer blocks read the plan's aligned slab
                # and write the aligned Z, so they keep the ring kernel where f allows it
                mixed = s and which == "in" and overlap and k > 1 and f % 128 == 0
                for r, p in enumerate(plans):
                    own = p.lp.owned
                    what = "k=%d f=%d shifts=%s overlap=%d relu=%d %s r%d" % (k, f, shifts, overlap, relu, which, r)
                    if mixed:
                        torch.testing.assert_close(z[r], zref[r], rtol=1e-4, atol=1e-5)
                    else:
                        assert_bits(z[r], zref[r], what + " fwd")
                    assert_bits(g[r], gref[r], what + " bwd")
                    want = np.maximum(pre64[own], 0.0) if relu else pre64[own]
                    assert_close_fp32(z[r].cpu().numpy(), want, tolZ[own], what + " fwd")
                    assert_close_fp32(g[r].cpu().numpy(), G64[own], tolG[own], what + " bwd")
    for p in plans:
        p.close()


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("w", [4, 128])
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_keep_halo_and_halo_rows_unaligned(k, w, shift):
    """pgcn_halo_rows with unaligned X_own / X_halo_out and pgcn_forward_keep_halo with an unaligned H_halo_out (alone,
    and with H_own and Z): the halo rows are exact copies of their owners' rows, Z is bit-identical to the aligned
    call (register kernel when H_own / Z are misaligned)."""
    A = skewed_graph(N, NNZ, seed=13)
    plans = random_plans(A, k)
    for p in plans:
        p.bind_values()
    X = np.random.RandomState(w + k).uniform(-1, 1, size=(N, w)).astype(np.float32)
    halo_want = [torch.from_numpy(X[p.lp.halo]).to(dev()) for p in plans]
    for which in ("X_own", "X_halo_out", "all"):
        xs = [offset_view((p.lp.m, w), shift if which in ("X_own", "all") else 0, X[p.lp.owned]) for p in plans]
        hs = [offset_view((p.lp.h, w), shift if which in ("X_halo_out", "all") else 0) for p in plans]
        run_ranks([lambda p=p, x=x, h=h: call("pgcn_halo_rows", p, x.data_ptr(), h.data_ptr(), w, stream())
                   for p, x, h in zip(plans, xs, hs)])
        for r in range(k):
            assert_bits(hs[r], halo_want[r], "halo_rows w=%d shift=%d %s r%d" % (w, shift, which, r))

    def keep(sh_main, sh_halo):
        xs = [offset_view((p.lp.m, w), sh_main, X[p.lp.owned]) for p in plans]
        zs = [offset_view((p.lp.m, w), sh_main) for p in plans]
        hs = [offset_view((p.lp.h, w), sh_halo) for p in plans]
        run_ranks([lambda p=p, x=x, z=z, h=h: call("pgcn_forward_keep_halo", p, x.data_ptr(), z.data_ptr(), h.data_ptr(),
                                                    w, stream()) for p, x, z, h in zip(plans, xs, zs, hs)])
        check_guards()
        return zs, hs

    zref0, _ = keep(0, 0)
    set_opts(plans, kernel=4)
    zref4, _ = keep(0, 0)
    set_opts(plans, kernel=0)
    Z64, tol = orc.truth_forward(A, X), fp32_tol(A, X, dmax(A))
    for which in ("H_halo_out", "all"):
        zs, hs = keep(shift if which == "all" else 0, shift)
        zref = zref4 if (which == "all" and shift) else zref0
        for r, p in enumerate(plans):
            what = "keep_halo w=%d shift=%d %s r%d" % (w, shift, which, r)
            assert_bits(hs[r], halo_want[r], what + " halo")
            assert_bits(zs[r], zref[r], what)
            assert_close_fp32(zs[r].cpu().numpy(), Z64[p.lp.owned], tol[p.lp.owned], what)
    for p in plans:
        p.close()


def edge_rows(lp):
    return np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))


def sddmm64(lp, gZ, Hcat):
    rows, cols = edge_rows(lp), lp.colidx.astype(np.int64)
    g, h = gZ.astype(np.float64)[rows], Hcat.astype(np.float64)[cols]
    with np.errstate(invalid="ignore", over="ignore"):
        return (g * h).sum(1), (np.abs(g) * np.abs(h)).sum(1)


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("f", [12, 128, 256])
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_sddmm_softmax_set_values_unaligned(k, f, shift):
    """pgcn_sddmm (unaligned operands take the plain kernel: within the fp32 dot bound of fp64 and run-to-run
    identical), pgcn_edge_softmax(_backward) (bit-identical to the aligned call, every argument misaligned on its own
    and all at once), pgcn_plan_set_values from an unaligned array (the aggregation that follows is bit-identical)."""
    A = skewed_graph(N, NNZ, seed=15)
    plans = random_plans(A, k, link=False)
    rs = np.random.RandomState(f + shift)
    H = rs.uniform(-1, 1, size=(N, f)).astype(np.float32)
    for p in plans:
        p.bind_values()
        lp = p.lp
        gZ = rs.uniform(-1, 1, size=(lp.m, f)).astype(np.float32)
        Hown, Hhalo = H[lp.owned], H[lp.halo]
        d64, mag = sddmm64(lp, gZ, np.concatenate([Hown, Hhalo], 0))
        tol = 2.0 * (f + 2) * EPS * mag + 1e-30
        for which in ("gZ", "H_own", "H_halo", "dvals", "all"):
            s = lambda nm: shift if which in (nm, "all") else 0
            runs = []
            for _ in range(2):
                dv = offset_view((lp.nnz(),), s("dvals"))
                call("pgcn_sddmm", p, offset_view((lp.m, f), s("gZ"), gZ).data_ptr(),
                     offset_view((lp.m, f), s("H_own"), Hown).data_ptr(),
                     offset_view((lp.h, f), s("H_halo"), Hhalo).data_ptr() if lp.h else None, dv.data_ptr(), f, stream())
                runs.append(dv.clone())
            assert_bits(runs[0], runs[1], "sddmm run to run")
            err = np.abs(runs[0].cpu().numpy().astype(np.float64) - d64)
            assert (err <= tol).all(), "sddmm f=%d shift=%d %s: %d edges beyond the bound" % (f, shift, which,
                                                                                              int((err > tol).sum()))
        # edge softmax and its backward
        el = rs.uniform(-2, 2, lp.m).astype(np.float32)
        er = rs.uniform(-2, 2, N).astype(np.float32)
        dal = rs.uniform(-1, 1, lp.nnz()).astype(np.float32)
        names = ("el", "er_own", "er_halo", "alpha", "dalpha", "dpre", "d_el")

        def softmax(which):
            s = lambda nm: shift if which in (nm, "all") else 0
            a_el, a_own = offset_view((lp.m,), s("el"), el), offset_view((lp.m,), s("er_own"), er[lp.owned])
            a_halo = offset_view((lp.h,), s("er_halo"), er[lp.halo])
            alpha = offset_view((lp.nnz(),), s("alpha"))
            call("pgcn_edge_softmax", p, a_el.data_ptr(), a_own.data_ptr(), a_halo.data_ptr(), 0.2, alpha.data_ptr(),
                 stream())
            dalpha, dpre, d_el = offset_view((lp.nnz(),), s("dalpha"), dal), offset_view((lp.nnz(),), s("dpre")), \
                offset_view((lp.m,), s("d_el"))
            call("pgcn_edge_softmax_backward", p, a_el.data_ptr(), a_own.data_ptr(), a_halo.data_ptr(), alpha.data_ptr(),
                 dalpha.data_ptr(), 0.2, dpre.data_ptr(), d_el.data_ptr(), stream())
            check_guards()
            return alpha.clone(), dpre.clone(), d_el.clone()

        want = softmax("none")
        assert bool(torch.isfinite(want[0]).all())
        for which in names + ("all",):
            for a, b, nm in zip(softmax(which), want, ("alpha", "dpre", "d_el")):
                assert_bits(a, b, "softmax f=%d shift=%d %s: %s" % (f, shift, which, nm))
        # set_values from an unaligned array, then the aggregation
        vals = rs.uniform(0.1, 1, lp.nnz()).astype(np.float32)
        Hd = offset_view((lp.m, f), 0, Hown)
        Hh = offset_view((lp.h, f), 0, Hhalo) if lp.h else None
        out = []
        for sh in (0, shift):
            call("pgcn_plan_set_values", p, offset_view((lp.nnz(),), sh, vals).data_ptr(), stream())
            z = offset_view((lp.m, f), 0)
            call("pgcn_spmm", p, 0, Hd.data_ptr(), ptr(Hh), z.data_ptr(), None, f, stream())
            out.append(z.clone())
        assert_bits(out[1], out[0], "set_values f=%d shift=%d" % (f, shift))
        call("pgcn_plan_set_values", p, None, stream())
    for p in plans:
        p.close()


@pytest.mark.parametrize("f", [64, 128])
@pytest.mark.parametrize("shift", [1, 2, 3])
def test_autograd_ops_take_unaligned_views_uncopied(f, shift):
    """PSpMM, PSpMMRelu, PSpMMWeighted and PGATAttention (local layout) fed unaligned views: _check_feat passes them
    through uncopied, and outputs and gradients are bit-identical to aligned copies on the register kernel."""
    A = skewed_graph(N, NNZ, seed=19)
    p = random_plans(A, 1)[0]
    p.bind_values()
    rs = np.random.RandomState(f * shift)
    X = torch.from_numpy(rs.uniform(-1, 1, size=(N, f)).astype(np.float32)).to(dev())
    Gt = torch.from_numpy(rs.uniform(-1, 1, size=(N, f)).astype(np.float32)).to(dev())
    vals = torch.from_numpy(rs.uniform(0.1, 1, p.lp.nnz()).astype(np.float32)).to(dev())
    el = torch.from_numpy(rs.uniform(-1, 1, N).astype(np.float32)).to(dev())
    er = torch.from_numpy(rs.uniform(-1, 1, N).astype(np.float32)).to(dev())

    def inputs(tensors, unaligned):
        out = []
        for t in tensors:
            v = offset_view(t.shape, shift, t) if unaligned else t.clone()
            if unaligned and v.dim() == 2:
                assert op._check_feat(p, v, N, "H").data_ptr() == v.data_ptr()
            out.append(v.requires_grad_(True))
        return out

    cases = {
        "PSpMM": (lambda: [X], lambda x: PSpMM.apply(p, x)),
        "PSpMMRelu": (lambda: [X], lambda x: PSpMMRelu.apply(p, x)),
        "PSpMMWeighted": (lambda: [vals, X], lambda v, x: PSpMMWeighted.apply(p, v, x)),
        "PGATAttention": (lambda: [X, el, er], lambda z, a, b: PGATAttention.apply(p, z, a, b, 0.2)),
    }
    for name, (tensors, fn) in cases.items():
        res = {}
        for unaligned in (False, True):
            p.set_option("kernel", 0 if unaligned else 4)
            ins = inputs(tensors(), unaligned)
            out = fn(*ins)
            out.backward(offset_view((N, f), shift, Gt) if unaligned else Gt.clone())
            res[unaligned] = [out.detach().clone()] + [x.grad.clone() for x in ins]
        for i, (a, b) in enumerate(zip(res[True], res[False])):
            if name == "PSpMMRelu" and i == 1 and f % 128 == 0:
                # its backward aggregates grad * (out > 0), a fresh aligned tensor: the ring kernel, not bitwise
                torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
            else:
                assert_bits(a, b, "%s f=%d shift=%d" % (name, f, shift))
    p.close()


@pytest.mark.parametrize("f", [12, 128])
@pytest.mark.parametrize("shift", [1, 3])
def test_capture_with_unaligned_buffers(f, shift):
    """One rank, plan.prepare(f), then PSpMM and PSpMMRelu forward + backward captured in one CUDA graph on unaligned
    buffers: the capture is not refused, and replays on new inputs are bit-identical to eager calls on the same
    unaligned buffers."""
    A = skewed_graph(N, NNZ, seed=23)
    p = random_plans(A, 1)[0]
    p.prepare(f)
    rs = np.random.RandomState(f + shift)
    xs = [rs.uniform(-1, 1, size=(N, f)).astype(np.float32) for _ in range(3)]
    gs = [rs.uniform(-1, 1, size=(N, f)).astype(np.float32) for _ in range(3)]
    x = offset_view((N, f), shift, np.zeros((N, f), np.float32)).requires_grad_(True)
    xr = offset_view((N, f), shift, np.zeros((N, f), np.float32)).requires_grad_(True)
    g_in = offset_view((N, f), shift, np.zeros((N, f), np.float32))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z = PSpMM.apply(p, x)
        z.backward(g_in)
        zr = PSpMMRelu.apply(p, xr)
        zr.backward(g_in)
    for i in range(3):
        with torch.no_grad():
            x.copy_(torch.from_numpy(xs[i])); xr.copy_(torch.from_numpy(xs[i])); g_in.copy_(torch.from_numpy(gs[i]))
        graph.replay()
        torch.cuda.synchronize()
        for fn, zc, xc in ((PSpMM, z, x), (PSpMMRelu, zr, xr)):
            xe = offset_view((N, f), shift, xs[i]).requires_grad_(True)
            ze = fn.apply(p, xe)
            ze.backward(offset_view((N, f), shift, gs[i]))
            assert_bits(zc, ze, "%s replay %d" % (fn.__name__, i))
            assert_bits(xc.grad, xe.grad, "%s grad replay %d" % (fn.__name__, i))
    Z64 = orc.truth_forward(A, xs[-1])
    assert_close_fp32(z.detach().cpu().numpy(), Z64, fp32_tol(A, xs[-1], dmax(A)), "captured f=%d" % f)
    p.close()


# ---- B. IEEE special values ----------------------------------------------------------------------------------------

def assert_ieee(got, want, tol, what):
    """NaN, +Inf and -Inf exactly where the fp64 result has them; finite entries within `tol`."""
    got = np.asarray(got, np.float64)
    for name, mask in (("NaN", np.isnan), ("+Inf", lambda a: a == np.inf), ("-Inf", lambda a: a == -np.inf)):
        mw, mg = mask(want), mask(got)
        assert np.array_equal(mw, mg), "%s: %s at %d places, expected at %d (%d disagree)" % (
            what, name, int(mg.sum()), int(mw.sum()), int((mw != mg).sum()))
    fin = np.isfinite(want)
    assert_close_fp32(got[fin], want[fin], tol[fin], what)


def special_graph():
    """skewed_graph with every entry of a few columns dropped: those rows of H are referenced by nothing. Returns
    (A, dead columns, pad rows).

    The pad rows are the rows behind local column 0 on one rank (global row 0) and on each rank of the 2-way
    partition random_plans uses (its first owned row). Padding entries of the piece records, and the register kernel's
    lanes past a block's end, hold column 0 with value 0. So a kernel that multiplied them in would read exactly these
    rows. They are dead columns, and their rows of A are emptied too, so that nothing references them in the transposed
    product either."""
    A = skewed_graph(4000, 120000, seed=17)
    n = A.shape[0]
    pv = graphio.random_partvec(n, 2, seed=5)
    pads = np.unique([0] + [int(np.flatnonzero(pv == r)[0]) for r in range(2)])
    dead = np.union1d([7, 777, 2500, 3999], pads)
    keep = ~np.isin(A.col, dead) & ~np.isin(A.row, pads)
    return sp.coo_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape), dead, pads


def plant(X, rows, rs, nfeat=None):
    """+Inf, -Inf and NaN, in turn, in `nfeat` (default: a quarter) of the features of each of `rows`."""
    X = X.copy()
    f = X.shape[1]
    for i, r in enumerate(rows):
        feats = rs.choice(f, size=nfeat or max(1, f // 4), replace=False)
        X[r, feats] = (np.inf, -np.inf, np.nan)[i % 3]
    return X


def special_rows(A, unreferenced, k2_halo, rs):
    """Rows to plant in: referenced by the hub row (which is split into segments), by ordinary rows, halo rows on
    k = 2, and rows no stored entry references."""
    csr = sp.csr_matrix(A)
    deg = np.diff(csr.indptr)
    hub = int(np.argmax(deg))
    hub_cols = rs.choice(csr.indices[csr.indptr[hub]:csr.indptr[hub + 1]], 3, replace=False)
    ordinary = np.flatnonzero((deg >= 2) & (deg <= 8))
    ord_cols = [csr.indices[csr.indptr[r]] for r in rs.choice(ordinary, 4, replace=False)]
    halo = rs.choice(k2_halo, 3, replace=False)
    return np.unique(np.concatenate([hub_cols, ord_cols, halo])), np.asarray(unreferenced)


SPECIAL_CFGS = [("ring128", 128, {}), ("ring256", 256, {}), ("slices64", 256, {"ring_tile_floats": 64}),
                ("register40", 40, {}), ("register128", 128, {"kernel": 4})]


def k2_forward_backward(plans, H, G, f):
    """Per-rank pgcn_spmm with the halo rows copied in wire order, and A^T g with the partials routed to their owners
    and summed by pgcn_unpack_add: the k = 2 aggregation, all outputs NaN-filled first."""
    Z, own, part = [], [], []
    for p in plans:
        lp = p.lp
        Z.append(spmm_call(p, 0, f, H[lp.owned], H[lp.halo], None, {})[0])
        g, gh = spmm_call(p, 1, f, G[lp.owned], None, None, {})
        own.append(g); part.append(gh)
    Gd = []
    for r, p in enumerate(plans):
        lp, q = p.lp, 1 - r
        lq = plans[q].lp
        recv = offset_view((lp.S, f), 0, part[q][lq.recv_off[r]:lq.recv_off[r + 1]])
        g = offset_view((lp.m, f), 0, own[r])
        call("pgcn_unpack_add", p, recv.data_ptr(), g.data_ptr(), f, stream())
        Gd.append(g.clone())
    return Z, Gd


@pytest.mark.parametrize("cfg", SPECIAL_CFGS, ids=[c[0] for c in SPECIAL_CFGS])
def test_nonfinite_features(cfg):
    """+-Inf and NaN in chosen rows of H (forward) and of the upstream gradient (backward, the transposed product), on one
    rank (fused calls) and on two: NaN / +Inf / -Inf exactly where the fp64 product has them, the fp32 bound elsewhere.
    Finite magnitudes cannot overflow in any summation order, so the classes do not depend on it. A non-finite value in a
    row that no stored entry references changes no output bit: masked head / tail slots and padding lanes are never
    multiplied in."""
    name, f, opts = cfg
    A, dead_cols, pads = special_graph()
    n = A.shape[0]
    rs = np.random.RandomState(f)
    plans2 = random_plans(A, 2, link=False)
    p1 = random_plans(A, 1)[0]
    everyone = [p1] + plans2
    set_opts(everyone, edges_per_block=16, ring_edges_per_block=64, **opts)
    # local column 0 of every plan, where padding entries point, is one of the pad rows
    assert all(int(p.lp.owned[0]) in pads for p in everyone)
    empty_rows = np.flatnonzero(np.diff(sp.csr_matrix(A).indptr) == 0)       # unreferenced by the transposed product
    H0 = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G0 = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    hrows, hdead = special_rows(A, dead_cols, plans2[0].lp.halo, rs)
    grows, gdead = special_rows(sp.csr_matrix(A).T, np.union1d(pads, empty_rows[:4]), plans2[0].lp.halo, rs)
    assert np.isin(pads, hdead).all() and np.isin(pads, gdead).all() and np.isin(pads, empty_rows).all()
    H, G = plant(H0, np.concatenate([hrows, hdead]), rs), plant(G0, np.concatenate([grows, gdead]), rs)
    # NaN (0 * NaN = NaN) in every pad row, so a padding entry multiplied in cannot vanish as 0 * finite
    H[pads, 0], G[pads, 0] = np.nan, np.nan
    Hf, Gf = H.copy(), G.copy()                     # the same, with the unreferenced rows finite
    Hf[hdead], Gf[gdead] = H0[hdead], G0[gdead]
    with np.errstate(invalid="ignore"):
        Z64, G64 = orc.truth_forward(A, H), orc.truth_backward(A, G)
    assert np.isnan(Z64).any() and np.isinf(Z64).any() and np.isnan(G64).any() and np.isinf(G64).any()
    tolZ = fp32_tol(A, np.where(np.isfinite(H), H, 0), dmax(A))
    tolG = fp32_tol(A.T, np.where(np.isfinite(G), G, 0), dmax(A.T))

    def fused(X, Y):
        z = offset_view((n, f), 0)
        call("pgcn_forward", p1, offset_view((n, f), 0, X).data_ptr(), z.data_ptr(), f, stream())
        g = offset_view((n, f), 0)
        call("pgcn_backward", p1, offset_view((n, f), 0, Y).data_ptr(), g.data_ptr(), f, stream())
        return z.cpu().numpy(), g.cpu().numpy()

    z1, g1 = fused(H, G)
    assert p1.get_option("ring_long_rows_fwd" if (f % 128 == 0 and "kernel" not in opts) else "long_rows_fwd") > 0
    assert_ieee(z1, Z64, tolZ, "%s k=1 forward" % name)
    assert_ieee(g1, G64, tolG, "%s k=1 backward" % name)
    z1f, g1f = fused(Hf, Gf)
    assert np.array_equal(z1.view(np.int32), z1f.view(np.int32)), "%s: unreferenced rows changed the forward" % name
    assert np.array_equal(g1.view(np.int32), g1f.view(np.int32)), "%s: unreferenced rows changed the backward" % name
    Z2, G2 = k2_forward_backward(plans2, H, G, f)
    Z2f, G2f = k2_forward_backward(plans2, Hf, Gf, f)
    for r, p in enumerate(plans2):
        own = p.lp.owned
        assert_ieee(Z2[r].cpu().numpy(), Z64[own], tolZ[own], "%s k=2 r%d forward" % (name, r))
        assert_ieee(G2[r].cpu().numpy(), G64[own], tolG[own], "%s k=2 r%d backward" % (name, r))
        assert_bits(Z2[r], Z2f[r], "%s k=2 r%d: unreferenced rows changed the forward" % (name, r))
        assert_bits(G2[r], G2f[r], "%s k=2 r%d: unreferenced rows changed the backward" % (name, r))
    for p in everyone:
        p.close()


@pytest.mark.parametrize("f", [40, 128])
def test_zero_edge_values_times_inf_give_nan(f):
    """Edge values set to zero (a DropEdge mask) against +-Inf in H: the product 0 * Inf is NaN, as in torch.sparse.mm,
    which multiplies every stored entry. Rows that reach the Inf row through a zero edge are NaN in those features,
    rows that reach it through a non-zero edge are +-Inf."""
    A, _, _ = special_graph()
    n = A.shape[0]
    p = random_plans(A, 1)[0]
    p.bind_values()
    lp = p.lp
    rs = np.random.RandomState(f)
    H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    inf_rows = rs.choice(np.flatnonzero(np.bincount(lp.colidx, minlength=n) >= 4), 2, replace=False)
    H = plant(H, inf_rows, rs)                                          # a +Inf row and a -Inf row
    vals = lp.vals.copy()
    hit = np.flatnonzero(np.isin(lp.colidx, inf_rows))
    vals[hit[::2]] = 0.0                                                 # half of the edges into them are dropped
    vals[rs.choice(lp.nnz(), lp.nnz() // 10, replace=False)] = 0.0
    csr = local_csr(lp, vals)
    with np.errstate(invalid="ignore"):
        Z64 = csr @ H.astype(np.float64)
    assert np.isnan(Z64).any() and np.isinf(Z64).any()
    tol = fp32_tol(csr, np.where(np.isfinite(H), H, 0), dmax(csr))
    call("pgcn_plan_set_values", p, offset_view((lp.nnz(),), 0, vals).data_ptr(), stream())
    z = offset_view((n, f), 0)
    call("pgcn_forward", p, offset_view((n, f), 0, H).data_ptr(), z.data_ptr(), f, stream())
    assert_ieee(z.cpu().numpy(), Z64, tol, "zero edges f=%d" % f)
    p.close()


@pytest.mark.parametrize("f", [40, 128])
def test_sddmm_nonfinite(f):
    """NaN or Inf in a row of gZ or of H shows up in exactly the dvals of the edges that touch it (plain kernel at
    f = 40, ring kernel at f = 128), with the class of the fp64 dot product."""
    A, _, _ = special_graph()
    n = A.shape[0]
    p = random_plans(A, 1)[0]
    lp = p.lp
    rs = np.random.RandomState(f + 1)
    # one feature per row: a dot product with a single infinite term stays infinite
    H = plant(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.choice(n, 6, replace=False), rs, nfeat=1)
    gZ = plant(rs.uniform(-1, 1, size=(n, f)).astype(np.float32), rs.choice(n, 6, replace=False), rs, nfeat=1)
    d64, mag = sddmm64(lp, gZ, H)
    assert np.isnan(d64).any() and np.isinf(d64).any()
    dv = offset_view((lp.nnz(),), 0)
    call("pgcn_sddmm", p, offset_view((n, f), 0, gZ).data_ptr(), offset_view((n, f), 0, H).data_ptr(), None,
         dv.data_ptr(), f, stream())
    tol = 2.0 * (f + 2) * EPS * np.where(np.isfinite(mag), mag, 0) + 1e-30
    assert_ieee(dv.cpu().numpy(), d64, tol, "sddmm f=%d" % f)
    p.close()


def softmax64(rows, m, s):
    """torch.softmax semantics per row, in fp64: a row holding NaN or +Inf, or only -Inf, is all NaN; a single -Inf
    entry among finite ones gets 0."""
    with np.errstate(invalid="ignore", over="ignore"):
        mx = np.full(m, -np.inf)
        np.maximum.at(mx, rows, s)                    # np.maximum propagates NaN
        ex = np.exp(s - mx[rows])
        den = np.bincount(rows, ex, minlength=m)
        return ex / den[rows]


def test_edge_softmax_nonfinite_scores():
    """+-Inf and NaN in el and er: the NaN / zero / finite pattern of alpha, dpre and d_el equals that of an fp64 softmax
    with torch's semantics (checked against torch.softmax on the special rows); warp rows and a CTA hub row."""
    A = hub_graph()
    p = random_plans(A, 1)[0]
    p.bind_values()
    lp = p.lp
    m = lp.m
    rows, cols = edge_rows(lp), lp.colidx.astype(np.int64)
    deg = np.diff(lp.rowptr.astype(np.int64))
    rs = np.random.RandomState(3)
    el = rs.uniform(-2, 2, m).astype(np.float32)
    er = rs.uniform(-2, 2, m).astype(np.float32)
    hub = int(np.argmax(deg))
    assert deg[hub] > 1024
    hub_cols = cols[lp.rowptr[hub]:lp.rowptr[hub + 1]]
    busy = np.setdiff1d(np.flatnonzero(deg >= 3), [hub])
    el[rs.choice(busy, 3, replace=False)] = (np.inf, -np.inf, np.nan)
    er_cols = rs.choice(np.setdiff1d(np.flatnonzero(np.bincount(cols, minlength=m) >= 2), hub_cols), 9, replace=False)
    er[er_cols] = (np.inf, -np.inf, np.nan, -np.inf, -np.inf, -np.inf, -np.inf, np.inf, np.nan)
    er[hub_cols[5]] = -np.inf                                           # one -Inf entry in the CTA row
    slope = 0.2
    with np.errstate(invalid="ignore"):
        s = el.astype(np.float64)[rows] + er.astype(np.float64)[cols]
        s = np.where(s > 0, s, slope * s)
    a64 = softmax64(rows, m, s)
    special = np.unique(rows[~np.isfinite(s)])
    assert (a64 == 0).any() and np.isnan(a64).any() and (np.isfinite(a64) & (a64 > 0)).any()
    for r in special:                                                  # the fp64 reference is torch's softmax
        lo, hi = lp.rowptr[r], lp.rowptr[r + 1]
        t = torch.softmax(torch.from_numpy(s[lo:hi]), 0).numpy()
        assert np.array_equal(np.isnan(t), np.isnan(a64[lo:hi])) and np.array_equal(t == 0, a64[lo:hi] == 0)
    dal = rs.uniform(-1, 1, lp.nnz()).astype(np.float32)
    t = lambda x: offset_view(x.shape, 0, x)
    alpha = offset_view((lp.nnz(),), 0)
    call("pgcn_edge_softmax", p, t(el).data_ptr(), t(er).data_ptr(), None, slope, alpha.data_ptr(), stream())
    dpre, d_el = offset_view((lp.nnz(),), 0), offset_view((m,), 0)
    call("pgcn_edge_softmax_backward", p, t(el).data_ptr(), t(er).data_ptr(), None, alpha.data_ptr(),
         t(dal).data_ptr(), slope, dpre.data_ptr(), d_el.data_ptr(), stream())
    alpha, dpre, d_el = (x.cpu().numpy().astype(np.float64) for x in (alpha, dpre, d_el))
    sl = np.where(s > 0, 1.0, slope)
    with np.errstate(invalid="ignore"):
        c64 = np.bincount(rows, a64 * dal, minlength=m)
        p64 = a64 * (dal - c64[rows]) * sl
        e64 = np.bincount(rows, p64, minlength=m)
    assert (a64[lp.rowptr[hub]:lp.rowptr[hub + 1]] == 0).sum() == 1
    for got, want, nm in ((alpha, a64, "alpha"), (dpre, p64, "dpre"), (d_el, e64, "d_el")):
        assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN pattern" % nm
        if nm != "d_el":      # a row sum of dpre is 0 in exact arithmetic when its slopes agree: only empty rows are 0
            assert np.array_equal(got == 0, want == 0), "%s: zero pattern" % nm
        else:
            assert (got[deg == 0] == 0).all()
        assert np.isfinite(got[~np.isnan(want)]).all(), "%s: finite pattern" % nm
    fin = np.isfinite(s) & ~np.isnan(a64)
    smax = np.zeros(m)
    np.maximum.at(smax, rows[np.isfinite(s)], np.abs(s[np.isfinite(s)]))
    tol_a = a64 * EPS * (8 * smax[rows] + 4 * deg[rows] + 32) + 1e-38
    assert (np.abs(alpha - a64)[fin] <= tol_a[fin]).all()
    p.close()


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("f", [40, 128])
def test_fused_relu_keeps_nan(k, f):
    """The fused ReLU on a pre-activation holding NaN, +Inf and -Inf: NaN stays NaN (torch.relu), -Inf becomes 0, +Inf
    stays +Inf; on one rank and on three with overlap, where rows are clamped by the last writer (`final`) and split rows
    by the fixup. At the layer level PSpMMRelu(A, linear(H)) has the NaN pattern of relu(PSpMM(A, linear(H)))."""
    A, _, _ = special_graph()
    n = A.shape[0]
    plans = random_plans(A, k)
    rs = np.random.RandomState(k * f)
    X0 = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    hrows, _ = special_rows(A, [], planmod.build_local_plan(A, graphio.random_partvec(n, 2, seed=5), 0, 2).halo, rs)
    X = plant(X0, hrows, rs)
    with np.errstate(invalid="ignore"):
        pre64 = orc.truth_forward(A, X)
    want = np.where(np.isnan(pre64), np.nan, np.maximum(pre64, 0.0))
    assert np.isnan(want).any() and (want == np.inf).any() and (pre64 == -np.inf).any()
    tol = fp32_tol(A, np.where(np.isfinite(X), X, 0), dmax(A))
    set_opts(plans, overlap=1, relu=1, edges_per_block=16, ring_edges_per_block=64)
    ins = [offset_view((p.lp.m, f), 0, X[p.lp.owned]) for p in plans]
    outs = [offset_view((p.lp.m, f), 0) for p in plans]
    run_ranks([lambda p=p, x=x, y=y: call("pgcn_forward", p, x.data_ptr(), y.data_ptr(), f, stream())
               for p, x, y in zip(plans, ins, outs)])
    for r, p in enumerate(plans):
        own = p.lp.owned
        z = outs[r].cpu().numpy()
        assert_ieee(z, want[own], tol[own], "relu k=%d f=%d r%d" % (k, f, r))
        fin = np.isfinite(pre64[own]) & (pre64[own] < -tol[own])
        assert (z[fin] == 0).all()
        p.set_option("relu", 0)
    if k == 1:
        torch.manual_seed(f)
        lin = torch.nn.Linear(f, f).to(dev())
        Hd = torch.from_numpy(plant(X0, hrows[:3], rs)).to(dev())
        with torch.no_grad():
            a = PSpMMRelu.apply(plans[0], lin(Hd))
            b = F.relu(PSpMM.apply(plans[0], lin(Hd)))
        assert torch.isnan(b).any()
        assert torch.equal(torch.isnan(a), torch.isnan(b))
    for p in plans:
        p.close()


@pytest.mark.parametrize("cfg", SPECIAL_CFGS, ids=[c[0] for c in SPECIAL_CFGS])
def test_subnormal_products(cfg):
    """H scaled by 2^-140: every product and sum is subnormal. |Z - Z64| <= 2 (d+2) 2^-24 (|A||H|) + (d+1) 2^-149, and
    Z is non-zero wherever |Z64| exceeds that bound: a flush-to-zero or fast-math build, or approximate intrinsics, in
    the ring, register or SDDMM kernels fail here."""
    name, f, opts = cfg
    A, _, _ = special_graph()
    n = A.shape[0]
    p = random_plans(A, 1)[0]
    set_opts([p], edges_per_block=16, ring_edges_per_block=64, **opts)
    lp = p.lp
    rs = np.random.RandomState(f)
    H = (rs.uniform(-1, 1, size=(n, f)) * 2.0 ** -140).astype(np.float32)
    gZ = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
    assert (np.abs(H[H != 0]) < 2.0 ** -126).all()
    rdeg, tdeg = np.diff(lp.rowptr)[:, None], np.diff(lp.t_rowptr)[:, None]      # per-row additions of the kernels

    def check(got, want, mag, deg, what):
        bound = 2.0 * (deg + 2) * EPS * mag + (deg + 1) * 2.0 ** -149
        err = np.abs(got.astype(np.float64) - want)
        assert (err <= bound).all(), "%s: %d entries beyond the subnormal bound" % (what, int((err > bound).sum()))
        big = np.abs(want) > bound
        assert big.any() and (got[big] != 0).all(), "%s: %d results flushed to zero" % (what, int((got[big] == 0).sum()))

    z = offset_view((n, f), 0)
    call("pgcn_forward", p, offset_view((n, f), 0, H).data_ptr(), z.data_ptr(), f, stream())
    check(z.cpu().numpy(), orc.truth_forward(A, H), orc.abs_bound(A, H), rdeg, name + " forward")
    g = offset_view((n, f), 0)
    call("pgcn_backward", p, offset_view((n, f), 0, H).data_ptr(), g.data_ptr(), f, stream())
    check(g.cpu().numpy(), orc.truth_backward(A, H), orc.abs_bound(sp.csr_matrix(A).T, H), tdeg, name + " backward")
    d64, mag = sddmm64(lp, gZ, H)
    dv = offset_view((lp.nnz(),), 0)
    call("pgcn_sddmm", p, offset_view((n, f), 0, gZ).data_ptr(), offset_view((n, f), 0, H).data_ptr(), None,
         dv.data_ptr(), f, stream())
    check(dv.cpu().numpy(), d64, mag, f, name + " sddmm")
    p.close()


# ---- C. operands over 4 GiB ----------------------------------------------------------------------------------------

def test_operands_over_4_gib():
    """One plan with f_max = 1024 and n = 1 100 000 rows: H and Z are 4.5 GB each, and rows >= 2^20 lie past byte
    offset 2^32. R-MAT with hub rows, rows whose columns are all >= 2^20, and columns >= 2^20 that the hub rows
    reference. Forward on the ring (tile 256, 4 tiles) and register kernels, backward, and the SDDMM (plain kernel at
    f = 1024), each checked against fp64 on the top-degree rows, every planted row and a random sample."""
    free, _ = torch.cuda.mem_get_info(dev())
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GiB of free device memory, %.1f GiB free (the GPU is shared)" % (free / 2 ** 30))
    n, f, far = 1_100_000, 1024, 1 << 20
    rs = np.random.RandomState(0)
    A = sp.coo_matrix(graphio.synthetic_graph(n, 3_000_000, seed=2, permute=False))
    deg = np.bincount(A.row, minlength=n)
    hubs = np.argsort(deg)[-2:]
    planted = np.concatenate([rs.choice(far, 16, replace=False), rs.choice(np.arange(far, n), 16, replace=False)])
    keep = ~np.isin(A.row, planted)
    prow = np.repeat(planted, 24)
    hrow = np.repeat(hubs, 600)
    row = np.concatenate([A.row[keep], prow, hrow])
    col = np.concatenate([A.col[keep], rs.randint(far, n, prow.size), rs.randint(far, n, hrow.size)])
    val = np.concatenate([A.data[keep], rs.uniform(0.05, 0.5, prow.size + hrow.size).astype(np.float32)])
    A = sp.coo_matrix((val, (row, col)), shape=(n, n))
    p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev())
    lp = p.lp
    csr = sp.csr_matrix((lp.vals.astype(np.float64), lp.colidx, lp.rowptr), shape=(n, n))
    cdeg = np.diff(lp.rowptr)
    sample = np.unique(np.concatenate([np.argsort(cdeg)[-16:], planted, rs.choice(n, 512, replace=False)]))
    assert (sample >= far).any()

    def rows_of(X, idx):
        return X[torch.from_numpy(np.asarray(idx, np.int64)).to(dev())].cpu().numpy().astype(np.float64)

    def check_rows(M, X, Y, idx, what):
        sub = M[idx]
        used = np.unique(sub.indices)
        loc = sp.csr_matrix((sub.data, np.searchsorted(used, sub.indices), sub.indptr), shape=(len(idx), len(used)))
        Xu = rows_of(X, used)
        want, mag = loc @ Xu, abs(loc) @ np.abs(Xu)
        d = np.diff(sub.indptr)[:, None]
        assert_close_fp32(rows_of(Y, idx), want, 2.0 * (d + 2) * EPS * mag + 1e-30, what)

    gen = torch.Generator(device=dev()).manual_seed(3)
    H = torch.rand((n, f), device=dev(), generator=gen) * 2 - 1
    # the default path: kernel 0 and no tuned or set ring tile, i.e. the full width, 256 floats when f % 256 == 0 (4 tiles)
    assert p.get_option("kernel") == 0 and p.get_option("ring_tile_floats") == 0
    assert H.data_ptr() % 16 == 0
    Z = op.aggregate_forward(p, H)
    # only the ring schedule of the forward matrix exists: the forward ran on the ring kernel
    assert p.get_option("ring_blocks_fwd") > 0 and p.get_option("blocks_fwd") == 0
    check_rows(csr, H, Z, sample, "forward ring")
    p.set_option("kernel", 4)
    Z2 = op.aggregate_forward(p, H)
    assert p.get_option("blocks_fwd") > 0                          # the register kernel's schedule, built by this call
    check_rows(csr, H, Z2, sample, "forward register")
    del Z2
    p.set_option("kernel", 0)
    tsample = np.unique(np.concatenate([np.argsort(np.diff(lp.t_rowptr))[-16:], rs.randint(far, n, 64),
                                        rs.choice(n, 512, replace=False)]))
    Gt = op.aggregate_backward(p, Z)                               # A^T Z: H, Z and Gt alive
    tcsr = sp.csr_matrix((lp.t_vals.astype(np.float64), lp.t_colidx, lp.t_rowptr), shape=(n, n))
    check_rows(tcsr, Z, Gt, tsample, "backward")
    del Gt
    dv = torch.full((lp.nnz(),), float("nan"), device=dev())
    call("pgcn_sddmm", p, Z.data_ptr(), H.data_ptr(), None, dv.data_ptr(), f, stream())
    erow = np.repeat(np.arange(n), cdeg)
    edges = np.unique(np.concatenate([np.flatnonzero(np.isin(erow, planted)), np.flatnonzero(np.isin(erow, hubs)),
                                      rs.choice(lp.nnz(), 2048, replace=False)]))
    assert (lp.colidx[edges] >= far).any() and (erow[edges] >= far).any()
    g, h = rows_of(Z, erow[edges]), rows_of(H, lp.colidx[edges])
    want, mag = (g * h).sum(1), (np.abs(g) * np.abs(h)).sum(1)
    assert_close_fp32(rows_of(dv[:, None], edges)[:, 0], want, 2.0 * (f + 2) * EPS * mag + 1e-30, "sddmm")
    del H, Z, dv
    p.close()
    torch.cuda.empty_cache()
