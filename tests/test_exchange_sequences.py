"""Exchange sequences: every call that exchanges rows between ranks, in long scripts whose ranks run out of step.

The peer transport keeps one exchange epoch per plan in device memory and two slabs per direction, picked by the
epoch's parity (DESIGN.md §4, "Exchange"). A rank may run one exchange ahead of its peers, and an operand is free for
the caller in stream order once the call returns. This file drives that protocol the way training does, not in lockstep:

  * partitions, all ranks in this process, linked over the peer transport: karate on 3 ranks, a skewed R-MAT graph
    (20 000 vertices) on 4, a small R-MAT graph on 6, a hand-built degenerate partition on 4 (an empty rank, a rank
    without halo rows whose rows the others read, two ranks that exchange nothing, empty rows, one-entry rows and hub
    rows long enough to be split) and a "sender" partition on 4 whose rank 0 sends far more rows than it computes;
  * one script per partition, the same on every rank: every exchanging entry point of the header at both epoch
    parities, set_values between calls, widths that change between calls, fresh inputs for every call and outputs
    that start as NaN;
  * the script enqueued in lockstep (the baseline: every output against fp64), rank-major, reverse rank-major, and
    interleaved with seeded sleeps; every order must give the lockstep bits and advance every epoch once per exchange;
  * the sleep run and the reverse rank-major run once more with every operand in one buffer per rank, refilled before
    each call and poisoned with NaN right after it (the caller's operands are free in stream order once a call
    returns);
  * two-layer autograd stacks of every operator, forward and backward enqueued rank-major without a host
    synchronisation, their temporaries freed by Python, against the bits of the lockstep run;
  * CUDA-graph replays back to back, rank-major; the degenerate script in one process per rank over CUDA IPC with its
    own sleeps and the host-buffer forward; NCCL against the peer transport on two GPUs.

A new exchanging entry point of the header needs a place in EXCHANGES and in the script (the CPU tests fail until then).
"""
import os
import re

import numpy as np
import pytest
import torch

from harness import ROOT, EPS, bits, dev, identical, linked_plans, problem, run_ranks, spawn_ranks, stream
from helpers import fp32_tol
from pgcn_b200 import cabi, graphio, plan as planmod

HEADER = os.path.join(ROOT, "include", "pgcn_b200.h")
SEED = 2024
SLOPE = 0.2
NAN_BITS = 0x7FC00000

# Every function of the header, by whether it exchanges rows between ranks. An exchanging function names the script op
# that calls it, or why the script has none.
EXCHANGES = {
    "pgcn_forward": "fwd", "pgcn_backward": "bwd", "pgcn_forward_keep_halo": "keep", "pgcn_halo_rows": "halo",
    "pgcn_forward_heads": "fwd_heads", "pgcn_backward_heads": "bwd_heads", "pgcn_forward_max": "fwd_max",
    "pgcn_backward_max": "bwd_max", "pgcn_forward_gatv2": "fwd_v2", "pgcn_backward_gatv2": "bwd_v2",
    "pgcn_forward_host_async": "host", "pgcn_forward_host": "host",
    "pgcn_exchange": None,       # the NCCL step of the step-by-step pieces: no peer transport, no epoch
}
LOCAL = {
    "pgcn_version", "pgcn_device_count", "pgcn_last_error", "pgcn_plan_create", "pgcn_plan_destroy",
    "pgcn_plan_set_option", "pgcn_plan_get_option", "pgcn_plan_autotune", "pgcn_plan_prepare", "pgcn_debug_schedule",
    "pgcn_plan_slab", "pgcn_algorithmic_bytes", "pgcn_launch_count", "pgcn_comm_unique_id", "pgcn_comm_init",
    "pgcn_comm_share", "pgcn_p2p_export", "pgcn_p2p_import", "pgcn_spmm", "pgcn_pack", "pgcn_unpack_add",
    "pgcn_plan_bind_values", "pgcn_plan_set_values", "pgcn_sddmm", "pgcn_edge_softmax", "pgcn_edge_softmax_backward",
    "pgcn_edge_softmax_heads", "pgcn_edge_softmax_backward_heads", "pgcn_sddmm_heads", "pgcn_forward_host_wait",
}

# the inputs of each op: global feature arrays (n rows, a rank takes its owned rows), "xlh" the halo rows of xl,
# per-rank entry arrays (alpha, vals, arg) and att
INPUTS = {
    "fwd": ("H",), "host": ("H",), "bwd": ("gZ",), "keep": ("H",), "halo": ("X",), "fwd_heads": ("alpha", "H"),
    "bwd_heads": ("alpha", "gZ"), "fwd_max": ("H",), "bwd_max": ("arg", "gZ"), "fwd_v2": ("xl", "xr", "att"),
    "bwd_v2": ("alpha", "gZ", "xl", "xlh", "xr", "att"), "values": ("vals",),
}
NAMES = ("H", "gZ", "X", "alpha", "arg", "xl", "xr", "att", "vals")


# ---- partitions ------------------------------------------------------------------------------------------------------

def degenerate_graph():
    """(A, partvec) on 4 ranks. Ranks 0-2 own 1000 rows each and rank 3 none. Rank 2's rows read only rank 2's columns,
    ranks 0 and 1 read their own and rank 2's, never each other's. Every tenth row is empty and the next has one entry;
    row 7 (rank 0) has 1900 entries and row 2007 (rank 2) 990, more than either kernel's long-row threshold."""
    n = 3000
    rs = np.random.RandomState(41)
    pv = np.repeat(np.arange(3), 1000).astype(np.int64)
    allowed = {0: np.r_[0:1000, 2000:3000], 1: np.r_[1000:2000, 2000:3000], 2: np.arange(2000, 3000)}
    rows, cols = [], []
    for i in range(n):
        d = {3: 0, 4: 1}.get(i % 10, rs.randint(2, 14))
        d = {7: 1900, 2007: 990}.get(i, d)
        c = rs.choice(allowed[int(pv[i])], size=d, replace=False)
        if d > 1 and i % 7 == 0:
            c = np.r_[c, c[:1]]                             # a duplicated entry
        rows.append(np.full(len(c), i)); cols.append(c)
    row, col = np.concatenate(rows), np.concatenate(cols)
    import scipy.sparse as sp
    A = sp.coo_matrix((rs.uniform(0.25, 1.0, len(row)).astype(np.float32), (row, col)), shape=(n, n))
    return A, pv


def sender_graph():
    """(A, partvec) on 4 ranks where rank 0 sends far more than it computes. Rank 0 owns 18 000 rows, each with one entry
    in a column of another rank (among the first 32 rows of each), so its own-column block is empty and its halo block
    is small. Ranks 1-3 own 2 000 rows each, with ten entries in rank 0's columns and two in their own: rank 0's puts
    carry about 10 000 rows to each peer."""
    import scipy.sparse as sp
    rs = np.random.RandomState(43)
    pv = np.r_[np.zeros(18000), np.repeat([1, 2, 3], 2000)].astype(np.int64)
    r0 = np.arange(18000)
    c0 = 18000 + 2000 * rs.randint(0, 3, 18000) + rs.randint(0, 32, 18000)
    r1 = np.repeat(np.arange(18000, 24000), 12)
    c1 = np.concatenate([np.r_[rs.choice(18000, 10, replace=False), 18000 + 2000 * ((i - 18000) // 2000) +
                               rs.randint(0, 2000, 2)] for i in range(18000, 24000)])
    row, col = np.r_[r0, r1], np.r_[c0, c1]
    return sp.coo_matrix((rs.uniform(0.25, 1.0, len(row)).astype(np.float32), (row, col)), shape=(24000, 24000)), pv


PARTS = ("karate", "skewed", "rmat_k6", "degenerate", "sender")


class Part:
    """A partition: the local plans of its ranks, its width limit and the cycle of widths its script walks."""

    def __init__(self, name, k=None):
        self.name = name
        if name == "karate":
            A, pv, k = problem("karate")
            self.fmax, self.widths = 64, (64, 36, 64, 16)
        elif name == "skewed":
            from test_gpu_parity import skewed_graph
            A = skewed_graph(20000, 400000, seed=17)
            k = k or 4
            pv = graphio.random_partvec(20000, k, seed=6)
            self.fmax, self.widths = 128, (128, 36, 128, 64, 16)
        elif name == "rmat_k6":
            A, k = graphio.synthetic_graph(3000, 40000, seed=23), 6
            pv = graphio.random_partvec(3000, k, seed=8)
            self.fmax, self.widths = 16, (16, 8, 16, 12)
        elif name == "sender":
            (A, pv), k = sender_graph(), 4
            self.fmax, self.widths = 128, (128, 36, 128, 64)
        else:
            (A, pv), k = degenerate_graph(), 4
            self.fmax, self.widths = 128, (128, 36, 128, 16)
        self.A, self.pv, self.k, self.n = A, pv, k, A.shape[0]
        self.lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
        self._edges = None

    def edges(self):
        """Per rank (local rows, global rows, global columns) of its entries, int64, and the largest row or column
        count of the whole matrix."""
        if self._edges is None:
            out, cdeg, rdeg = [], np.zeros(self.n, np.int64), 0
            for lp in self.lps:
                rl = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
                gc = np.concatenate([lp.owned, lp.halo]).astype(np.int64)[lp.colidx.astype(np.int64)]
                np.add.at(cdeg, gc, 1)
                rdeg = max(rdeg, int(np.bincount(rl, minlength=1).max()) if lp.m else 0)
                out.append((rl, lp.owned[rl].astype(np.int64), gc))
            self._edges = out, max(rdeg, int(cdeg.max()))
        return self._edges


_PARTS = {}


def part(name):
    if name not in _PARTS:
        _PARTS[name] = Part(name)
    return _PARTS[name]


# ---- the script ------------------------------------------------------------------------------------------------------

def variants():
    """Every exchanging call shape once; an even number, so that a script of two copies and one call between them meets
    each at both epoch parities."""
    return [dict(op="fwd", overlap=1), dict(op="fwd", overlap=0), dict(op="fwd", overlap=1, relu=1),
            dict(op="bwd", overlap=1), dict(op="bwd", overlap=0), dict(op="keep"), dict(op="halo", w=4),
            dict(op="halo", w=0), dict(op="fwd_heads", K=2), dict(op="fwd_heads", K=4), dict(op="bwd_heads", K=2),
            dict(op="bwd_heads", K=4), dict(op="fwd_max"), dict(op="bwd_max"), dict(op="fwd_v2", K=2),
            dict(op="bwd_v2", K=4)]


def make_script(seed, fmax, widths, host=False):
    """The call script of a partition: the same on every rank, from the seed alone. Each call carries its op, its options
    (overlap, relu; they change only between calls), its width f and the key its inputs are drawn from. host=True adds
    the host-buffer forward four times (pgcn_forward_host_async + pgcn_forward_host_wait, and pgcn_forward_host), for
    the ranks that run in processes of their own; the other calls and their keys are the same."""
    rs = np.random.RandomState(seed)
    base = variants()
    half = [dict(base[i]) for i in rs.permutation(len(base))]
    calls = half + [dict(op="fwd", overlap=1)] + [dict(c) for c in half]
    for pos, restore in ((4, 0), (13, 0), (27, 1)):
        calls.insert(pos, dict(op="values", restore=restore))
    for j, c in enumerate(calls):
        c["key"] = j
        c.setdefault("overlap", 1)
        c.setdefault("relu", 0)
        if c["op"] != "values":
            f = widths[j % len(widths)]
            c["f"] = min(f, 36) if c["op"] in ("fwd_v2", "bwd_v2") else f     # keeps the numpy GATv2 bound small
            if c["op"] == "halo" and c["w"] == 0:
                c["w"] = c["f"]
    if host:
        # in pairs, so that every other call keeps its epoch parity, and each form meets both parities
        for n, (pos, sync) in enumerate(((20, 1), (20, 0), (9, 0), (9, 1))):
            calls.insert(pos, dict(op="host", sync=sync, overlap=1, relu=0, f=widths[n % len(widths)], key=1000 + n))
    return calls


def exchanges(script):
    return sum(c["op"] != "values" for c in script)


def parities(script):
    """The epoch parity of each exchanging call (its exchange number, counted from 1, mod 2)."""
    out, e = [], 0
    for c in script:
        e += c["op"] != "values"
        out.append(e & 1 if c["op"] != "values" else None)
    return out


def draw(P, seed, call):
    """The inputs of one call as host arrays: {name: global array} and [{name: per-rank array}], drawn from (seed, the
    call's key, the name[, the rank]) alone."""
    f, K, op = call.get("f"), call.get("K", 1), call["op"]
    glob, per = {}, [{} for _ in range(P.k)]
    for name in INPUTS[op]:
        if name == "xlh":
            continue
        key = [seed, call["key"], NAMES.index(name)]
        if name in ("H", "gZ", "xl", "xr", "X"):
            glob[name] = np.random.RandomState(key).uniform(-1, 1, (P.n, call["w"] if name == "X" else f)).astype(
                np.float32)
        elif name == "att":
            glob[name] = (np.random.RandomState(key).standard_normal((K, f // K)) / np.sqrt(f // K)).astype(np.float32)
        for r, lp in enumerate(P.lps):
            rs = np.random.RandomState(key + [1 + r])
            if name == "alpha":
                per[r][name] = rs.uniform(0, 1, (lp.nnz(), K)).astype(np.float32)
            elif name == "vals" and not call["restore"]:
                per[r][name] = rs.uniform(0.5, 1.5, lp.nnz()).astype(np.float32)
            elif name == "arg":
                deg = np.diff(lp.rowptr.astype(np.int64))
                pick = (rs.uniform(0, 1, (lp.m, f)) * deg[:, None]).astype(np.int64)
                per[r][name] = np.where(deg[:, None] > 0, lp.rowptr[:-1, None] + pick, -1).astype(np.int32)
    return glob, per


def stage(P, seed, script, ranks=None):
    """Every call's inputs on the device, per rank, before anything is enqueued (a host-to-device copy behind a spinning
    wait would never finish); also the global arrays, for the fp64 references."""
    staged, globs = [], []
    for c in script:
        glob, per = draw(P, seed, c)
        row = []
        for r, lp in enumerate(P.lps):
            if ranks is not None and r not in ranks:
                row.append(None)
                continue
            x = {}
            for name in INPUTS[c["op"]]:
                if name == "xlh":
                    u = glob["xl"][lp.halo]
                elif name == "att":
                    u = glob[name]
                elif name in glob:
                    u = glob[name][lp.owned]
                elif name in per[r]:
                    u = per[r][name]
                else:
                    continue                                # restore the creation values
                x[name] = torch.from_numpy(np.ascontiguousarray(u)).to(dev())
            row.append(x)
        staged.append(row)
        globs.append({name: torch.from_numpy(u).to(dev()) for name, u in glob.items()} if ranks is None else None)
    return staged, globs


# ---- enqueueing ------------------------------------------------------------------------------------------------------

def out_shapes(lp, c):
    m, h, nnz, f, K = lp.m, lp.h, lp.nnz(), c.get("f"), c.get("K", 1)
    return {"fwd": {"Z": (m, f)}, "host": {"Z": (m, f)}, "bwd": {"G": (m, f)}, "keep": {"Z": (m, f), "Hh": (h, f)},
            "halo": {"Xh": (h, c.get("w"))}, "fwd_heads": {"Z": (m, f), "Hh": (h, f)}, "bwd_heads": {"G": (m, f)},
            "fwd_max": {"Z": (m, f), "arg": (m, f)}, "bwd_max": {"G": (m, f)},
            "fwd_v2": {"alpha": (nnz, K), "Z": (m, f), "Hh": (h, f)},
            "bwd_v2": {"work": (nnz, K), "dxl": (m, f), "dxr": (m, f), "datt": (K, f // K if f else 0)},
            "values": {}}[c["op"]]


def poisoned(shape, name):
    if name == "arg":
        return torch.full(shape, NAN_BITS, dtype=torch.int32, device=dev())
    return torch.full(shape, float("nan"), device=dev())


def _p(u):
    return u.data_ptr() if u is not None and u.numel() else None


def enqueue(lib, plan, c, x, y):
    """The C-ABI call of script call c for one rank on the current stream: x its inputs, y its outputs."""
    h, s, f, K, op = plan.handle, stream(), c.get("f"), c.get("K", 1), c["op"]
    plan.set_option("overlap", c["overlap"])
    plan.set_option("relu", c["relu"])
    g = lambda name: _p(x.get(name))
    o = lambda name: _p(y.get(name))
    if op == "values":
        rc = lib.pgcn_plan_set_values(h, g("vals"), s)
    elif op == "fwd":
        rc = lib.pgcn_forward(h, g("H"), o("Z"), f, s)
    elif op == "bwd":
        rc = lib.pgcn_backward(h, g("gZ"), o("G"), f, s)
    elif op == "keep":
        rc = lib.pgcn_forward_keep_halo(h, g("H"), o("Z"), o("Hh"), f, s)
    elif op == "halo":
        rc = lib.pgcn_halo_rows(h, g("X"), o("Xh"), c["w"], s)
    elif op == "fwd_heads":
        rc = lib.pgcn_forward_heads(h, K, g("alpha"), g("H"), o("Z"), o("Hh"), f, s)
    elif op == "bwd_heads":
        rc = lib.pgcn_backward_heads(h, K, g("alpha"), g("gZ"), o("G"), f, s)
    elif op == "fwd_max":
        rc = lib.pgcn_forward_max(h, g("H"), o("Z"), o("arg"), f, s)
    elif op == "bwd_max":
        rc = lib.pgcn_backward_max(h, g("arg"), g("gZ"), o("G"), f, s)
    elif op == "fwd_v2":
        rc = lib.pgcn_forward_gatv2(h, K, g("xl"), g("xr"), g("att"), SLOPE, o("alpha"), o("Z"), o("Hh"), f, s)
    elif op == "bwd_v2":
        rc = lib.pgcn_backward_gatv2(h, K, g("alpha"), g("gZ"), g("xl"), g("xlh"), g("xr"), g("att"), SLOPE,
                                     o("work"), o("dxl"), o("dxr"), o("datt"), f, s)
    else:
        raise ValueError(op)
    plan.set_option("relu", 0)
    cabi.check(rc, h)


def fresh(P, script):
    """New linked plans of the partition, bound and prepared for every width of the script under both overlap settings
    (so that no call does set-up work while a peer's wait kernel spins)."""
    plans = linked_plans(P.lps, P.fmax, 1)
    for p in plans:
        for ov in (0, 1):
            p.set_option("overlap", ov)
            for f in sorted({c["f"] for c in script if "f" in c}):
                p.prepare(f)
    return plans


SLEEPS = (0, 10 ** 5, 10 ** 6)


def sleep_plan(seed, ncalls, k):
    """(cycles [ncalls, k], enqueue order of the ranks per call): each call delays a seeded subset of the ranks."""
    rs = np.random.RandomState([seed, 99])
    cyc = np.asarray(SLEEPS)[rs.choice(3, size=(ncalls, k), p=(0.5, 0.25, 0.25))]
    return cyc, [rs.permutation(k) for _ in range(ncalls)]


def warm_torch_kernels(streams):
    """Launch, once on every stream, each torch kernel the out-of-step runs enqueue behind a spinning wait: the first
    launch of a kernel loads its module, and that load synchronises with the device, i.e. with a wait kernel whose peer
    this host thread has not enqueued yet (every rank would hang). A new torch op or dtype in run() belongs here."""
    for s in streams:
        with torch.cuda.stream(s):
            for dt in (torch.float32, torch.int32):
                u = poisoned((64, 8), "arg" if dt == torch.int32 else "Z")
                v = u.clone()
                v[:32].copy_(u[:32])
                v.fill_(NAN_BITS if dt == torch.int32 else float("nan"))
            torch.cuda._sleep(1)
    torch.cuda.synchronize()


def run(P, script, staged, order, seed=SEED, reuse=False):
    """Enqueue the script on fresh plans in `order` (lockstep, rank-major, reverse, skewed); returns
    (outputs[call][rank], epochs)."""
    lib = cabi.load()
    plans = fresh(P, script)
    # reused operands: the callers' streams at the exchange stream's (highest) priority, so that the poisoning after a
    # call competes with the call's puts instead of queueing behind them
    streams = [torch.cuda.Stream(device=dev(), priority=-100 if reuse else 0) for _ in plans]
    warm_torch_kernels(streams)
    k = P.k
    outs = [[None] * k for _ in script]
    bufs = None
    if reuse:
        # one buffer per operand and rank, sized for its largest use, NaN until a call fills it
        bufs = [{} for _ in range(k)]
        for j, c in enumerate(script):
            for r, lp in enumerate(P.lps):
                shapes = {n: (tuple(u.shape), u.dtype) for n, u in staged[j][r].items()}
                shapes.update({"out_" + n: (s, torch.int32 if n == "arg" else torch.float32)
                               for n, s in out_shapes(lp, c).items()})
                for n, (s, dt) in shapes.items():
                    need = int(np.prod(s))
                    if n not in bufs[r] or bufs[r][n][0] < need:
                        bufs[r][n] = (need, dt)
        bufs = [{n: poisoned((need,), "arg" if dt == torch.int32 else n) for n, (need, dt) in b.items()}
                for b in bufs]

    def one(r, j):
        c, lp = script[j], P.lps[r]
        if not reuse:
            y = {n: poisoned(s, n) for n, s in out_shapes(lp, c).items()}
            enqueue(lib, plans[r], c, staged[j][r], y)
            outs[j][r] = y
            return
        x = {}
        for n, u in staged[j][r].items():
            x[n] = bufs[r][n][:u.numel()].view(u.shape)
            x[n].copy_(u)
        y = {n: bufs[r]["out_" + n][:int(np.prod(s))].view(s) for n, s in out_shapes(lp, c).items()}
        enqueue(lib, plans[r], c, x, y)
        for u in list(x.values()):                    # the inputs first: the earliest a caller may reuse them
            u.fill_(NAN_BITS if u.dtype == torch.int32 else float("nan"))
        outs[j][r] = {n: u.clone() for n, u in y.items()}
        for u in y.values():
            u.fill_(NAN_BITS if u.dtype == torch.int32 else float("nan"))

    if order == "lockstep":
        for j in range(len(script)):
            run_ranks(plans, lambda r: one(r, j), streams)
    else:
        torch.cuda.synchronize()
        if order in ("rank-major", "reverse"):
            for r in (range(k) if order == "rank-major" else reversed(range(k))):
                with torch.cuda.stream(streams[r]):
                    for j in range(len(script)):
                        one(r, j)
        else:
            cyc, perm = sleep_plan(seed, len(script), k)
            for j in range(len(script)):
                for r in perm[j]:
                    with torch.cuda.stream(streams[r]):
                        if cyc[j, r]:
                            torch.cuda._sleep(int(cyc[j, r]))
                        one(r, j)
        torch.cuda.synchronize()
    epochs = [p.get_option("epoch") for p in plans]
    for p in plans:
        p.close()
    return outs, epochs


# ---- fp64 references -------------------------------------------------------------------------------------------------

def _close(got, want, tol, what):
    u = got.cpu().numpy().astype(np.float64)
    err = np.abs(u - want)
    assert np.isfinite(u).all() and (err <= tol).all(), "%s: %d entries beyond the fp32 bound" % (
        what, int((~(err <= tol)).sum()))


def _bound(mag, dmax):
    """helpers.fp32_tol's bound of a sum whose absolute terms add up to mag."""
    return 2.0 * (dmax + 2) * EPS * mag + 1e-30


def check_fp64(P, script, staged, globs, outs):
    """Every output of every call of a run against the suite's fp64 references and bounds (helpers.fp32_tol, heads64,
    sage_oracle's max, test_gatv2's GATv2 bound); copied rows and maxima exactly."""
    import scipy.sparse as sp
    import sage_oracle as so
    from test_gatv2 import bounds as v2_bounds
    from test_multihead_attention import heads64
    E, dmax = P.edges()
    n = P.n
    vals = [lp.vals.astype(np.float64) for lp in P.lps]
    grows = np.concatenate([e[1] for e in E])
    gcols = np.concatenate([e[2] for e in E])
    for j, c in enumerate(script):
        op, f, K = c["op"], c.get("f"), c.get("K", 1)
        x, y = staged[j], outs[j]
        glob = {name: u.cpu().numpy() for name, u in globs[j].items()}
        per = [{name: u.cpu().numpy() for name, u in xr.items()} for xr in x]
        what = lambda r, name: "%s call %d (%s f=%s) rank %d %s" % (P.name, j, op, f, r, name)
        if op == "values":
            vals = [per[r]["vals"].astype(np.float64) if "vals" in per[r] else lp.vals.astype(np.float64)
                    for r, lp in enumerate(P.lps)]
            continue
        if op == "bwd":                                   # A^T gZ over every rank's entries, with its values now
            At = sp.csr_matrix((np.concatenate(vals), (gcols, grows)), shape=(n, n))
            G, tol = At @ glob["gZ"].astype(np.float64), fp32_tol(At, glob["gZ"], dmax)
        elif op == "bwd_heads":
            G, mag = heads64(gcols, grows, n, np.concatenate([per[r]["alpha"] for r in range(P.k)]), glob["gZ"], K)
            tol = _bound(mag, dmax)
        elif op == "bwd_max":
            G = sum(so.max_backward(e[2], per[r]["arg"], glob["gZ"][P.lps[r].owned], n) for r, e in enumerate(E))
            tol = _bound(sum(so.max_backward(e[2], per[r]["arg"], np.abs(glob["gZ"][P.lps[r].owned]), n)
                             for r, e in enumerate(E)), dmax)
        if op in ("bwd", "bwd_heads", "bwd_max"):
            for r, lp in enumerate(P.lps):
                _close(y[r]["G"], G[lp.owned], tol[lp.owned], what(r, "G"))
            continue
        if op == "bwd_v2":
            alpha = np.concatenate([per[r]["alpha"] for r in range(P.k)])
            ref = v2_bounds(grows, gcols, n, glob["xl"], glob["xr"], glob["att"], SLOPE, glob["gZ"], alpha)
            for r, lp in enumerate(P.lps):
                for name in ("dxl", "dxr"):
                    want, tol = ref[name]
                    _close(y[r][name], want[lp.owned], 2 * tol[lp.owned] + 64 * EPS * np.abs(want[lp.owned]),
                           what(r, name))
            want, tol = ref["datt"]
            datt = sum(y[r]["datt"].cpu().numpy().astype(np.float64) for r in range(P.k))
            assert (np.abs(datt - want) <= 2 * tol + 64 * EPS * np.abs(want) * P.k).all(), what(-1, "datt summed")
            continue
        for r, (lp, (rl, gr, gc)) in enumerate(zip(P.lps, E)):
            if op == "halo":
                assert np.array_equal(bits(y[r]["Xh"]), glob["X"][lp.halo].view(np.uint32)), what(r, "halo rows")
                continue
            if op in ("keep", "fwd_heads"):
                assert np.array_equal(bits(y[r]["Hh"]), glob["H"][lp.halo].view(np.uint32)), what(r, "halo rows")
            if op in ("fwd", "host", "keep"):
                Ar = sp.csr_matrix((vals[r], (rl, gc)), shape=(lp.m, n))
                z = Ar @ glob["H"].astype(np.float64)
                _close(y[r]["Z"], np.maximum(z, 0) if c["relu"] else z, fp32_tol(Ar, glob["H"], dmax), what(r, "Z"))
            elif op == "fwd_heads":
                z, mag = heads64(rl, gc, lp.m, per[r]["alpha"], glob["H"], K)
                _close(y[r]["Z"], z, _bound(mag, dmax), what(r, "Z"))
            elif op == "fwd_max":                           # exact: the first maximum of each row in local order
                Xl = np.concatenate([glob["H"][lp.owned], glob["H"][lp.halo]])
                z, arg = so.max_aggregate(lp.rowptr, lp.colidx, Xl)
                assert np.array_equal(bits(y[r]["Z"]), z.view(np.uint32)), what(r, "Z")
                assert np.array_equal(bits(y[r]["arg"]), arg), what(r, "arg")
            elif op == "fwd_v2":
                assert np.array_equal(bits(y[r]["Hh"]), glob["xl"][lp.halo].view(np.uint32)), what(r, "halo rows")
                ref = v2_bounds(gr, gc, n, glob["xl"], glob["xr"], glob["att"], SLOPE, np.zeros_like(glob["xl"]),
                                y[r]["alpha"].cpu().numpy())
                for name, u, rows in (("alpha", y[r]["alpha"], slice(None)), ("Z", y[r]["Z"], lp.owned)):
                    want, tol = ref[name]
                    _close(u, want[rows], tol[rows], what(r, name))


def assert_same_bits(base, outs, what):
    for j, (row_b, row_o) in enumerate(zip(base, outs)):
        for r, (b, o) in enumerate(zip(row_b, row_o)):
            for name, u in b.items():
                assert identical(o[name], u), "%s: call %d rank %d %s differs from lockstep" % (what, j, r, name)


_LOCKSTEP = {}


def lockstep(name):
    """(Part, script, staged inputs, lockstep outputs) of a partition, run once per session and checked against fp64."""
    if name not in _LOCKSTEP:
        P = part(name)
        script = make_script(SEED, P.fmax, P.widths)
        staged, globs = stage(P, SEED, script)
        outs, epochs = run(P, script, staged, "lockstep")
        assert epochs == [exchanges(script)] * P.k
        check_fp64(P, script, staged, globs, outs)
        _LOCKSTEP[name] = (P, script, staged, outs)
    return _LOCKSTEP[name]


# ---- CPU tests -------------------------------------------------------------------------------------------------------

def header_functions():
    src = open(HEADER).read()
    return re.findall(r"^\s*(?:const\s+)?\w+\**\s+\**(pgcn_\w+)\s*\(", src, flags=re.M)


def test_every_header_function_is_classified():
    names = header_functions()
    assert len(names) == len(set(names)) == 43
    assert set(names) == set(EXCHANGES) | LOCAL and not set(EXCHANGES) & LOCAL, \
        "unclassified: %s" % sorted(set(names) - set(EXCHANGES) - LOCAL)
    assert set(names) == set(cabi.SYMBOLS)


@pytest.mark.parametrize("name", ["karate", "rmat_k6", "degenerate"])
@pytest.mark.parametrize("host", [False, True])
def test_script_covers_every_exchange_at_both_parities(name, host):
    P = part(name)
    script = make_script(SEED, P.fmax, P.widths, host)
    assert script == make_script(SEED, P.fmax, P.widths, host)          # from the seed alone
    assert 30 <= len(script) <= 45
    par = parities(script)
    seen = {}
    for c, p in zip(script, par):
        if p is not None:
            seen.setdefault(c["op"], set()).add(p)
            if c["op"] == "host":
                seen.setdefault(("host", c["sync"]), set()).add(p)
            assert c["f"] % 4 == 0 and c["f"] <= P.fmax and c["f"] % c.get("K", 1) == 0
    ops = {op for op in EXCHANGES.values() if op is not None and (host or op != "host")}
    for op in ops:
        assert seen.get(op) == {0, 1}, "%s is not called at both epoch parities" % op
    if host:
        assert seen[("host", 0)] == seen[("host", 1)] == {0, 1}
    for v in variants():                                  # every call shape, at both parities
        v = dict(dict(overlap=1, relu=0), **v)
        hits = {p for c, p in zip(script, par) if all(c.get(key) == val for key, val in v.items() if key != "w")
                and ("w" not in v or c["w"] == (v["w"] or c["f"]))}
        assert hits == {0, 1}, v
    assert any(c["op"] == "values" and c["restore"] for c in script)
    assert sum(c["op"] == "values" and not c["restore"] for c in script) >= 2
    assert {c.get("overlap") for c in script if c["op"] in ("fwd", "bwd")} == {0, 1}
    fs = [c["f"] for c in script if "f" in c]
    assert len(set(fs)) >= 3 and sum(a != b for a, b in zip(fs, fs[1:])) >= len(fs) // 2
    keys = [c["key"] for c in script]
    assert len(set(keys)) == len(keys)
    if host:                                              # the host calls are inserted, the other calls keep their keys
        assert [c for c in script if c["op"] != "host"] == make_script(SEED, P.fmax, P.widths)


@pytest.mark.parametrize("name", ["karate", "degenerate"])
def test_inputs_are_fresh_on_every_call(name):
    """Calls j - 1 and j - 2 (the other slab parity and the same one) never hold call j's value at the same place of an
    input of the same name, over the whole arrays."""
    P = part(name)
    script = make_script(SEED, P.fmax, P.widths)
    drawn = [draw(P, SEED, c) for c in script]

    def values(d):
        glob, per = d
        out = {n: [u] for n, u in glob.items()}
        for p in per:
            for n, u in p.items():
                out.setdefault(n, []).append(u)
        return out
    for j in range(1, len(script)):
        now = values(drawn[j])
        assert now or script[j]["op"] == "values"
        for i in range(max(0, j - 2), j):
            for n, us in values(drawn[i]).items():
                for u in now.get(n, []):
                    for w in us:
                        if n == "arg" or not u.size or not w.size:      # entry indices: only their draws differ
                            continue
                        rows, cols = min(u.shape[0], w.shape[0]), min(u.reshape(len(u), -1).shape[1],
                                                                     w.reshape(len(w), -1).shape[1])
                        a = u.reshape(len(u), -1)[:rows, :cols]
                        b = w.reshape(len(w), -1)[:rows, :cols]
                        assert not (a == b).any(), (j, i, n)


def test_degenerate_partition_keeps_its_degeneracy():
    lps = part("degenerate").lps
    assert [lp.k for lp in lps] == [4] * 4
    assert lps[3].m == 0 and lps[3].h == 0 and lps[3].S == 0                  # rank 3 owns no rows
    assert lps[2].h == 0 and lps[2].S > 0                                    # reads no halo, others read it
    for a, b in ((0, 1), (1, 0)):                                            # ranks 0 and 1 exchange nothing
        assert lps[a].send_off[b + 1] == lps[a].send_off[b] and lps[a].recv_off[b + 1] == lps[a].recv_off[b]
    for r in (0, 1):
        assert lps[r].h > 0 and lps[r].recv_off[3] - lps[r].recv_off[2] == lps[r].h     # all halo rows from rank 2
        assert lps[2].send_off[r + 1] > lps[2].send_off[r]
    for lp in lps[:3]:
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert (deg == 0).any() and (deg == 1).any()
    for r, long_rows in ((0, 1900), (2, 990)):
        deg = np.diff(lps[r].rowptr.astype(np.int64))
        assert deg.max() >= long_rows and deg.max() > 512        # beyond the register kernel's default long-row split
    assert np.diff(lps[0].rowptr.astype(np.int64)).max() > 1024  # and the ring kernel's


def test_sleep_plan_keeps_every_rank_within_budget():
    for name in PARTS[::3]:
        P = part(name)
        script = make_script(SEED, P.fmax, P.widths)
        cyc, perm = sleep_plan(SEED, len(script), P.k)
        assert (cyc.sum(0) <= 40 * 10 ** 6).all()                          # ~22 ms at 1.8 GHz
        assert set(np.unique(cyc)) == set(SLEEPS)
        assert all(sorted(p) == list(range(P.k)) for p in perm)
        slowest = set(cyc.argmax(1)[cyc.max(1) > 0])
        assert len(slowest) > 1                                  # the slowest rank changes from call to call


# ---- GPU: enqueue orders ---------------------------------------------------------------------------------------------

def sleep_ms(cycles):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    torch.cuda._sleep(cycles)
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


@pytest.mark.gpu
@pytest.mark.parametrize("name", PARTS)
def test_lockstep_against_fp64(name):
    lockstep(name)


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["rank-major", "reverse", "skewed", "reused", "reused-reverse"])
@pytest.mark.parametrize("name", PARTS)
def test_enqueue_order_gives_the_lockstep_bits(name, order):
    P, script, staged, base = lockstep(name)
    if order in ("skewed", "reused"):
        cyc, _ = sleep_plan(SEED, len(script), P.k)
        ms = sleep_ms(10 ** 6)
        print("torch.cuda._sleep(10**6) took %.3f ms; the longest rank sleeps %.1f ms in all" % (
            ms, cyc.sum(0).max() / 1e6 * ms))
        assert cyc.sum(0).max() / 1e6 * ms < 50
    # the reused variants: under "reverse" the last rank is enqueued after every peer has already put its rows, so its
    # own puts are the only work still reading its operands when the call returns
    outs, epochs = run(P, script, staged, {"reused": "skewed", "reused-reverse": "reverse"}.get(order, order),
                       reuse=order.startswith("reused"))
    assert epochs == [exchanges(script)] * P.k
    assert_same_bits(base, outs, "%s %s" % (name, order))


# ---- GPU: autograd stacks --------------------------------------------------------------------------------------------

OPERATORS = ("PSpMM", "PSpMMRelu", "PSpMMWeighted", "PGATAttention", "PGATMultiHeadAttention", "PSpMMMax",
             "PGATv2Attention")
STACK_F = 32


def stack_leaves(n, m, nnz, owned, opname, f, seed):
    """The leaves of a two-layer stack on m rows (x, then the operator's parameters) and the upstream gradient; global
    draws (n rows) sliced by `owned`, the edge values of the nnz entries from `seed`."""
    rs = lambda i: np.random.RandomState([SEED, 500 + OPERATORS.index(opname), i])
    own = lambda a: torch.from_numpy(np.ascontiguousarray(a[owned])).to(dev())
    x = own(rs(0).uniform(-1, 1, (n, f)).astype(np.float32))
    g = own(rs(1).uniform(-1, 1, (n, f)).astype(np.float32))
    params = []
    if opname == "PSpMMWeighted":
        params = [torch.from_numpy(np.random.RandomState([seed, i]).uniform(0.5, 1.5, nnz).astype(np.float32)).to(dev())
                  for i in range(2)]
    elif opname in ("PGATAttention", "PGATMultiHeadAttention"):
        width = 2 if opname == "PGATAttention" else 8
        params = [torch.from_numpy((rs(2 + i).standard_normal((f, width)) / np.sqrt(f)).astype(np.float32)).to(dev())
                  for i in range(2)]
    elif opname == "PGATv2Attention":
        params = [torch.from_numpy((rs(2 + i).standard_normal((2, f // 2)) / np.sqrt(f)).astype(np.float32)).to(dev())
                  for i in range(2)]
    return [u.requires_grad_(True) for u in [x] + params], g


def layer(opname, plan, z, i, params):
    from pgcn_b200 import op as O
    if opname in ("PSpMM", "PSpMMRelu", "PSpMMMax"):
        return getattr(O, opname).apply(plan, z)
    if opname == "PSpMMWeighted":
        return O.PSpMMWeighted.apply(plan, params[i], z)
    if opname == "PGATAttention":
        s = z @ params[i]
        return O.PGATAttention.apply(plan, z, s[:, 0].contiguous(), s[:, 1].contiguous(), SLOPE)
    if opname == "PGATMultiHeadAttention":
        s = z @ params[i]
        return O.PGATMultiHeadAttention.apply(plan, z, s[:, :4].contiguous(), s[:, 4:].contiguous(), SLOPE)
    return O.PGATv2Attention.apply(plan, z, z * 0.5, params[i], SLOPE)


def stack(opname, plan, leaves, g):
    """Output and leaf gradients of the two-layer stack: the temporaries between the layers are Python's to free."""
    out = layer(opname, plan, layer(opname, plan, leaves[0], 0, leaves[1:]), 1, leaves[1:])
    (out * g).sum().backward()
    return [out.detach()] + [u.grad for u in leaves]


def warm_stack(P, opname, f, streams):
    """Every torch kernel of rank r's stack, launched once on its stream at rank r's shapes (a one-rank plan of the rows
    it owns), before anything waits on the device: a kernel's first launch synchronises with the device (see
    warm_torch_kernels), and cuBLAS picks its kernels by shape. The score exchange's padding and slicing as well."""
    for r, (lp, s) in enumerate(zip(P.lps, streams)):
        if lp.m == 0:
            continue
        A = P.A.tocsr()[lp.owned][:, lp.owned].tocoo()
        one = planmod.PgcnPlan(planmod.build_local_plan(A, np.zeros(lp.m, dtype=np.int64), 0, 1), P.fmax, device=dev())
        one.bind_values()
        with torch.cuda.stream(s):
            leaves, g = stack_leaves(lp.m, lp.m, one.lp.nnz(), np.arange(lp.m), opname, f, 0)
            stack(opname, one, leaves, g)
            for w, K in ((4, 1), (4, 4)):
                padded = torch.zeros((lp.m, w), device=dev())
                padded[:, slice(0, K) if K > 1 else 0] = torch.ones((lp.m, K) if K > 1 else (lp.m,), device=dev())
                halo = torch.empty((lp.h, w), device=dev())
                halo[:, slice(0, K) if K > 1 else 0].contiguous()
        torch.cuda.synchronize()
        one.close()


def run_stack(P, opname, f, order):
    """Output and leaf gradients of every rank's two-layer stack. lockstep: the forward of every rank, a device
    synchronisation, then the backward; rank-major / reverse: each rank's forward and backward back to back, rank by
    rank, with no host synchronisation until the end."""
    plans = linked_plans(P.lps, P.fmax, 1)
    for p in plans:
        for w in (f, 16, 4):                          # the layer width and the score rows of the backward
            p.prepare(w)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    warm_stack(P, opname, f, streams)
    ins = [stack_leaves(P.n, lp.m, lp.nnz(), lp.owned, opname, f, 600 + r) for r, lp in enumerate(P.lps)]
    res = [None] * P.k
    torch.cuda.synchronize()
    if order == "lockstep":
        outs = run_ranks(plans, lambda r: layer(opname, plans[r], layer(opname, plans[r], ins[r][0][0], 0,
                                                                        ins[r][0][1:]), 1, ins[r][0][1:]), streams)

        def backward(r):
            (outs[r] * ins[r][1]).sum().backward()
            res[r] = [outs[r].detach()] + [u.grad for u in ins[r][0]]
        run_ranks(plans, backward, streams)
    else:
        for r in (range(P.k) if order == "rank-major" else reversed(range(P.k))):
            with torch.cuda.stream(streams[r]):
                res[r] = stack(opname, plans[r], *ins[r])
        torch.cuda.synchronize()
    for p in plans:
        p.close()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["skewed", "degenerate"])
@pytest.mark.parametrize("opname", OPERATORS)
def test_autograd_stack_rank_major_gives_the_lockstep_bits(opname, name):
    P = part(name)
    base = run_stack(P, opname, STACK_F, "lockstep")
    for r in range(P.k):
        assert all(u is not None and bool(torch.isfinite(u).all()) for u in base[r]), "rank %d" % r
    for order in ("rank-major", "reverse"):
        got = run_stack(P, opname, STACK_F, order)
        for r in range(P.k):
            for i, (u, w) in enumerate(zip(got[r], base[r])):
                assert identical(u, w), "%s %s %s rank %d: output/gradient %d differs" % (name, opname, order, r, i)


# ---- GPU: CUDA graphs -------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["skewed", "degenerate"])
def test_graph_replays_back_to_back_rank_major(name):
    """The script's first 14 calls captured per rank, replayed three times in a row per rank, rank by rank, with new
    inputs copied in on the stream between replays: each replay has the bits of the eager run of its inputs."""
    P = part(name)
    script = make_script(SEED, P.fmax, P.widths)[:14]
    sets = [stage(P, SEED + 1 + i, script)[0] for i in range(3)]
    lib = cabi.load()
    plans = fresh(P, script)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    cap = [[{n: u.clone() for n, u in sets[0][j][r].items()} for j in range(len(script))] for r in range(P.k)]
    graphs, gouts = [], []
    torch.cuda.synchronize()
    for r, lp in enumerate(P.lps):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=streams[r]):
            ys = []
            for j, c in enumerate(script):
                ys.append({n: poisoned(s, n) for n, s in out_shapes(lp, c).items()})
                enqueue(lib, plans[r], c, cap[r][j], ys[-1])
        graphs.append(graph)
        gouts.append(ys)
    got = [[None] * 3 for _ in range(P.k)]
    for r in range(P.k):
        with torch.cuda.stream(streams[r]):
            for i in range(3):
                for j in range(len(script)):
                    for n, u in cap[r][j].items():
                        u.copy_(sets[i][j][r][n])
                graphs[r].replay()
                got[r][i] = [{n: u.clone() for n, u in ys.items()} for ys in gouts[r]]
    torch.cuda.synchronize()
    assert [p.get_option("epoch") for p in plans] == [3 * exchanges(script)] * P.k
    for p in plans:
        p.close()
    for i in range(3):
        eager, _ = run(P, script, sets[i], "lockstep")
        assert_same_bits(eager, [[got[r][i][j] for r in range(P.k)] for j in range(len(script))],
                         "%s replay %d" % (name, i))


# ---- GPU: processes and GPUs ------------------------------------------------------------------------------------------

def _run_own_rank(P, rank, plan, script, seed, sleep):
    """One rank's whole script on its own stream, without a host synchronisation except around the host-buffer forward
    (which enqueues on the plan's own stream: the caller's stream is drained first and the host waits for it)."""
    lib = cabi.load()
    lp = P.lps[rank]
    staged, _ = stage(P, seed, script, ranks=[rank])
    cyc, _ = sleep_plan(seed + rank, len(script), P.k)
    outs = []
    torch.cuda.synchronize()
    for j, c in enumerate(script):
        if sleep and cyc[j, rank]:
            torch.cuda._sleep(int(cyc[j, rank]))
        x = staged[j][rank]
        if c["op"] == "host":
            torch.cuda.current_stream().synchronize()
            plan.set_option("overlap", 1)
            H = x["H"].cpu().pin_memory()
            Z = torch.full((lp.m, c["f"]), float("nan")).pin_memory()
            if c["sync"]:
                cabi.check(lib.pgcn_forward_host(plan.handle, _p(H), _p(Z), c["f"]), plan.handle)
            else:
                cabi.check(lib.pgcn_forward_host_async(plan.handle, _p(H), _p(Z), c["f"]), plan.handle)
                cabi.check(lib.pgcn_forward_host_wait(plan.handle), plan.handle)
            outs.append({"Z": Z.numpy().copy()})
            continue
        y = {n: poisoned(s, n) for n, s in out_shapes(lp, c).items()}
        enqueue(lib, plan, c, x, y)
        outs.append(y)
    torch.cuda.synchronize()
    return [{n: (u if isinstance(u, np.ndarray) else u.cpu().numpy()) for n, u in o.items()} for o in outs]


def _ipc_worker(rank, k, port, seed):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=k)
    torch.cuda.set_device(0)
    P = Part("degenerate")
    script = make_script(seed, P.fmax, P.widths, host=True)
    plan = planmod.PgcnPlan(P.lps[rank], P.fmax, device=dev())
    assert plan.init_comm(transport="p2p", nccl_fallback=False) == "p2p"
    plan.bind_values()
    for ov in (0, 1):
        plan.set_option("overlap", ov)
        for f in sorted({c["f"] for c in script if "f" in c}):
            plan.prepare(f)
    dist.barrier()
    outs = _run_own_rank(P, rank, plan, script, seed, sleep=True)
    epoch = plan.get_option("epoch")
    dist.barrier()
    plan.close()
    dist.destroy_process_group()
    return outs, epoch


@pytest.mark.gpu
def test_processes_over_cuda_ipc_give_the_lockstep_bits():
    """The degenerate partition in one process per rank (4) on this GPU, over CUDA IPC: each runs the script with the
    host-buffer forward inserted, its own sleeps and no host synchronisation between the other calls."""
    P, script, _, base = lockstep("degenerate")
    hscript = make_script(SEED, P.fmax, P.widths, host=True)
    res = spawn_ranks(_ipc_worker, P.k, (29871, SEED))
    E, dmax = P.edges()
    for r in range(P.k):
        outs, epoch = res[r]
        assert epoch == exchanges(hscript)
        keyed = {c["key"]: o for c, o in zip(hscript, outs)}
        for j, c in enumerate(script):
            for n, u in base[j][r].items():
                assert np.array_equal(keyed[c["key"]][n].view(np.uint32), u.cpu().numpy().view(np.uint32)), \
                    "rank %d call %d (%s) %s differs from the in-process lockstep run" % (r, j, c["op"], n)
        import scipy.sparse as sp
        rl, gr, gc = E[r]
        lp = P.lps[r]
        vals = lp.vals.astype(np.float64)
        for c, o in zip(hscript, outs):
            if c["op"] == "values":
                per = draw(P, SEED, c)[1][r]
                vals = per["vals"].astype(np.float64) if "vals" in per else lp.vals.astype(np.float64)
            if c["op"] == "host":
                H = draw(P, SEED, c)[0]["H"]
                Ar = sp.csr_matrix((vals, (rl, gc)), shape=(lp.m, P.n))
                _close(torch.from_numpy(o["Z"]), Ar @ H.astype(np.float64), fp32_tol(Ar, H, dmax),
                       "rank %d host forward" % r)


def _gpu_worker(rank, k, port, transport, seed):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["CUDA_VISIBLE_DEVICES"] = str(rank)           # before CUDA starts: this rank's GPU is cuda:0
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=dev())
    P = Part("skewed", k=2)
    script = make_script(seed, P.fmax, P.widths)
    plan = planmod.PgcnPlan(P.lps[rank], P.fmax, device=dev())
    used = plan.init_comm(transport=transport)
    plan.bind_values()
    outs = _run_own_rank(P, rank, plan, script, seed, sleep=False)
    dist.barrier()
    plan.close()
    dist.destroy_process_group()
    return used, outs


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_gpus_nccl_and_peer_transport_give_the_same_bits():
    """The skewed graph on two ranks, one GPU each: the whole script over NCCL and over the peer transport."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_gpu_worker, 2, (29881, "nccl", SEED))
    b = spawn_ranks(_gpu_worker, 2, (29882, "p2p", SEED))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        for j, (u, w) in enumerate(zip(a[r][1], b[r][1])):
            for n in u:
                assert np.array_equal(u[n].view(np.uint32), w[n].view(np.uint32)), "rank %d call %d %s" % (r, j, n)
