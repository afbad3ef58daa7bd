"""PSpMM — the operator boundary of the hot path (GPU/PGCN.py:121-134), H100-native.

    PSpMM.apply(A, H)     A = PgcnPlan (the opaque plan handle standing in for the sparse tensor)
                          H = fp32 CUDA tensor

forward  = pack boundary rows -> all-to-all-v -> Z = A_local * [H_own ; H_halo]     (:123-127)
backward = G = A_local^T * gZ, halo-row partials sent back to their owners and SUMMED (:129-134;
           the reference ASSIGNS the received rows, quirk Q3 of SURVEY.md §8a — this op implements
           the intended semantics and the tests pin the difference).

Layouts (plan.layout):
  "local"  : H is [m, f] (owned rows only), Z is [m, f] — no n-sized tensors anywhere.
  "global" : H is [n, f] like the reference (rows it does not own are ignored = the reference's
             precondition Q0 that they are zero), Z is [n, f] with non-owned rows exactly 0.

All arithmetic happens in libpgcn_b200.so on the current CUDA stream; there is no CPU path.
Every operator takes its inputs through _own / _own_scores, returns its outputs through _to_layout and makes each C
call through _call, so an operator is its validation and its sequence of C calls.
"""
import ctypes as C

import torch

from . import cabi


def _stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def _ptr(x):
    return None if x is None else x.data_ptr()


def _call(plan, dev, name, *args, exchange=None):
    """lib.<name>(plan, *args, stream) on `dev`'s current stream, its status checked. exchange=False / True: the call ran
    the forward / backward exchange, which plan.stats counts (nothing on one rank)."""
    with torch.cuda.device(dev):
        cabi.check(getattr(cabi.load(), name)(plan.handle, *args, _stream_ptr()), plan.handle)
    if exchange is not None:
        plan.count_exchange(backward=exchange)


def _check_f32(x, what):
    if not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the PGCN H100 path has no CPU fallback" % what)
    if x.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (what, x.dtype))


def _check_feat(plan, H, rows, what):
    _check_f32(H, what)
    if H.dim() != 2 or H.shape[0] != rows:
        raise ValueError("%s must be [%d, f], got %s" % (what, rows, tuple(H.shape)))
    if H.shape[1] > plan.f_max:
        raise ValueError("f=%d exceeds the plan's f_max=%d" % (H.shape[1], plan.f_max))
    return H.contiguous()


def _rows(plan):
    return plan.n if plan.layout == "global" else plan.m


def _owned(plan, x):
    return x.index_select(0, plan.owned_index()) if plan.layout == "global" else x.contiguous()


def _own(plan, x, what):
    """x, a [rows, f] feature tensor in the plan's layout, checked: its owned rows [m, f], contiguous."""
    return _owned(plan, _check_feat(plan, x, _rows(plan), what))


def _own_scores(plan, x, what, heads=None):
    """x, per-row scores [rows] (heads None) or [rows, heads] in the plan's layout, checked: its owned rows, contiguous."""
    shape = (_rows(plan),) if heads is None else (_rows(plan), heads)
    _check_f32(x, what)
    if tuple(x.shape) != shape:
        raise ValueError("%s must be [%s], got %s" % (what, ", ".join(map(str, shape)), tuple(x.shape)))
    return _owned(plan, x.detach())


def _to_layout(plan, x_own):
    """x_own [m, ...] in the plan's layout: itself in "local", [n, ...] with zero rows where other ranks own them in
    "global"."""
    if plan.layout != "global":
        return x_own
    out = torch.zeros((plan.n,) + tuple(x_own.shape[1:]), dtype=torch.float32, device=x_own.device)
    out.index_copy_(0, plan.owned_index(), x_own)
    return out


def _require_bound(plan, what):
    if not plan._bound:
        raise RuntimeError("%s: call PgcnPlan.bind_values() once (set-up, before any CUDA-graph capture)" % what)


def _aggregate(plan, H_own, keep_halo=False):
    """(Z, H_halo): Z [m, f] = A [H_own; H_halo] with the plan's resident values, exchange included. keep_halo: H_halo is
    the [h, f] halo rows the exchange brought (pgcn_forward_keep_halo) where there are any; otherwise None."""
    lp, f, dev = plan.lp, H_own.shape[1], H_own.device
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    if keep_halo and lp.k > 1 and lp.h > 0:
        H_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
        _call(plan, dev, "pgcn_forward_keep_halo", H_own.data_ptr(), Z.data_ptr(), H_halo.data_ptr(), f, exchange=False)
        return Z, H_halo
    _call(plan, dev, "pgcn_forward", H_own.data_ptr(), Z.data_ptr(), f, exchange=False)
    return Z, None


def _aggregate_t(plan, gZ_own):
    """G [m, f] = A^T gZ_own with the plan's resident values, the halo partials summed at their owners."""
    f = gZ_own.shape[1]
    G = torch.empty((plan.lp.m, f), dtype=torch.float32, device=gZ_own.device)
    _call(plan, gZ_own.device, "pgcn_backward", gZ_own.data_ptr(), G.data_ptr(), f, exchange=True)
    return G


def _score_halo(plan, s_own):
    """Per-row scores of the halo columns from their owners: s_own [m] or [m, K] gives [h] or [h, K]. pgcn_halo_rows
    carries rows padded to a multiple of 4 floats, the width the peer transport takes; [m] travels as column 0 of 4."""
    lp, dev = plan.lp, s_own.device
    if lp.k == 1:
        return torch.empty((lp.h,) + tuple(s_own.shape[1:]), dtype=torch.float32, device=dev)
    K = s_own.shape[1] if s_own.dim() == 2 else 1
    col = slice(0, K) if s_own.dim() == 2 else 0
    w = (K + 3) // 4 * 4
    padded = torch.zeros((lp.m, w), dtype=torch.float32, device=dev)
    padded[:, col] = s_own
    halo = torch.empty((lp.h, w), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", padded.data_ptr(), halo.data_ptr(), w, exchange=False)
    return halo[:, col].contiguous()


def aggregate_forward(plan, H_own, relu=False):
    """Z_own = (A * H)[owned rows]; H_own, Z_own are [m, f]. relu=True: Z_own = max(0, .), clamped inside the store of
    the launch that writes each row last (plan option "relu")."""
    H_own = _check_feat(plan, H_own, plan.m, "H")
    plan.use_values(None)                 # PSpMM / PSpMMRelu aggregate with the plan's own values
    if relu:
        plan.set_option("relu", 1)
    try:
        return _aggregate(plan, H_own)[0]
    finally:
        if relu:
            plan.set_option("relu", 0)


def aggregate_backward(plan, gZ_own):
    """G_own = (A^T * gZ)[owned rows] with every peer's contribution added; [m, f]."""
    gZ_own = _check_feat(plan, gZ_own, plan.m, "grad_output")
    plan.use_values(None)
    return _aggregate_t(plan, gZ_own)


class PSpMM(torch.autograd.Function):
    """Same call shape as the reference operator: PSpMM.apply(A, H) (GPU/PGCN.py:145)."""

    @staticmethod
    def forward(ctx, A, H):
        ctx.plan = A
        return _to_layout(A, aggregate_forward(A, _own(A, H, "H")))

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        return None, _to_layout(A, aggregate_backward(A, _own(A, grad_output, "grad_output")))


class PSpMMRelu(torch.autograd.Function):
    """relu(A * X) with the clamp fused into the aggregation's output store (SURVEY.md §8f rank 1). Feeding it
    X = linear(H) gives the reference layer relu(linear(PSpMM(A, H))) of GPU/PGCN.py:144-148 up to fp32 association
    ((A H) W^T == A (H W^T)); the dense step then also runs before the aggregation instead of after it.
    Backward: relu's mask comes from the saved output (out > 0), then the regular PSpMM backward."""

    @staticmethod
    def forward(ctx, A, X):
        ctx.plan = A
        out = aggregate_forward(A, X, relu=True)
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (out,) = ctx.saved_tensors
        return None, aggregate_backward(ctx.plan, grad_output * (out > 0))


class PSpMMWeighted(torch.autograd.Function):
    """Z = A(vals) * H with the edge values given per call, like torch.sparse.mm(A, H) on a sparse A whose values
    require grad (GPU/PGCN.py:127 with learned edge weights, an edge mask or attention scores).

        PSpMMWeighted.apply(A, vals, H)     vals = fp32 CUDA [nnz] in A's local forward CSR order (A.edge_index())

    Backward returns (None, dvals, dH): dH = A(vals)^T gZ with the exchange (pgcn_backward, vals resident), and, when
    vals needs grad, dvals[e] = <gZ[row(e)], [H_own; H_halo][col(e)]> from the SDDMM kernel (pgcn_sddmm); on k > 1 the
    forward keeps the halo rows it received for it (pgcn_forward_keep_halo). Several layers may share one plan with
    different values: each launch first makes its own values resident (PgcnPlan.use_values). Layouts as PSpMM.

    The plan must be bound first (PgcnPlan.bind_values, synchronous set-up). A rewrite is skipped when `vals` is the
    tensor set last and its version counter has not moved: in-place updates through autograd-visible ops (optimizer
    steps, `with torch.no_grad(): w.mul_(...)`) are seen, writes through `w.data` or raw pointers are not — call
    A.set_values(w) after those."""

    @staticmethod
    def forward(ctx, A, vals, H):
        from .plan import check_values
        check_values(A, vals)
        ctx.plan = A
        H_own = _own(A, H, "H")
        want_dvals = ctx.needs_input_grad[1]
        A.use_values(vals)
        Z, H_halo = _aggregate(A, H_own, keep_halo=want_dvals)
        ctx.save_for_backward(vals, H_own if want_dvals else None, H_halo)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        vals, H_own, H_halo = ctx.saved_tensors
        g = _own(A, grad_output, "grad_output")
        dvals = dH = None
        if ctx.needs_input_grad[2]:
            A.use_values(vals)
            dH = _to_layout(A, _aggregate_t(A, g))
        if ctx.needs_input_grad[1]:
            dvals = torch.empty((A.lp.nnz(),), dtype=torch.float32, device=g.device)
            _call(A, g.device, "pgcn_sddmm", g.data_ptr(), H_own.data_ptr(), _ptr(H_halo), dvals.data_ptr(), g.shape[1])
        return None, dvals, dH


# ---- edge dropout (libpgcn_dropout.so) -------------------------------------------------------------------------------

def dropout_constants(p):
    """(threshold, scale) of drop probability p in [0, 1): threshold = floor(p 2^32) in fp64, an entry is kept when its
    Philox word is >= threshold; scale = float32(1 / (1 - p)), the fp64 quotient rounded once."""
    import math
    import numpy as np
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError("dropout probability p=%r must lie in [0, 1)" % p)
    return int(math.floor(p * 4294967296.0)), float(np.float32(1.0 / (1.0 - p)))


class EdgeDropout:
    """Dropout on per-edge arrays in forward-CSR order whose mask is a pure function of the global edge (include/
    pgcn_dropout.h): entry (global row gi, global column gj), head h, keep iff word h & 3 of Philox4x32-10(counter =
    (gi, gj, c, h >> 2), key) >= floor(p 2^32); kept values are scaled by float32(1 / (1 - p)), dropped ones multiplied
    by 0. Any partition of a graph, and one GPU or k, draw the same mask.

        EdgeDropout(p, key, device)     p in [0, 1), key a 64-bit integer

    `state` is the device int64 [key, c]. Every use on an operator (edge_dropout, PGATAttention,
    PGATMultiHeadAttention) adds 1 to c on the device, in stream order, and uses the new value, so the first use draws
    with c = 1 and a captured CUDA graph draws a new mask on every replay; the backward reuses its own forward's c. With
    p == 0 the operators make no dropout launch at all."""

    def __init__(self, p, key, device=None):
        self.p = float(p)
        self.threshold, self.scale = dropout_constants(self.p)
        key = int(key)
        if not 0 <= key < 2 ** 64:
            raise ValueError("key=%d must lie in [0, 2^64)" % key)
        self.state = torch.tensor([key - 2 ** 64 if key >= 2 ** 63 else key, 0], dtype=torch.int64,
                                  device=torch.device("cuda", torch.cuda.current_device()) if device is None else device)

    def draw(self):
        """Advance the call counter (on the device, current stream) and return a snapshot [key, c] of the new state."""
        self.state[1:].add_(1)
        return self.state.clone()


def _active(drop):
    return drop if drop is not None and drop.p > 0 else None


def _mask(pairs, snap, drop, x, y):
    """y = the mask of `drop` at the state `snap` applied to x ([nnz] or [nnz, K], contiguous); y may be x."""
    K = x.shape[1] if x.dim() == 2 else 1
    with torch.cuda.device(x.device):
        cabi.check_dropout(cabi.load_dropout().pgcn_edge_dropout(pairs.data_ptr(), pairs.shape[0], K, drop.threshold,
                                                                 drop.scale, snap.data_ptr(), x.data_ptr(),
                                                                 y.data_ptr(), _stream_ptr()))
    return y


def _dropout_pairs(A, drop):
    """A.edge_pairs() when `drop` is active, else None. Operators call it before anything else, so that a capture that
    needs the pairs before they exist is refused before it enqueues any work."""
    if drop is None:
        return None
    if drop.state.device != A.device:
        raise ValueError("the EdgeDropout state lives on %s, the plan on %s" % (drop.state.device, A.device))
    return A.edge_pairs()


class EdgeDropoutFunction(torch.autograd.Function):
    """y = mask(x) for x [nnz] or [nnz, K] (K in 1, 2, 4, 8) in A's forward-CSR order; the gradient is the same map
    with the same counter. Use edge_dropout()."""

    @staticmethod
    def forward(ctx, A, x, drop):
        pairs = _dropout_pairs(A, drop)
        snap = drop.draw()
        y = _mask(pairs, snap, drop, x, torch.empty_like(x))
        ctx.plan, ctx.drop = A, drop
        ctx.save_for_backward(snap)
        return y

    @staticmethod
    def backward(ctx, grad_output):
        (snap,) = ctx.saved_tensors
        g = grad_output.contiguous()
        return None, _mask(ctx.plan.edge_pairs(), snap, ctx.drop, g, torch.empty_like(g)), None


def edge_dropout(A, x, drop):
    """Edge dropout of a per-edge array: x is fp32 CUDA [nnz] or [nnz, K] (K in 1, 2, 4, 8) in A's local forward-CSR
    order (A.edge_index()), drop an EdgeDropout or None. Differentiable. With drop None or p == 0 it returns x itself.
    DropEdge-style value dropout: PSpMMWeighted.apply(A, edge_dropout(A, vals, drop), H)."""
    if _active(drop) is None:
        return x
    _dropout_pairs(A, drop)
    _check_f32(x, "x")
    nnz = A.lp.nnz()
    if x.dim() not in (1, 2) or x.shape[0] != nnz or (x.dim() == 2 and x.shape[1] not in HEADS):
        raise ValueError("x must be [%d] or [%d, K] with K in 1, 2, 4, 8, got %s" % (nnz, nnz, tuple(x.shape)))
    if x.device != A.device:
        raise ValueError("x lives on %s, the plan on %s" % (x.device, A.device))
    return EdgeDropoutFunction.apply(A, x.contiguous(), drop)


HEADS = (1, 2, 4, 8)


class PGATAttention(torch.autograd.Function):
    """Single-head sparse graph attention over the plan's stored pattern (GPU/PGAT.py:139-148 without the dense n x n
    score matrix):

        PGATAttention.apply(A, Z, el, er, negative_slope, dropout=None)
        s_e = LeakyReLU(el[row(e)] + er[col(e)]),  alpha = softmax of s over each row's stored entries,  out = A(alpha) Z

    Z is [rows, f], el and er are [rows] fp32 CUDA tensors (rows = m in the "local" layout, n in the "global" one, whose
    non-owned rows are ignored and come back zero), out is [rows, f]. er of the halo columns comes from their owners
    (pgcn_halo_rows, padded to rows of 4 floats so that the peer transport carries it). Forward: the edge softmax kernel
    writes alpha, which becomes the resident values of A for pgcn_forward_keep_halo(Z). Backward: dZ = A(alpha)^T gOut
    with the exchange; dalpha = SDDMM(gOut, [Z_own; Z_halo]); the softmax backward kernel gives dpre and d_el; and
    d_er = A(dpre)^T 1, the column sums of dpre with the halo partials summed at their owners (pgcn_backward on an
    m x 4 matrix of ones). Everything is deterministic. Gradients to W and a flow through torch, since el and er are
    computed outside. The plan must be bound (PgcnPlan.bind_values); a later PSpMM on it restores the creation values.

    dropout (an EdgeDropout with p > 0) applies attention dropout between the softmax and the aggregation: alpha_d =
    mask(alpha) aggregates Z, and the backward takes dZ with alpha_d, dalpha = mask(dalpha_d) and the softmax backward
    with the undropped alpha. alpha_d is kept for the backward (4 B per entry). None or p == 0: no dropout launch."""

    @staticmethod
    def forward(ctx, A, Z, el, er, negative_slope=0.2, dropout=None):
        drop = _active(dropout)
        pairs = _dropout_pairs(A, drop)
        Z_own = _own(A, Z, "Z")
        el_own = _own_scores(A, el, "el")
        er_own = _own_scores(A, er, "er")
        _require_bound(A, "PGATAttention sets the plan's edge values")
        snap = drop.draw() if drop else None
        lp, dev, slope = A.lp, Z_own.device, float(negative_slope)
        er_halo = _score_halo(A, er_own)
        alpha = torch.empty((lp.nnz(),), dtype=torch.float32, device=dev)
        _call(A, dev, "pgcn_edge_softmax", el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(), slope,
              alpha.data_ptr())
        alpha_d = _mask(pairs, snap, drop, alpha, torch.empty_like(alpha)) if drop else alpha
        A.use_values(alpha_d)
        out, Z_halo = _aggregate(A, Z_own, keep_halo=True)
        ctx.plan, ctx.slope, ctx.drop = A, slope, drop
        ctx.save_for_backward(alpha, Z_own, Z_halo, el_own, er_own, er_halo, alpha_d if drop else None, snap)
        return _to_layout(A, out)

    @staticmethod
    def backward(ctx, grad_output):
        A, slope, drop = ctx.plan, ctx.slope, ctx.drop
        alpha, Z_own, Z_halo, el_own, er_own, er_halo, alpha_d, snap = ctx.saved_tensors
        g = _own(A, grad_output, "grad_output")
        lp, f, dev = A.lp, g.shape[1], g.device
        dZ = d_el = d_er = None
        if ctx.needs_input_grad[1]:
            A.use_values(alpha_d if drop else alpha)
            dZ = _to_layout(A, _aggregate_t(A, g))
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            dalpha = torch.empty_like(alpha)
            _call(A, dev, "pgcn_sddmm", g.data_ptr(), Z_own.data_ptr(), _ptr(Z_halo), dalpha.data_ptr(), f)
            if drop:
                _mask(A.edge_pairs(), snap, drop, dalpha, dalpha)
            dpre = torch.empty_like(alpha)
            gel = torch.empty((lp.m,), dtype=torch.float32, device=dev)
            _call(A, dev, "pgcn_edge_softmax_backward", el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(),
                  alpha.data_ptr(), dalpha.data_ptr(), slope, dpre.data_ptr(), gel.data_ptr())
            d_el = _to_layout(A, gel) if ctx.needs_input_grad[2] else None
            if ctx.needs_input_grad[3]:
                A.use_values(dpre)
                ones = torch.ones((lp.m, 4), dtype=torch.float32, device=dev)
                d_er = _to_layout(A, _aggregate_t(A, ones)[:, 0].contiguous())
        return None, dZ, d_el, d_er, None, None


class PGATMultiHeadAttention(torch.autograd.Function):
    """Multi-head sparse graph attention over the plan's stored pattern: K = el.shape[1] heads (1, 2, 4 or 8) of width
    d = f / K, concatenated.

        PGATMultiHeadAttention.apply(A, Z, el, er, negative_slope, dropout=None)
        s_eh = LeakyReLU(el[row(e), h] + er[col(e), h]),  alpha_.h = softmax of s_.h over each row's stored entries,
        out[:, h d:(h+1) d] = A(alpha[:, h]) Z[:, h d:(h+1) d]

    Z is [rows, f], el and er are [rows, K] fp32 CUDA tensors, out is [rows, f] (rows = m in the "local" layout, n in the
    "global" one, as PGATAttention). One exchange per layer carries the f-wide Z for every head, and er of the halo
    columns travels once for all heads (pgcn_halo_rows, rows padded to a multiple of 4 floats). The kernels take alpha
    ([nnz, K]) as an argument, so the plan's resident values are never rewritten: a PSpMM on the same plan needs no
    restore. Backward: dZ = A(alpha)^T gOut per head (pgcn_backward_heads), dalpha from pgcn_sddmm_heads, dpre and d_el
    from the softmax backward, d_er[:, h] = A(dpre[:, h])^T 1 (pgcn_backward_heads on an m x 4K matrix of ones, column
    4h), so the plan's f_max must be at least max(f, 4K). Deterministic. The exchange is the unsplit one (no per-source
    overlap). The plan must be bound (PgcnPlan.bind_values).

    dropout (an EdgeDropout with p > 0): attention dropout on every head, as PGATAttention; alpha_d = mask(alpha)
    ([nnz, K]) is the alpha argument of the aggregation and is kept for the backward (4K B per entry)."""

    @staticmethod
    def forward(ctx, A, Z, el, er, negative_slope=0.2, dropout=None):
        drop = _active(dropout)
        pairs = _dropout_pairs(A, drop)
        if el.dim() != 2:
            raise ValueError("el must be [%d, heads], got %s" % (_rows(A), tuple(el.shape)))
        K = el.shape[1]
        if K not in HEADS:
            raise ValueError("heads=%d: the multi-head kernels take 1, 2, 4 or 8 heads" % K)
        Z_own = _own(A, Z, "Z")
        f = Z_own.shape[1]
        if f % K:
            raise ValueError("f=%d is not a multiple of heads=%d" % (f, K))
        if A.f_max < 4 * K:
            raise ValueError("heads=%d: the backward aggregates rows of 4 x heads = %d floats, the plan's f_max is %d"
                             % (K, 4 * K, A.f_max))
        el_own = _own_scores(A, el, "el", K)
        er_own = _own_scores(A, er, "er", K)
        _require_bound(A, "PGATMultiHeadAttention reads the plan's value maps")
        snap = drop.draw() if drop else None
        lp, dev, slope = A.lp, Z_own.device, float(negative_slope)
        er_halo = _score_halo(A, er_own)
        alpha = torch.empty((lp.nnz(), K), dtype=torch.float32, device=dev)
        _call(A, dev, "pgcn_edge_softmax_heads", K, el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(), slope,
              alpha.data_ptr())
        alpha_d = _mask(pairs, snap, drop, alpha, torch.empty_like(alpha)) if drop else alpha
        out = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        Z_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev) if lp.k > 1 and lp.h > 0 else None
        _call(A, dev, "pgcn_forward_heads", K, alpha_d.data_ptr(), Z_own.data_ptr(), out.data_ptr(), _ptr(Z_halo), f,
              exchange=False)
        ctx.plan, ctx.slope, ctx.heads, ctx.drop = A, slope, K, drop
        ctx.save_for_backward(alpha, Z_own, Z_halo, el_own, er_own, er_halo, alpha_d if drop else None, snap)
        return _to_layout(A, out)

    @staticmethod
    def backward(ctx, grad_output):
        A, slope, K, drop = ctx.plan, ctx.slope, ctx.heads, ctx.drop
        alpha, Z_own, Z_halo, el_own, er_own, er_halo, alpha_d, snap = ctx.saved_tensors
        g = _own(A, grad_output, "grad_output")
        lp, f, dev = A.lp, g.shape[1], g.device
        dZ = d_el = d_er = None
        if ctx.needs_input_grad[1]:
            G = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            _call(A, dev, "pgcn_backward_heads", K, (alpha_d if drop else alpha).data_ptr(), g.data_ptr(), G.data_ptr(),
                  f, exchange=True)
            dZ = _to_layout(A, G)
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            dalpha = torch.empty_like(alpha)
            _call(A, dev, "pgcn_sddmm_heads", K, g.data_ptr(), Z_own.data_ptr(), _ptr(Z_halo), dalpha.data_ptr(), f)
            if drop:
                _mask(A.edge_pairs(), snap, drop, dalpha, dalpha)
            dpre = torch.empty_like(alpha)
            gel = torch.empty((lp.m, K), dtype=torch.float32, device=dev)
            _call(A, dev, "pgcn_edge_softmax_backward_heads", K, el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(),
                  alpha.data_ptr(), dalpha.data_ptr(), slope, dpre.data_ptr(), gel.data_ptr())
            d_el = _to_layout(A, gel) if ctx.needs_input_grad[2] else None
            if ctx.needs_input_grad[3]:
                ones = torch.ones((lp.m, 4 * K), dtype=torch.float32, device=dev)
                D = torch.empty((lp.m, 4 * K), dtype=torch.float32, device=dev)
                _call(A, dev, "pgcn_backward_heads", K, dpre.data_ptr(), ones.data_ptr(), D.data_ptr(), 4 * K,
                      exchange=True)
                d_er = _to_layout(A, D[:, 0::4].contiguous())
        return None, dZ, d_el, d_er, None, None


class PGATv2Attention(torch.autograd.Function):
    """GATv2 attention (dynamic attention, Brody et al.) over the plan's stored pattern: K = att.shape[0] heads (1, 2, 4
    or 8) of width d = f / K, concatenated.

        PGATv2Attention.apply(A, XL, XR, att, negative_slope=0.2)
        s_eh = sum_c att[h, c] * LeakyReLU(XL[col(e), h d + c] + XR[row(e), h d + c]),
        alpha_.h = softmax of s_.h over each row's stored entries,  out[:, h d:(h+1) d] = A(alpha[:, h]) XL[:, h d:(h+1) d]

    XL and XR are [rows, f] and att is [K, d], fp32 CUDA tensors; out is [rows, f] (rows = m in the "local" layout, n in
    the "global" one, as PGATMultiHeadAttention). This is PyG GATv2Conv(share_weights=False, concat=True, bias=False,
    add_self_loops=False) on XL = lin_l(x), XR = lin_r(x); passing one tensor as XL and XR is share_weights=True, and
    its gradient is the sum of both. One exchange per layer carries XL's halo rows (pgcn_forward_gatv2), which the
    backward reuses. Gradients for XL, XR and att come from pgcn_backward_gatv2. The plan's resident values are never
    read or written. Deterministic. The plan must be bound (PgcnPlan.bind_values)."""

    @staticmethod
    def forward(ctx, A, XL, XR, att, negative_slope=0.2):
        if att.dim() != 2:
            raise ValueError("att must be [heads, f / heads], got %s" % (tuple(att.shape),))
        K = att.shape[0]
        if K not in HEADS:
            raise ValueError("heads=%d: the GATv2 kernels take 1, 2, 4 or 8 heads" % K)
        XL_own = _own(A, XL, "XL")
        XR_own = _own(A, XR, "XR")
        f = XL_own.shape[1]
        if XR_own.shape[1] != f:
            raise ValueError("XL and XR must have the same width, got %d and %d" % (f, XR_own.shape[1]))
        if f % K:
            raise ValueError("f=%d is not a multiple of heads=%d" % (f, K))
        if tuple(att.shape) != (K, f // K):
            raise ValueError("att must be [%d, %d], got %s" % (K, f // K, tuple(att.shape)))
        if not att.is_cuda or att.dtype != torch.float32:
            raise TypeError("att must be a float32 CUDA tensor")
        att_c = att.detach().contiguous()
        _require_bound(A, "PGATv2Attention reads the plan's value maps")
        lp, dev, slope = A.lp, XL_own.device, float(negative_slope)
        alpha = torch.empty((lp.nnz(), K), dtype=torch.float32, device=dev)
        out = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        XL_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev) if lp.k > 1 and lp.h > 0 else None
        _call(A, dev, "pgcn_forward_gatv2", K, XL_own.data_ptr(), XR_own.data_ptr(), att_c.data_ptr(), slope,
              alpha.data_ptr(), out.data_ptr(), _ptr(XL_halo), f, exchange=False)
        ctx.plan, ctx.slope, ctx.heads = A, slope, K
        ctx.save_for_backward(alpha, XL_own, XL_halo, XR_own, att_c)
        return _to_layout(A, out)

    @staticmethod
    def backward(ctx, grad_output):
        A, slope, K = ctx.plan, ctx.slope, ctx.heads
        alpha, XL_own, XL_halo, XR_own, att = ctx.saved_tensors
        g = _own(A, grad_output, "grad_output")
        lp, f, dev = A.lp, g.shape[1], g.device
        work = torch.empty_like(alpha)
        dxl = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        dxr = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        datt = torch.empty_like(att)
        _call(A, dev, "pgcn_backward_gatv2", K, alpha.data_ptr(), g.data_ptr(), XL_own.data_ptr(), _ptr(XL_halo),
              XR_own.data_ptr(), att.data_ptr(), slope, work.data_ptr(), dxl.data_ptr(), dxr.data_ptr(),
              datt.data_ptr(), f, exchange=True)
        return None, _to_layout(A, dxl), _to_layout(A, dxr), datt, None


# ---- max aggregation -------------------------------------------------------------------------------------------------

def aggregate_max(plan, H_own):
    """(Z_own, arg): the element-wise maximum over each owned row's stored entries of [H_own ; H_halo] (pgcn_forward_max).
    Z_own is [m, f] fp32, arg [m, f] int32: the winning entry, the first in forward CSR order (lp.colidx's order) with
    the largest value, NaN above every number; lp.colidx[arg] is its local column. Rows without an entry give 0 / -1."""
    H_own = _check_feat(plan, H_own, plan.m, "H")
    _require_bound(plan, "aggregate_max walks the transposed records through the plan's value maps")
    f = H_own.shape[1]
    Z = torch.empty((plan.m, f), dtype=torch.float32, device=H_own.device)
    arg = torch.empty((plan.m, f), dtype=torch.int32, device=H_own.device)
    _call(plan, H_own.device, "pgcn_forward_max", H_own.data_ptr(), Z.data_ptr(), arg.data_ptr(), f, exchange=False)
    return Z, arg


def aggregate_max_backward(plan, arg, gZ_own):
    """G_own [m, f]: gZ routed to the winning entries named by `arg` (aggregate_max's), summed per column on its owner
    (pgcn_backward_max)."""
    gZ_own = _check_feat(plan, gZ_own, plan.m, "grad_output")
    _require_bound(plan, "aggregate_max_backward walks the transposed records through the plan's value maps")
    f = gZ_own.shape[1]
    if arg.dtype != torch.int32 or arg.device != gZ_own.device or tuple(arg.shape) != (plan.m, f):
        raise ValueError("arg must be int32 [%d, %d] on %s, got %s %s on %s"
                         % (plan.m, f, gZ_own.device, arg.dtype, tuple(arg.shape), arg.device))
    arg = arg.contiguous()
    G = torch.empty((plan.m, f), dtype=torch.float32, device=gZ_own.device)
    _call(plan, gZ_own.device, "pgcn_backward_max", arg.data_ptr(), gZ_own.data_ptr(), G.data_ptr(), f, exchange=True)
    return G


class PSpMMMax(torch.autograd.Function):
    """Z = max over each row's neighbours, element-wise (the GraphSAGE "pool" aggregator, PyG aggr="max"), with the call
    shape of PSpMM: PSpMMMax.apply(A, H). The pattern of A is used, not its values. The gradient goes to the winning
    entry of every (row, feature), the first one on ties (aggregate_max), including winners in other ranks' rows.
    Layouts as PSpMM. The plan must be bound (PgcnPlan.bind_values)."""

    @staticmethod
    def forward(ctx, A, H):
        ctx.plan = A
        _require_bound(A, "PSpMMMax walks the transposed records through the plan's value maps")
        Z_own, arg = aggregate_max(A, _own(A, H, "H"))
        ctx.save_for_backward(arg)
        return _to_layout(A, Z_own)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        (arg,) = ctx.saved_tensors
        return None, _to_layout(A, aggregate_max_backward(A, arg, _own(A, grad_output, "grad_output")))


# ---- gated aggregation (libpgcn_gated.so) ----------------------------------------------------------------------------

def _gated(dev, name, *args):
    """libpgcn_gated.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_gated(getattr(cabi.load_gated(), name)(*args, _stream_ptr()))


def _gated_operands(plan, K_own, Q_own, V_own, what):
    """The walks, then K_own, Q_own, V_own checked ([m, f] each, 2f <= f_max, a bound plan). The walks come first, so
    that a capture that needs them before they exist is refused before any work is enqueued."""
    walks = plan.gated_walks()
    f = K_own.shape[-1]
    if 2 * f > plan.f_max:
        raise ValueError("f=%d: %s exchanges [Q | V] rows of 2f = %d floats, the plan's f_max is %d: build the plan "
                         "with f_max >= 2f" % (f, what, 2 * f, plan.f_max))
    K_own = _check_feat(plan, K_own, plan.m, "K")
    Q_own = _check_feat(plan, Q_own, plan.m, "Q")
    V_own = _check_feat(plan, V_own, plan.m, "V")
    if Q_own.shape[1] != f or V_own.shape[1] != f:
        raise ValueError("K, Q and V must have the same width, got %d, %d and %d" % (f, Q_own.shape[1], V_own.shape[1]))
    _require_bound(plan, "%s exchanges [Q | V] through pgcn_halo_rows" % what)
    return walks, K_own, Q_own, V_own


def aggregate_gated(plan, K_own, Q_own, V_own):
    """(Z_own, QV_own, QV_halo): Z_own[i] = sum over row i's stored entries (i, j) of sigmoid(K[i] + Q[j]) * V[j],
    element-wise, over [own | halo] columns (pgcn_gated_forward); K_own, Q_own, V_own, Z_own are [m, f]. QV_own is the
    [m, 2f] concatenation [Q | V] and QV_halo [h, 2f] its halo rows from one exchange (pgcn_halo_rows), which
    aggregate_gated_backward takes. Needs a bound plan with f_max >= 2f."""
    (fwd, _), K_own, Q_own, V_own = _gated_operands(plan, K_own, Q_own, V_own, "aggregate_gated")
    lp, f, dev = plan.lp, K_own.shape[1], K_own.device
    QV = torch.cat([Q_own, V_own], 1)
    QV_halo = torch.empty((lp.h, 2 * f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", QV.data_ptr(), QV_halo.data_ptr(), 2 * f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _gated(dev, "pgcn_gated_forward", C.byref(fwd.c), lp.m, lp.h, K_own.data_ptr(), QV.data_ptr(), QV_halo.data_ptr(),
           Z.data_ptr(), work.data_ptr(), f)
    return Z, QV, QV_halo


def aggregate_gated_backward(plan, K_own, QV_own, QV_halo, gZ_own):
    """(dK, dQ, dV), each [m, f]: the gradients of aggregate_gated's Z_own for the output gradient gZ_own [m, f], from
    its QV_own and QV_halo. dK comes from the row walk (pgcn_gated_backward_rows); dQ and dV from the column walk over
    the transposed entries (pgcn_gated_backward_cols), whose halo rows go back to their owners and are added there
    (pgcn_halo_rows_add)."""
    f = K_own.shape[-1]
    if QV_own.dim() != 2 or QV_own.shape[1] != 2 * f:
        raise ValueError("QV_own must be [%d, %d], got %s" % (plan.m, 2 * f, tuple(QV_own.shape)))
    (fwd, tr), K_own, gZ_own, _ = _gated_operands(plan, K_own, gZ_own, gZ_own, "aggregate_gated_backward")
    lp, dev = plan.lp, K_own.device
    QV_own = QV_own.contiguous()
    if QV_own.shape[0] != lp.m or tuple(QV_halo.shape) != (lp.h, 2 * f):
        raise ValueError("QV_own / QV_halo must be [%d, %d] / [%d, %d], got %s / %s" % (
            lp.m, 2 * f, lp.h, 2 * f, tuple(QV_own.shape), tuple(QV_halo.shape)))
    QV_halo = QV_halo.contiguous()
    dK = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _gated(dev, "pgcn_gated_backward_rows", C.byref(fwd.c), lp.m, lp.h, K_own.data_ptr(), QV_own.data_ptr(),
           QV_halo.data_ptr(), gZ_own.data_ptr(), dK.data_ptr(), work.data_ptr(), f)
    dQV = torch.empty((lp.m + lp.h, 2 * f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, 2 * f), dtype=torch.float32, device=dev)
    _gated(dev, "pgcn_gated_backward_cols", C.byref(tr.c), lp.m, lp.h, K_own.data_ptr(), QV_own.data_ptr(),
           QV_halo.data_ptr(), gZ_own.data_ptr(), dQV.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dQV[lp.m:].data_ptr(), dQV.data_ptr(), 2 * f, exchange=True)
    return dK, dQV[:lp.m, :f], dQV[:lp.m, f:]


class PSpMMGated(torch.autograd.Function):
    """Sigmoid-gated aggregation over the plan's stored pattern, the message of PyG's ResGatedGraphConv (GatedGCN's
    without the edge features and the normalisation):

        PSpMMGated.apply(A, K, Q, V)
        out[i] = sum over the stored entries (i, j) of  sigmoid(K[i] + Q[j]) * V[j]        (element-wise, f features)

    K, Q and V are [rows, f] fp32 CUDA tensors, out is [rows, f] (rows = m in the "local" layout, n in the "global"
    one, as PSpMM). The values of A are not read; every stored entry contributes, duplicates included. One exchange
    per layer carries [Q | V] (2f floats per row), so the plan's f_max must be at least 2f; the backward returns the
    halo rows' partial dQ and dV to their owners in one reverse exchange. Nothing is stored per entry: the backward
    recomputes the gates from K, Q and V. Gradients go to K, Q and V. Deterministic. The exchange is the unsplit one
    (no per-source overlap). The plan must be bound (PgcnPlan.bind_values); the first call builds its index tables
    (PgcnPlan.gated_walks)."""

    @staticmethod
    def forward(ctx, A, K, Q, V):
        A.gated_walks()
        K_own = _own(A, K, "K")
        Z, QV, QV_halo = aggregate_gated(A, K_own, _own(A, Q, "Q"), _own(A, V, "V"))
        ctx.plan = A
        ctx.save_for_backward(K_own, QV, QV_halo)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        K_own, QV, QV_halo = ctx.saved_tensors
        dK, dQ, dV = aggregate_gated_backward(A, K_own, QV, QV_halo, _own(A, grad_output, "grad_output"))
        return None, _to_layout(A, dK), _to_layout(A, dQ), _to_layout(A, dV)


# ---- graph transformer attention (libpgcn_transformer.so) -----------------------------------------------------------

TRANSFORMER_MAX_F = 256


def transformer_scale(f, heads):
    """The default score scale, float32(1 / sqrt(f / heads)): 1 / sqrt of the head width."""
    import math
    import numpy as np
    return float(np.float32(1.0 / math.sqrt(f / heads)))


def _transformer(dev, name, *args):
    """libpgcn_transformer.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_transformer(getattr(cabi.load_transformer(), name)(*args, _stream_ptr()))


def _transformer_operands(plan, Q_own, K_own, V_own, heads, drop, what):
    """The walks and the global ids, then heads, width and Q_own, K_own, V_own checked ([m, f] each, f <= 256 and
    2f <= f_max, a bound plan). The walks and ids come first, so that a capture that needs them before they exist is
    refused before any work is enqueued."""
    walks = plan.gated_walks()
    gid = plan.global_ids()
    if drop is not None and drop.state.device != plan.device:
        raise ValueError("the EdgeDropout state lives on %s, the plan on %s" % (drop.state.device, plan.device))
    f = Q_own.shape[-1]
    if heads not in HEADS:
        raise ValueError("heads=%r: the transformer kernels take 1, 2, 4 or 8 heads" % (heads,))
    if f % heads:
        raise ValueError("f=%d is not a multiple of heads=%d" % (f, heads))
    if f > TRANSFORMER_MAX_F:
        raise ValueError("f=%d: the transformer kernels hold a row in registers, f <= %d" % (f, TRANSFORMER_MAX_F))
    if 2 * f > plan.f_max:
        raise ValueError("f=%d: %s exchanges [K | V] rows of 2f = %d floats, the plan's f_max is %d: build the plan "
                         "with f_max >= 2f" % (f, what, 2 * f, plan.f_max))
    Q_own = _check_feat(plan, Q_own, plan.m, "Q")
    K_own = _check_feat(plan, K_own, plan.m, "K")
    V_own = _check_feat(plan, V_own, plan.m, "V")
    if K_own.shape[1] != f or V_own.shape[1] != f:
        raise ValueError("Q, K and V must have the same width, got %d, %d and %d" % (f, K_own.shape[1], V_own.shape[1]))
    _require_bound(plan, "%s exchanges [K | V] through pgcn_halo_rows" % what)
    return walks, gid, Q_own, K_own, V_own


def _drop_args(drop, snap):
    """(drop, threshold, keep_scale) of the kernels: the snapshot's pointer, or NULL, 0, 1 without dropout."""
    return (None, 0, 1.0) if drop is None else (snap.data_ptr(), drop.threshold, drop.scale)


def aggregate_transformer(plan, Q_own, K_own, V_own, heads, scale=None, drop=None):
    """(Z_own, L, KV_own, KV_halo, snap): scaled dot-product attention over the plan's stored pattern with `heads` heads
    of width C = f / heads (pgcn_transformer_forward): s_eh = scale <Q[i, h], K[j, h]>, alpha = softmax of s over each
    row's stored entries per head, Z_own[i, h] = sum_e alpha_eh M_eh V[j, h]. Q_own, K_own, V_own, Z_own are [m, f],
    L [m, heads] the rows' log-sum-exp. KV_own is [K | V] ([m, 2f]) and KV_halo [h, 2f] its halo rows from one exchange
    (pgcn_halo_rows). scale None: float32(1 / sqrt(C)). drop (an EdgeDropout) with p > 0 draws a new counter (its
    snapshot `snap`, else None) and applies the mask M; aggregate_transformer_backward takes the same snapshot. Needs a
    bound plan with f_max >= 2f."""
    drop = _active(drop)
    (fwd, _), gid, Q_own, K_own, V_own = _transformer_operands(plan, Q_own, K_own, V_own, heads, drop,
                                                               "aggregate_transformer")
    lp, f, dev = plan.lp, Q_own.shape[1], Q_own.device
    scale = transformer_scale(f, heads) if scale is None else float(scale)
    snap = drop.draw() if drop else None
    KV = torch.cat([K_own, V_own], 1)
    KV_halo = torch.empty((lp.h, 2 * f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", KV.data_ptr(), KV_halo.data_ptr(), 2 * f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    L = torch.empty((lp.m, heads), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f + 2 * heads), dtype=torch.float32, device=dev)
    _transformer(dev, "pgcn_transformer_forward", C.byref(fwd.c), lp.m, lp.h, heads, Q_own.data_ptr(), KV.data_ptr(),
                 KV_halo.data_ptr(), scale, gid.data_ptr(), *_drop_args(drop, snap), Z.data_ptr(), L.data_ptr(),
                 work.data_ptr(), f)
    return Z, L, KV, KV_halo, snap


def aggregate_transformer_backward(plan, Q_own, KV_own, KV_halo, Z_own, L, gZ_own, heads, scale=None, drop=None,
                                   snap=None):
    """(dQ, dK, dV), each [m, f]: the gradients of aggregate_transformer's Z_own for the output gradient gZ_own [m, f],
    from its KV_own, KV_halo, Z_own and L and, with dropout, the same `drop` and its forward's `snap`. dQ and the rows'
    D = <gZ, Z> come from the row walk (pgcn_transformer_backward_rows); dK and dV from the column walk over the
    transposed entries (pgcn_transformer_backward_cols), whose halo rows go back to their owners and are added there
    (pgcn_halo_rows_add)."""
    drop = _active(drop)
    f = Q_own.shape[-1]
    if drop is not None and snap is None:
        raise ValueError("aggregate_transformer_backward with dropout needs the forward's snapshot")
    (fwd, tr), gid, Q_own, gZ_own, Z_own = _transformer_operands(plan, Q_own, gZ_own, Z_own, heads, drop,
                                                                 "aggregate_transformer_backward")
    lp, dev = plan.lp, Q_own.device
    KV_own, KV_halo, L = KV_own.contiguous(), KV_halo.contiguous(), L.contiguous()
    if tuple(KV_own.shape) != (lp.m, 2 * f) or tuple(KV_halo.shape) != (lp.h, 2 * f):
        raise ValueError("KV_own / KV_halo must be [%d, %d] / [%d, %d], got %s / %s" % (
            lp.m, 2 * f, lp.h, 2 * f, tuple(KV_own.shape), tuple(KV_halo.shape)))
    if tuple(L.shape) != (lp.m, heads):
        raise ValueError("L must be [%d, %d], got %s" % (lp.m, heads, tuple(L.shape)))
    scale = transformer_scale(f, heads) if scale is None else float(scale)
    dargs = _drop_args(drop, snap)
    dQ = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    D = torch.empty((lp.m, heads), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _transformer(dev, "pgcn_transformer_backward_rows", C.byref(fwd.c), lp.m, lp.h, heads, Q_own.data_ptr(),
                 KV_own.data_ptr(), KV_halo.data_ptr(), scale, gid.data_ptr(), *dargs, gZ_own.data_ptr(),
                 Z_own.data_ptr(), L.data_ptr(), dQ.data_ptr(), D.data_ptr(), work.data_ptr(), f)
    dKV = torch.empty((lp.m + lp.h, 2 * f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, 2 * f), dtype=torch.float32, device=dev)
    _transformer(dev, "pgcn_transformer_backward_cols", C.byref(tr.c), lp.m, lp.h, heads, Q_own.data_ptr(),
                 KV_own.data_ptr(), KV_halo.data_ptr(), scale, gid.data_ptr(), *dargs, gZ_own.data_ptr(), L.data_ptr(),
                 D.data_ptr(), dKV.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dKV[lp.m:].data_ptr(), dKV.data_ptr(), 2 * f, exchange=True)
    return dQ, dKV[:lp.m, :f], dKV[:lp.m, f:]


class PTransformerAttention(torch.autograd.Function):
    """Scaled dot-product attention over the plan's stored pattern, the attention of PyG's TransformerConv (concat=True,
    without edge features), with K heads of width C = f / K concatenated:

        PTransformerAttention.apply(A, Q, K, V, heads, scale=None, dropout=None)
        s_eh = scale <Q[i, h], K[j, h]>,  alpha_.h = softmax of s_.h over row i's stored entries,
        out[i, h] = sum over the stored entries e = (i, j) of  alpha_eh V[j, h]

    Q, K and V are [rows, f] fp32 CUDA tensors (f <= 256, heads 1, 2, 4 or 8 dividing f), out is [rows, f] (rows = m in
    the "local" layout, n in the "global" one, as PSpMM). scale None: float32(1 / sqrt(C)). The values of A are not
    read; every stored entry contributes, duplicates included; a row without entries gives 0. One exchange per layer
    carries [K | V] (2f floats per row), so the plan's f_max must be at least 2f; the backward returns the halo rows'
    partial dK and dV to their owners in one reverse exchange. Only the rows' log-sum-exp ([rows, K]) is kept besides
    the operands: the backward recomputes the probabilities. Gradients go to Q, K and V. Deterministic. The exchanges
    are the unsplit ones (no per-source overlap). The plan must be bound (PgcnPlan.bind_values); the first call builds
    its index tables (PgcnPlan.gated_walks, PgcnPlan.global_ids).

    dropout (an op.EdgeDropout with p > 0): attention dropout on every head, the mask of op.edge_dropout drawn inline
    from the global (row, column) of each entry, so every partition draws the same mask. Each forward advances the
    dropout's counter on the device and the backward reuses that forward's snapshot, so CUDA-graph replays draw new
    masks. None or p == 0: no mask is drawn."""

    @staticmethod
    def forward(ctx, A, Q, K, V, heads, scale=None, dropout=None):
        drop = _active(dropout)
        A.gated_walks()
        A.global_ids()
        Q_own = _own(A, Q, "Q")
        Z, L, KV, KV_halo, snap = aggregate_transformer(A, Q_own, _own(A, K, "K"), _own(A, V, "V"), heads, scale, drop)
        ctx.plan, ctx.heads, ctx.drop = A, heads, drop
        ctx.scale = transformer_scale(Q_own.shape[1], heads) if scale is None else float(scale)
        ctx.save_for_backward(Q_own, KV, KV_halo, Z, L, snap)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        Q_own, KV, KV_halo, Z, L, snap = ctx.saved_tensors
        dQ, dK, dV = aggregate_transformer_backward(A, Q_own, KV, KV_halo, Z, L, _own(A, grad_output, "grad_output"),
                                                    ctx.heads, ctx.scale, ctx.drop, snap)
        return None, _to_layout(A, dQ), _to_layout(A, dK), _to_layout(A, dV), None, None, None


# ---- GatedGCN (libpgcn_gatedgcn.so) ----------------------------------------------------------------------------------

GATEDGCN_EPS = 1e-6


def _gatedgcn(dev, name, *args):
    """libpgcn_gatedgcn.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_gatedgcn(getattr(cabi.load_gatedgcn(), name)(*args, _stream_ptr()))


def _check_eps(eps):
    import math
    eps = float(eps)
    if not (eps >= 0.0) or math.isinf(eps):
        raise ValueError("eps=%r: GatedGCN's eps must be finite and >= 0" % (eps,))
    return eps


def _check_edges(plan, x, f, what):
    """x, a per-entry tensor: fp32 CUDA [nnz_local, f] in the plan's forward-entry order. Returns it contiguous."""
    _check_f32(x, what)
    nnz = plan.lp.nnz()
    if x.dim() != 2 or tuple(x.shape) != (nnz, f):
        raise ValueError("%s must be [%d, %d] (the plan's local entries, edge_pairs() order), got %s" % (
            what, nnz, f, tuple(x.shape)))
    return x.contiguous()


def _gatedgcn_operands(plan, Dx_own, Ex_own, Bx_own, eps, what):
    """The walks and the transposed entries, then eps and Dx_own, Ex_own, Bx_own checked ([m, f] each, 2f <= f_max, a
    bound plan), then the kernels loaded (pgcn_gatedgcn_load). The tables come first, so that a capture that needs them
    before they exist is refused before any work is enqueued."""
    walks = plan.gated_walks()
    perm = plan.transposed_entries()
    eps = _check_eps(eps)
    f = Dx_own.shape[-1]
    if 2 * f > plan.f_max:
        raise ValueError("f=%d: %s exchanges [Ex | Bx] rows of 2f = %d floats, the plan's f_max is %d: build the plan "
                         "with f_max >= 2f" % (f, what, 2 * f, plan.f_max))
    Dx_own = _check_feat(plan, Dx_own, plan.m, "Dx")
    Ex_own = _check_feat(plan, Ex_own, plan.m, "Ex")
    Bx_own = _check_feat(plan, Bx_own, plan.m, "Bx")
    if Ex_own.shape[1] != f or Bx_own.shape[1] != f:
        raise ValueError("Dx, Ex and Bx must have the same width, got %d, %d and %d" % (f, Ex_own.shape[1],
                                                                                       Bx_own.shape[1]))
    _require_bound(plan, "%s exchanges [Ex | Bx] through pgcn_halo_rows" % what)
    with torch.cuda.device(plan.device):
        # every kernel loaded before the exchange: ranks of one process must not load one behind a waiting exchange
        cabi.check_gatedgcn(cabi.load_gatedgcn().pgcn_gatedgcn_load())
    return walks, perm, Dx_own, Ex_own, Bx_own, eps


def aggregate_gatedgcn(plan, Dx_own, Ex_own, Bx_own, Ce, eps=GATEDGCN_EPS):
    """(Z_own, Ehat, den, EB_own, EB_halo): GatedGCN's edge-gated aggregation over the plan's stored pattern
    (pgcn_gatedgcn_forward). For every local entry e = (i, j): Ehat_e = (Dx[i] + Ex[j]) + Ce_e, s_e = sigmoid(Ehat_e),
    Z_own[i] = sum_e s_e Bx[j] / (sum_e s_e + eps), element-wise. Dx_own, Ex_own, Bx_own, Z_own and den (the rows' sums
    of gates) are [m, f]; Ce and Ehat are [nnz_local, f] in edge_pairs() order. EB_own is [Ex | Bx] ([m, 2f]) and EB_halo
    [h, 2f] its halo rows from one exchange (pgcn_halo_rows), which aggregate_gatedgcn_backward takes. Needs a bound
    plan with f_max >= 2f."""
    (fwd, _), _, Dx_own, Ex_own, Bx_own, eps = _gatedgcn_operands(plan, Dx_own, Ex_own, Bx_own, eps,
                                                                  "aggregate_gatedgcn")
    lp, f, dev = plan.lp, Dx_own.shape[1], Dx_own.device
    Ce = _check_edges(plan, Ce, f, "Ce")
    EB = torch.cat([Ex_own, Bx_own], 1)
    EB_halo = torch.empty((lp.h, 2 * f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", EB.data_ptr(), EB_halo.data_ptr(), 2 * f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    den = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    Ehat = torch.empty((lp.nnz(), f), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, 2 * f), dtype=torch.float32, device=dev)
    _gatedgcn(dev, "pgcn_gatedgcn_forward", C.byref(fwd.c), lp.m, lp.h, Dx_own.data_ptr(), EB.data_ptr(),
              EB_halo.data_ptr(), Ce.data_ptr(), eps, Z.data_ptr(), den.data_ptr(), Ehat.data_ptr(), work.data_ptr(), f)
    return Z, Ehat, den, EB, EB_halo


def aggregate_gatedgcn_backward(plan, Ehat, EB_own, EB_halo, Z_own, den, gZ_own, gEhat=None, eps=GATEDGCN_EPS):
    """(dDx, dEx, dBx, dCe): the gradients of aggregate_gatedgcn's outputs for the output gradients gZ_own [m, f] and
    gEhat [nnz_local, f] (None: zero), from its Ehat, EB_own, EB_halo, Z_own and den and the same eps. The row walk
    (pgcn_gatedgcn_backward_rows) forms U = gZ / (den + eps) once per row and gives dCe ([nnz_local, f], the gradient of
    Ehat and of Ce) and dDx; the column walk over the transposed entries (pgcn_gatedgcn_backward_cols) gives dEx and dBx,
    whose halo rows go back to their owners and are added there (pgcn_halo_rows_add)."""
    f = Z_own.shape[-1]
    (fwd, tr), perm, Z_own, den, gZ_own, eps = _gatedgcn_operands(plan, Z_own, den, gZ_own, eps,
                                                                  "aggregate_gatedgcn_backward")
    lp, dev = plan.lp, Z_own.device
    Ehat = _check_edges(plan, Ehat, f, "Ehat")
    if gEhat is not None:
        gEhat = _check_edges(plan, gEhat, f, "gEhat")
    EB_own, EB_halo = EB_own.contiguous(), EB_halo.contiguous()
    if tuple(EB_own.shape) != (lp.m, 2 * f) or tuple(EB_halo.shape) != (lp.h, 2 * f):
        raise ValueError("EB_own / EB_halo must be [%d, %d] / [%d, %d], got %s / %s" % (
            lp.m, 2 * f, lp.h, 2 * f, tuple(EB_own.shape), tuple(EB_halo.shape)))
    U = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    dDx = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    dCe = torch.empty((lp.nnz(), f), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _gatedgcn(dev, "pgcn_gatedgcn_backward_rows", C.byref(fwd.c), lp.m, lp.h, EB_own.data_ptr(), EB_halo.data_ptr(),
              Ehat.data_ptr(), _ptr(gEhat), Z_own.data_ptr(), den.data_ptr(), gZ_own.data_ptr(), eps, U.data_ptr(),
              dCe.data_ptr(), dDx.data_ptr(), work.data_ptr(), f)
    dEB = torch.empty((lp.m + lp.h, 2 * f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, 2 * f), dtype=torch.float32, device=dev)
    _gatedgcn(dev, "pgcn_gatedgcn_backward_cols", C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, Ehat.data_ptr(),
              dCe.data_ptr(), U.data_ptr(), dEB.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dEB[lp.m:].data_ptr(), dEB.data_ptr(), 2 * f, exchange=True)
    return dDx, dEB[:lp.m, :f], dEB[:lp.m, f:], dCe


class PGatedGCN(torch.autograd.Function):
    """GatedGCN's edge-gated aggregation over the plan's stored pattern (Bresson & Laurent; the layer of Dwivedi et
    al.'s benchmarking-gnns and GraphGPS's default local layer), with an edge-feature stream:

        Z, Ehat = PGatedGCN.apply(A, Dx, Ex, Bx, Ce, eps=1e-6)
        Ehat_e = (Dx[i] + Ex[j]) + Ce_e                      for every stored entry e = (i, j)
        Z[i]   = sum_e sigmoid(Ehat_e) Bx[j] / (sum_e sigmoid(Ehat_e) + eps)          (element-wise, f features)

    Dx, Ex and Bx are [rows, f] fp32 CUDA tensors and Z is [rows, f] (rows = m in the "local" layout, n in the "global"
    one, as PSpMM). Ce and Ehat are [nnz_local, f] in both layouts: one row per local entry in the order of
    PgcnPlan.edge_pairs(). They never cross ranks, since every entry belongs to the rank that owns its row. The values of
    A are not read; every stored entry contributes, duplicates included. A row without entries gives 0 (NaN when
    eps == 0). One exchange per layer carries [Ex | Bx] (2f floats per row), so the plan's f_max must be at least 2f; the
    backward returns the halo rows' partial dEx and dBx to their owners in one reverse exchange. Saved for the backward:
    Ehat (the output), Z, the rows' gate sums and the [Ex | Bx] own and halo rows; the gates are recomputed. An unused
    Ehat costs no gradient tensor: its gradient reaches the kernel as NULL. Gradients go to Dx, Ex, Bx and Ce.
    Deterministic. The exchanges are the unsplit ones (no per-source overlap). The plan must be bound
    (PgcnPlan.bind_values); the first call builds its index tables (PgcnPlan.gated_walks,
    PgcnPlan.transposed_entries)."""

    @staticmethod
    def forward(ctx, A, Dx, Ex, Bx, Ce, eps=GATEDGCN_EPS):
        ctx.set_materialize_grads(False)
        A.gated_walks()
        A.transposed_entries()
        Z, Ehat, den, EB, EB_halo = aggregate_gatedgcn(A, _own(A, Dx, "Dx"), _own(A, Ex, "Ex"), _own(A, Bx, "Bx"),
                                                       Ce, eps)
        ctx.plan, ctx.eps = A, _check_eps(eps)
        ctx.save_for_backward(Ehat, Z, den, EB, EB_halo)
        return _to_layout(A, Z), Ehat

    @staticmethod
    def backward(ctx, gZ, gEhat):
        A = ctx.plan
        Ehat, Z, den, EB, EB_halo = ctx.saved_tensors
        gZ = torch.zeros_like(Z) if gZ is None else _own(A, gZ, "grad Z")
        dDx, dEx, dBx, dCe = aggregate_gatedgcn_backward(A, Ehat, EB, EB_halo, Z, den, gZ, gEhat, ctx.eps)
        return None, _to_layout(A, dDx), _to_layout(A, dEx), _to_layout(A, dBx), dCe, None


# ---- graph transformer attention with edge features (libpgcn_transformer_edge.so) ----------------------------------

def _transformer_edge(dev, name, *args):
    """libpgcn_transformer_edge.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_transformer_edge(getattr(cabi.load_transformer_edge(), name)(*args, _stream_ptr()))


def _transformer_edge_operands(plan, Q_own, K_own, V_own, E, heads, drop, what):
    """_transformer_operands, then the transposed entries, E checked ([nnz_local, f]) and the kernels loaded
    (pgcn_transformer_edge_load). Every table comes before any work is enqueued, so that a capture that needs one
    before it exists is refused first."""
    walks, gid, Q_own, K_own, V_own = _transformer_operands(plan, Q_own, K_own, V_own, heads, drop, what)
    perm = plan.transposed_entries()
    E = _check_edges(plan, E, Q_own.shape[1], "E")
    with torch.cuda.device(plan.device):
        # every kernel loaded before the exchange: ranks of one process must not load one behind a waiting exchange
        cabi.check_transformer_edge(cabi.load_transformer_edge().pgcn_transformer_edge_load())
    return walks, perm, gid, Q_own, K_own, V_own, E


def aggregate_transformer_edge(plan, Q_own, K_own, V_own, E, heads, scale=None, drop=None):
    """(Z_own, L, KV_own, KV_halo, snap): aggregate_transformer with an edge term E ([nnz_local, f] in edge_pairs()
    order) added to the keys and values of every local entry e = (i, j) (pgcn_transformer_edge_forward):
    s_eh = scale <Q[i, h], K[j, h] + E_e[h]>, alpha = softmax of s over each row's stored entries per head,
    Z_own[i, h] = sum_e alpha_eh M_eh (V[j, h] + E_e[h]). Outputs, scale and drop as aggregate_transformer;
    aggregate_transformer_edge_backward takes them. E never crosses ranks. Needs a bound plan with f_max >= 2f."""
    drop = _active(drop)
    (fwd, _), _, gid, Q_own, K_own, V_own, E = _transformer_edge_operands(plan, Q_own, K_own, V_own, E, heads, drop,
                                                                          "aggregate_transformer_edge")
    lp, f, dev = plan.lp, Q_own.shape[1], Q_own.device
    scale = transformer_scale(f, heads) if scale is None else float(scale)
    snap = drop.draw() if drop else None
    KV = torch.cat([K_own, V_own], 1)
    KV_halo = torch.empty((lp.h, 2 * f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", KV.data_ptr(), KV_halo.data_ptr(), 2 * f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    L = torch.empty((lp.m, heads), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f + 2 * heads), dtype=torch.float32, device=dev)
    _transformer_edge(dev, "pgcn_transformer_edge_forward", C.byref(fwd.c), lp.m, lp.h, heads, Q_own.data_ptr(),
                      KV.data_ptr(), KV_halo.data_ptr(), E.data_ptr(), scale, gid.data_ptr(), *_drop_args(drop, snap),
                      Z.data_ptr(), L.data_ptr(), work.data_ptr(), f)
    return Z, L, KV, KV_halo, snap


def aggregate_transformer_edge_backward(plan, Q_own, KV_own, KV_halo, E, Z_own, L, gZ_own, heads, scale=None,
                                        drop=None, snap=None, need_dE=True):
    """(dQ, dK, dV, dE): the gradients of aggregate_transformer_edge's Z_own for the output gradient gZ_own [m, f], from
    its KV_own, KV_halo, Z_own and L, the same E and, with dropout, the same `drop` and its forward's `snap`. The row
    walk (pgcn_transformer_edge_backward_rows) gives dQ, dE ([nnz_local, f]; None when need_dE is false, and then it is
    not computed) and each entry's [P | ds] ([nnz_local, 2 heads]); the column walk over the transposed entries
    (pgcn_transformer_edge_backward_cols) reads those and gives dK and dV, whose halo rows go back to their owners and
    are added there (pgcn_halo_rows_add)."""
    drop = _active(drop)
    f = Q_own.shape[-1]
    if drop is not None and snap is None:
        raise ValueError("aggregate_transformer_edge_backward with dropout needs the forward's snapshot")
    (fwd, tr), perm, gid, Q_own, gZ_own, Z_own, E = _transformer_edge_operands(
        plan, Q_own, gZ_own, Z_own, E, heads, drop, "aggregate_transformer_edge_backward")
    lp, dev = plan.lp, Q_own.device
    KV_own, KV_halo, L = KV_own.contiguous(), KV_halo.contiguous(), L.contiguous()
    if tuple(KV_own.shape) != (lp.m, 2 * f) or tuple(KV_halo.shape) != (lp.h, 2 * f):
        raise ValueError("KV_own / KV_halo must be [%d, %d] / [%d, %d], got %s / %s" % (
            lp.m, 2 * f, lp.h, 2 * f, tuple(KV_own.shape), tuple(KV_halo.shape)))
    if tuple(L.shape) != (lp.m, heads):
        raise ValueError("L must be [%d, %d], got %s" % (lp.m, heads, tuple(L.shape)))
    scale = transformer_scale(f, heads) if scale is None else float(scale)
    dQ = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    D = torch.empty((lp.m, heads), dtype=torch.float32, device=dev)
    PS = torch.empty((lp.nnz(), 2 * heads), dtype=torch.float32, device=dev)
    dE = torch.empty((lp.nnz(), f), dtype=torch.float32, device=dev) if need_dE else None
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _transformer_edge(dev, "pgcn_transformer_edge_backward_rows", C.byref(fwd.c), lp.m, lp.h, heads,
                      Q_own.data_ptr(), KV_own.data_ptr(), KV_halo.data_ptr(), E.data_ptr(), scale, gid.data_ptr(),
                      *_drop_args(drop, snap), gZ_own.data_ptr(), Z_own.data_ptr(), L.data_ptr(), dQ.data_ptr(),
                      D.data_ptr(), PS.data_ptr(), _ptr(dE), work.data_ptr(), f)
    dKV = torch.empty((lp.m + lp.h, 2 * f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, 2 * f), dtype=torch.float32, device=dev)
    _transformer_edge(dev, "pgcn_transformer_edge_backward_cols", C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, heads,
                      Q_own.data_ptr(), gZ_own.data_ptr(), PS.data_ptr(), scale, dKV.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dKV[lp.m:].data_ptr(), dKV.data_ptr(), 2 * f, exchange=True)
    return dQ, dKV[:lp.m, :f], dKV[:lp.m, f:], dE


class PTransformerEdgeAttention(torch.autograd.Function):
    """PTransformerAttention with edge features, the attention of PyG's TransformerConv(edge_dim=..., concat=True,
    beta=False) with E = lin_edge(edge_attr) formed by the caller:

        PTransformerEdgeAttention.apply(A, Q, K, V, E, heads, scale=None, dropout=None)
        s_eh = scale <Q[i, h], K[j, h] + E_e[h]>,  alpha_.h = softmax of s_.h over row i's stored entries,
        out[i, h] = sum over the stored entries e = (i, j) of  alpha_eh (V[j, h] + E_e[h])

    Q, K, V and out as PTransformerAttention's ([rows, f] in the plan's layout). E is [nnz_local, f] in both layouts:
    one row per local entry in the order of PgcnPlan.edge_pairs(). It never crosses ranks, since every entry belongs to
    the rank that owns its row. Gradients go to Q, K, V and E; dE is computed only when E requires it. The backward
    stores each entry's [P | ds] (2 heads floats) between its two walks, so that the column walk reads no E. dropout,
    heads, scale, the exchanges and the plan's tables as PTransformerAttention's; the first call also builds
    PgcnPlan.transposed_entries. Deterministic."""

    @staticmethod
    def forward(ctx, A, Q, K, V, E, heads, scale=None, dropout=None):
        drop = _active(dropout)
        A.gated_walks()
        A.global_ids()
        A.transposed_entries()
        Q_own = _own(A, Q, "Q")
        Z, L, KV, KV_halo, snap = aggregate_transformer_edge(A, Q_own, _own(A, K, "K"), _own(A, V, "V"), E, heads,
                                                             scale, drop)
        ctx.plan, ctx.heads, ctx.drop = A, heads, drop
        ctx.scale = transformer_scale(Q_own.shape[1], heads) if scale is None else float(scale)
        ctx.save_for_backward(Q_own, KV, KV_halo, E.contiguous(), Z, L, snap)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        Q_own, KV, KV_halo, E, Z, L, snap = ctx.saved_tensors
        dQ, dK, dV, dE = aggregate_transformer_edge_backward(A, Q_own, KV, KV_halo, E, Z, L,
                                                             _own(A, grad_output, "grad_output"), ctx.heads,
                                                             ctx.scale, ctx.drop, snap, ctx.needs_input_grad[4])
        return None, _to_layout(A, dQ), _to_layout(A, dK), _to_layout(A, dV), dE, None, None, None


# ---- GINE (libpgcn_gine.so) ------------------------------------------------------------------------------------------

def _gine(dev, name, *args):
    """libpgcn_gine.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_gine(getattr(cabi.load_gine(), name)(*args, _stream_ptr()))


def _gine_operands(plan, X_own, E, what):
    """The walks and the transposed entries, then X_own ([m, f], f <= f_max) and E ([nnz_local, f]) checked and the plan
    bound, then the kernels loaded (pgcn_gine_load). The tables come first, so that a capture that needs them before
    they exist is refused before any work is enqueued."""
    walks = plan.gated_walks()
    perm = plan.transposed_entries()
    X_own = _check_feat(plan, X_own, plan.m, "X")
    E = _check_edges(plan, E, X_own.shape[1], "E")
    _require_bound(plan, "%s exchanges X through pgcn_halo_rows" % what)
    with torch.cuda.device(plan.device):
        # every kernel loaded before the exchange: ranks of one process must not load one behind a waiting exchange
        cabi.check_gine(cabi.load_gine().pgcn_gine_load())
    return walks, perm, X_own, E


def aggregate_gine(plan, X_own, E):
    """(Z_own, X_halo): GINE's aggregation over the plan's stored pattern (pgcn_gine_forward). For every local entry
    e = (i, j): Z_own[i] = sum_e relu(X[j] + E_e), element-wise, over [own | halo] columns. X_own and Z_own are [m, f],
    E is [nnz_local, f] in edge_pairs() order; X_halo [h, f] is X's halo rows from one exchange (pgcn_halo_rows), which
    aggregate_gine_backward takes. Needs a bound plan with f_max >= f."""
    (fwd, _), _, X_own, E = _gine_operands(plan, X_own, E, "aggregate_gine")
    lp, f, dev = plan.lp, X_own.shape[1], X_own.device
    X_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", X_own.data_ptr(), X_halo.data_ptr(), f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f), dtype=torch.float32, device=dev)
    _gine(dev, "pgcn_gine_forward", C.byref(fwd.c), lp.m, lp.h, X_own.data_ptr(), X_halo.data_ptr(), E.data_ptr(),
          Z.data_ptr(), work.data_ptr(), f)
    return Z, X_halo


def aggregate_gine_backward(plan, X_own, X_halo, E, gZ_own, need_dE=True):
    """(dX_own, dE): the gradients of aggregate_gine's Z_own for the output gradient gZ_own [m, f], from the same X_own
    and E and its X_halo. One column walk over the transposed entries (pgcn_gine_backward) recomputes each entry's ReLU
    mask and gives dE ([nnz_local, f]; None when need_dE is false, and then it is not computed) and dX, whose halo rows
    go back to their owners and are added there (pgcn_halo_rows_add)."""
    (_, tr), perm, X_own, E = _gine_operands(plan, X_own, E, "aggregate_gine_backward")
    lp, f, dev = plan.lp, X_own.shape[1], X_own.device
    gZ_own = _check_feat(plan, gZ_own, plan.m, "gZ")
    if gZ_own.shape[1] != f:
        raise ValueError("X and gZ must have the same width, got %d and %d" % (f, gZ_own.shape[1]))
    X_halo = X_halo.contiguous()
    if tuple(X_halo.shape) != (lp.h, f):
        raise ValueError("X_halo must be [%d, %d], got %s" % (lp.h, f, tuple(X_halo.shape)))
    dE = torch.empty((lp.nnz(), f), dtype=torch.float32, device=dev) if need_dE else None
    dX = torch.empty((lp.m + lp.h, f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, f), dtype=torch.float32, device=dev)
    _gine(dev, "pgcn_gine_backward", C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, X_own.data_ptr(), X_halo.data_ptr(),
          E.data_ptr(), gZ_own.data_ptr(), _ptr(dE), dX.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dX[lp.m:].data_ptr(), dX.data_ptr(), f, exchange=True)
    return dX[:lp.m], dE


class PGINE(torch.autograd.Function):
    """GINE's aggregation over the plan's stored pattern (Hu et al.; the message of PyG's GINEConv, without the self
    term (1 + eps) x_i and the MLP, which the layer adds):

        Z = PGINE.apply(A, X, E)
        Z[i] = sum over the stored entries e = (i, j) of  relu(X[j] + E_e)                (element-wise, f features)

    X and Z are [rows, f] fp32 CUDA tensors (rows = m in the "local" layout, n in the "global" one, as PSpMM). E is
    [nnz_local, f] in both layouts: one row per local entry in the order of PgcnPlan.edge_pairs(). It never crosses
    ranks, since every entry belongs to the rank that owns its row. The values of A are not read; every stored entry
    contributes, duplicates included. relu is torch's: NaN propagates, -0 stays -0, and the gradient passes where
    X[j] + E_e > 0 or is NaN. One exchange per layer carries X (f floats per row), so the plan's f_max must be at least
    f; the backward returns the halo rows' partial dX to their owners in one reverse exchange. Saved for the backward:
    X's own and halo rows and E; the ReLU mask is recomputed. Gradients go to X and E; dE is computed only when E
    requires it. Deterministic. The exchanges are the unsplit ones (no per-source overlap). The plan must be bound
    (PgcnPlan.bind_values); the first call builds its index tables (PgcnPlan.gated_walks,
    PgcnPlan.transposed_entries)."""

    @staticmethod
    def forward(ctx, A, X, E):
        A.gated_walks()
        A.transposed_entries()
        X_own = _own(A, X, "X")
        Z, X_halo = aggregate_gine(A, X_own, E)
        ctx.plan = A
        ctx.save_for_backward(X_own, X_halo, E)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        X_own, X_halo, E = ctx.saved_tensors
        dX, dE = aggregate_gine_backward(A, X_own, X_halo, E, _own(A, grad_output, "grad_output"),
                                         ctx.needs_input_grad[2])
        return None, _to_layout(A, dX), dE


# ---- R-GCN relational aggregation (libpgcn_rgcn.so) ------------------------------------------------------------------

RGCN_AGGRS = ("add", "mean")


def _rgcn(dev, name, *args):
    """libpgcn_rgcn.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_rgcn(getattr(cabi.load_rgcn(), name)(*args, _stream_ptr()))


def rgcn_weights(plan, walks, w, aggr):
    """The entries' fp32 weights [nnz_local] the relational kernels take, in edge_pairs() order, or None for all ones:
    w for aggr="add", 1 / c for aggr="mean" (walks.mean, c the entries of the entry's (row, relation) pair), and the
    fp32 product w * (1 / c) for both. w has no gradient: one that requires it is refused."""
    from .plan import check_values
    if aggr not in RGCN_AGGRS:
        raise ValueError("aggr=%r: R-GCN aggregates with one of %s" % (aggr, ", ".join(map(repr, RGCN_AGGRS))))
    if w is not None:
        if torch.is_tensor(w) and w.requires_grad:
            raise ValueError("w requires grad, but the relational aggregation has no gradient for its edge weights: "
                             "pass w.detach()")
        w = check_values(plan, w)
    if aggr == "add":
        return w
    return walks.mean if w is None else w * walks.mean


def _rgcn_prepare(plan, what):
    """The plan bound, then the kernels loaded (pgcn_rgcn_load)."""
    _require_bound(plan, "%s exchanges through pgcn_halo_rows" % what)
    with torch.cuda.device(plan.device):
        # every kernel loaded before the exchange: ranks of one process must not load one behind a waiting exchange
        cabi.check_rgcn(cabi.load_rgcn().pgcn_rgcn_load())


def aggregate_rgcn(plan, walks, X_own, w):
    """(Z_own, X_halo): the per-relation aggregation over the plan's stored pattern (pgcn_rgcn_forward). With `walks`
    = plan.relation_walks(rel, R) and for every local entry e = (i, j): Z_own[i, rel_e] += w_e X[j], over [own | halo]
    columns, each relation's sum in forward CSR order. X_own is [m, f], Z_own [m, R, f]; w fp32 [nnz_local] in
    edge_pairs() order or None (all ones), e.g. rgcn_weights(...). X_halo [h, f] is X's halo rows from one exchange
    (pgcn_halo_rows), whatever R is. Needs a bound plan with f_max >= f."""
    X_own = _check_feat(plan, X_own, plan.m, "X")
    _rgcn_prepare(plan, "aggregate_rgcn")
    lp, f, dev, R = plan.lp, X_own.shape[1], X_own.device, walks.R
    X_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", X_own.data_ptr(), X_halo.data_ptr(), f, exchange=False)
    Z = torch.empty((lp.m, R, f), dtype=torch.float32, device=dev)
    work = torch.empty((walks.fwd.nslots, f), dtype=torch.float32, device=dev)
    _rgcn(dev, "pgcn_rgcn_forward", C.byref(walks.fwd.c), walks.perm_f.data_ptr(), lp.m, lp.h, R, X_own.data_ptr(),
          X_halo.data_ptr(), _ptr(w), Z.data_ptr(), work.data_ptr(), f)
    return Z, X_halo


def aggregate_rgcn_backward(plan, walks, gZ_own, w):
    """dX_own [m, f]: the gradient of aggregate_rgcn's Z_own for gZ_own [m, R, f] with the same walks and w. One column
    walk over the transposed entries (pgcn_rgcn_backward) gives dX[j] = sum_{e in column j} w_e gZ[i_e, rel_e] for the
    own and halo columns; the halo rows go back to their owners and are added there (pgcn_halo_rows_add)."""
    lp, R = plan.lp, walks.R
    _check_f32(gZ_own, "gZ")
    if gZ_own.dim() != 3 or tuple(gZ_own.shape[:2]) != (lp.m, R):
        raise ValueError("gZ must be [%d, %d, f], got %s" % (lp.m, R, tuple(gZ_own.shape)))
    f, dev = gZ_own.shape[2], gZ_own.device
    if f > plan.f_max:
        raise ValueError("f=%d exceeds the plan's f_max=%d" % (f, plan.f_max))
    gZ_own = gZ_own.contiguous()
    perm = plan.transposed_entries()
    _rgcn_prepare(plan, "aggregate_rgcn_backward")
    dX = torch.empty((lp.m + lp.h, f), dtype=torch.float32, device=dev)
    work = torch.empty((walks.tr.nslots, f), dtype=torch.float32, device=dev)
    _rgcn(dev, "pgcn_rgcn_backward", C.byref(walks.tr.c), perm.data_ptr(), lp.m, lp.h, R, gZ_own.data_ptr(), _ptr(w),
          dX.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dX[lp.m:].data_ptr(), dX.data_ptr(), f, exchange=True)
    return dX[:lp.m]


class PRGCN(torch.autograd.Function):
    """R-GCN's relational aggregation over the plan's stored pattern (Schlichtkrull et al.; the message of PyG's
    RGCNConv and DGL's RelGraphConv, before the per-relation weights, which the layer applies):

        Z = PRGCN.apply(A, X, rel, R, w=None, aggr="mean")
        Z[i, r] = sum over the stored entries e = (i, j) with rel_e = r of  w_e X[j]          (element-wise, f features)

    X is [rows, f] and Z [rows, R, f], fp32 CUDA tensors (rows = m in the "local" layout, n in the "global" one, as
    PSpMM). rel is an integer tensor [nnz_local] of relations in [0, R), w None (every weight 1) or fp32 [nnz_local],
    both in the order of PgcnPlan.edge_pairs() in both layouts. aggr="add" takes w_e as given; aggr="mean" (PyG's
    default) multiplies it by 1 / c, c the number of entries of the entry's (row, relation) pair. The values of A are
    not read; every stored entry contributes, duplicates included; a (row, relation) pair without entries gives zeros.
    One exchange per layer carries X (f floats per row, whatever R is), so the plan's f_max must be at least f; the
    backward returns the halo rows' partial dX to their owners in one reverse exchange. Nothing is saved for the
    backward but the weights. The gradient goes to X only: a w that requires grad is refused. Deterministic. The
    exchanges are the unsplit ones (no per-source overlap). The plan must be bound (PgcnPlan.bind_values); the first
    call with a rel tensor builds its tables (PgcnPlan.relation_walks)."""

    @staticmethod
    def forward(ctx, A, X, rel, R, w=None, aggr="mean"):
        walks = A.relation_walks(rel, R)
        weights = rgcn_weights(A, walks, w, aggr)
        Z, _ = aggregate_rgcn(A, walks, _own(A, X, "X"), weights)
        ctx.plan, ctx.walks = A, walks
        ctx.save_for_backward(weights)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A, walks = ctx.plan, ctx.walks
        (weights,) = ctx.saved_tensors
        dX = aggregate_rgcn_backward(A, walks, _owned(A, grad_output), weights)
        return None, _to_layout(A, dX), None, None, None, None


# ---- GATv2 attention with edge features (libpgcn_gatv2_edge.so) -----------------------------------------------------

GATV2_EDGE_MAX_F = 256


def _gatv2_edge(dev, name, *args):
    """libpgcn_gatv2_edge.<name>(*args, stream) on `dev`'s current stream, its status checked."""
    with torch.cuda.device(dev):
        cabi.check_gatv2_edge(getattr(cabi.load_gatv2_edge(), name)(*args, _stream_ptr()))


def _gatv2_att(att, f):
    """att checked as PGATv2Attention checks it ([K, f / K], K in HEADS, fp32 CUDA): (its heads, att detached and
    contiguous)."""
    if att.dim() != 2:
        raise ValueError("att must be [heads, f / heads], got %s" % (tuple(att.shape),))
    K = att.shape[0]
    if K not in HEADS:
        raise ValueError("heads=%d: the GATv2 kernels take 1, 2, 4 or 8 heads" % K)
    if f % K:
        raise ValueError("f=%d is not a multiple of heads=%d" % (f, K))
    if tuple(att.shape) != (K, f // K):
        raise ValueError("att must be [%d, %d], got %s" % (K, f // K, tuple(att.shape)))
    if not att.is_cuda or att.dtype != torch.float32:
        raise TypeError("att must be a float32 CUDA tensor")
    return K, att.detach().contiguous()


def _gatv2_edge_operands(plan, XL_own, XR_own, att, E, drop, what):
    """The walks, the transposed entries and the global ids, then XL_own and XR_own ([m, f] each, f <= 256 and
    f <= f_max), att ([K, f / K]) and E ([nnz_local, f]) checked and the plan bound, then the kernels loaded
    (pgcn_gatv2_edge_load). The tables come first, so that a capture that needs them before they exist is refused
    before any work is enqueued."""
    walks = plan.gated_walks()
    perm = plan.transposed_entries()
    gid = plan.global_ids()
    if drop is not None and drop.state.device != plan.device:
        raise ValueError("the EdgeDropout state lives on %s, the plan on %s" % (drop.state.device, plan.device))
    XL_own = _check_feat(plan, XL_own, plan.m, "XL")
    XR_own = _check_feat(plan, XR_own, plan.m, "XR")
    f = XL_own.shape[1]
    if XR_own.shape[1] != f:
        raise ValueError("XL and XR must have the same width, got %d and %d" % (f, XR_own.shape[1]))
    if f > GATV2_EDGE_MAX_F:
        raise ValueError("f=%d: the GATv2 edge kernels hold a row in registers, f <= %d" % (f, GATV2_EDGE_MAX_F))
    K, att = _gatv2_att(att, f)
    E = _check_edges(plan, E, f, "E")
    _require_bound(plan, "%s exchanges XL through pgcn_halo_rows" % what)
    with torch.cuda.device(plan.device):
        # every kernel loaded before the exchange: ranks of one process must not load one behind a waiting exchange
        cabi.check_gatv2_edge(cabi.load_gatv2_edge().pgcn_gatv2_edge_load())
    return walks, perm, gid, XL_own, XR_own, K, att, E


def aggregate_gatv2_edge(plan, XL_own, XR_own, att, E, negative_slope=0.2, drop=None):
    """(Z_own, L, XL_halo, snap): GATv2 attention with an edge term in the score over the plan's stored pattern
    (pgcn_gatv2_edge_forward). For every local entry e = (i, j), K = att.shape[0] heads of width d = f / K:
    t_e = (XR[i] + XL[j]) + E_e, s_eh = sum_c att[h, c] LeakyReLU(t_e[h d + c]), p = softmax of s over each row's stored
    entries per head, Z_own[i, h] = sum_e M_eh p_eh XL[j, h]. XL_own, XR_own and Z_own are [m, f], E [nnz_local, f] in
    edge_pairs() order, L [m, K] the rows' log-sum-exp. XL_halo [h, f] is XL's halo rows from one exchange
    (pgcn_halo_rows). drop (an EdgeDropout) with p > 0 draws a new counter (its snapshot `snap`, else None) and applies
    the mask M; aggregate_gatv2_edge_backward takes the same snapshot. E never crosses ranks. Needs a bound plan with
    f_max >= f."""
    drop = _active(drop)
    (fwd, _), _, gid, XL_own, XR_own, K, att, E = _gatv2_edge_operands(plan, XL_own, XR_own, att, E, drop,
                                                                       "aggregate_gatv2_edge")
    lp, f, dev = plan.lp, XL_own.shape[1], XL_own.device
    snap = drop.draw() if drop else None
    XL_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_halo_rows", XL_own.data_ptr(), XL_halo.data_ptr(), f, exchange=False)
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    L = torch.empty((lp.m, K), dtype=torch.float32, device=dev)
    work = torch.empty((fwd.nslots, f + 2 * K), dtype=torch.float32, device=dev)
    _gatv2_edge(dev, "pgcn_gatv2_edge_forward", C.byref(fwd.c), lp.m, lp.h, K, XL_own.data_ptr(), XL_halo.data_ptr(),
                XR_own.data_ptr(), att.data_ptr(), E.data_ptr(), float(negative_slope), gid.data_ptr(),
                *_drop_args(drop, snap), Z.data_ptr(), L.data_ptr(), work.data_ptr(), f)
    return Z, L, XL_halo, snap


def aggregate_gatv2_edge_backward(plan, XL_own, XL_halo, XR_own, att, E, Z_own, L, gZ_own, negative_slope=0.2,
                                  drop=None, snap=None, need_dE=True):
    """(dXL, dXR, datt, dE): the gradients of aggregate_gatv2_edge's Z_own for the output gradient gZ_own [m, f], from
    the same XL_own, XR_own, att, E and negative_slope, its XL_halo, Z_own and L and, with dropout, the same `drop` and
    its forward's `snap`. The row walk (pgcn_gatv2_edge_backward_rows) gives dXR, datt ([K, f / K]), each entry's
    g ([nnz_local, f], which is dE; None is returned when need_dE is false, and the buffer is scratch) and [P | ds]
    ([nnz_local, 2K]); the column walk over the transposed entries (pgcn_gatv2_edge_backward_cols) reads those and gives
    dXL, whose halo rows go back to their owners and are added there (pgcn_halo_rows_add)."""
    drop = _active(drop)
    if drop is not None and snap is None:
        raise ValueError("aggregate_gatv2_edge_backward with dropout needs the forward's snapshot")
    (fwd, tr), perm, gid, XL_own, XR_own, K, att, E = _gatv2_edge_operands(
        plan, XL_own, XR_own, att, E, drop, "aggregate_gatv2_edge_backward")
    lp, f, dev = plan.lp, XL_own.shape[1], XL_own.device
    gZ_own = _check_feat(plan, gZ_own, plan.m, "gZ")
    Z_own = _check_feat(plan, Z_own, plan.m, "Z")
    if gZ_own.shape[1] != f or Z_own.shape[1] != f:
        raise ValueError("XL, Z and gZ must have the same width, got %d, %d and %d" % (f, Z_own.shape[1],
                                                                                      gZ_own.shape[1]))
    XL_halo, L = XL_halo.contiguous(), L.contiguous()
    if tuple(XL_halo.shape) != (lp.h, f):
        raise ValueError("XL_halo must be [%d, %d], got %s" % (lp.h, f, tuple(XL_halo.shape)))
    if tuple(L.shape) != (lp.m, K):
        raise ValueError("L must be [%d, %d], got %s" % (lp.m, K, tuple(L.shape)))
    dXR = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    D = torch.empty((lp.m, K), dtype=torch.float32, device=dev)
    PS = torch.empty((lp.nnz(), 2 * K), dtype=torch.float32, device=dev)
    G = torch.empty((lp.nnz(), f), dtype=torch.float32, device=dev)
    datt = torch.empty((K, f // K), dtype=torch.float32, device=dev)
    work = torch.empty((cabi.load_gatv2_edge().pgcn_gatv2_edge_work_rows(C.byref(fwd.c)), f), dtype=torch.float32,
                       device=dev)
    _gatv2_edge(dev, "pgcn_gatv2_edge_backward_rows", C.byref(fwd.c), lp.m, lp.h, K, XL_own.data_ptr(),
                XL_halo.data_ptr(), XR_own.data_ptr(), att.data_ptr(), E.data_ptr(), float(negative_slope),
                gid.data_ptr(), *_drop_args(drop, snap), gZ_own.data_ptr(), Z_own.data_ptr(), L.data_ptr(),
                dXR.data_ptr(), D.data_ptr(), PS.data_ptr(), G.data_ptr(), datt.data_ptr(), work.data_ptr(), f)
    dXL = torch.empty((lp.m + lp.h, f), dtype=torch.float32, device=dev)
    work = torch.empty((tr.nslots, f), dtype=torch.float32, device=dev)
    _gatv2_edge(dev, "pgcn_gatv2_edge_backward_cols", C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, K,
                gZ_own.data_ptr(), PS.data_ptr(), G.data_ptr(), dXL.data_ptr(), work.data_ptr(), f)
    _call(plan, dev, "pgcn_halo_rows_add", dXL[lp.m:].data_ptr(), dXL.data_ptr(), f, exchange=True)
    return dXL[:lp.m], dXR, datt, G if need_dE else None


class PGATv2EdgeAttention(torch.autograd.Function):
    """PGATv2Attention with edge features in the score and attention dropout, the attention of PyG's
    GATv2Conv(edge_dim=..., dropout=p, concat=True, bias=False, add_self_loops=False) with XL = lin_l(x),
    XR = lin_r(x) and E = lin_edge(edge_attr) formed by the caller:

        PGATv2EdgeAttention.apply(A, XL, XR, att, E, negative_slope=0.2, dropout=None)
        t_e = (XR[i] + XL[j]) + E_e,  s_eh = sum_c att[h, c] * LeakyReLU(t_e[h d + c]),
        p_.h = softmax of s_.h over row i's stored entries,  out[i, h] = sum over the stored entries e = (i, j) of
        M_eh p_eh XL[j, h]

    XL, XR, att and out as PGATv2Attention's (K = att.shape[0] heads of width d = f / K, [rows, f] in the plan's layout;
    f <= 256). E is [nnz_local, f] in both layouts: one row per local entry in the order of PgcnPlan.edge_pairs(). It
    enters the score only and never crosses ranks, since every entry belongs to the rank that owns its row. Passing one
    tensor as XL and XR is share_weights=True. The values of A are not read; every stored entry contributes, duplicates
    included; a row without entries gives 0. One exchange per layer carries XL (f floats per row, so f_max >= f); the
    backward returns the halo rows' partial dXL to their owners in one reverse exchange. Only the rows' log-sum-exp
    ([rows, K]) is kept besides the operands: the backward recomputes the probabilities. Gradients go to XL, XR, att and
    E; dE is returned only when E requires it. Deterministic. The plan must be bound (PgcnPlan.bind_values); the first
    call builds its index tables (PgcnPlan.gated_walks, PgcnPlan.transposed_entries, PgcnPlan.global_ids).

    dropout (an op.EdgeDropout with p > 0): attention dropout on every head, the mask of op.edge_dropout drawn inline
    from the global (row, column) of each entry, as PTransformerAttention's. None or p == 0: no mask is drawn."""

    @staticmethod
    def forward(ctx, A, XL, XR, att, E, negative_slope=0.2, dropout=None):
        drop = _active(dropout)
        A.gated_walks()
        A.transposed_entries()
        A.global_ids()
        XL_own = _own(A, XL, "XL")
        XR_own = _own(A, XR, "XR")
        Z, L, XL_halo, snap = aggregate_gatv2_edge(A, XL_own, XR_own, att, E, negative_slope, drop)
        ctx.plan, ctx.slope, ctx.drop = A, float(negative_slope), drop
        ctx.save_for_backward(XL_own, XL_halo, XR_own, att.detach(), E.detach().contiguous(), Z, L, snap)
        return _to_layout(A, Z)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        XL_own, XL_halo, XR_own, att, E, Z, L, snap = ctx.saved_tensors
        dXL, dXR, datt, dE = aggregate_gatv2_edge_backward(A, XL_own, XL_halo, XR_own, att, E, Z, L,
                                                           _own(A, grad_output, "grad_output"), ctx.slope, ctx.drop,
                                                           snap, ctx.needs_input_grad[4])
        return None, _to_layout(A, dXL), _to_layout(A, dXR), datt, dE, None, None


# ---- the pieces, individually callable (NCCL transport), mirroring communicate_fgm ----------------

def spmm_local(plan, H_own, H_halo=None, transpose=False):
    """torch.sparse.mm(A, H) / torch.sparse.mm(A.t(), g) of GPU/PGCN.py:127,132 on the local matrix.
    transpose=False: returns Z [m, f].  transpose=True: returns (G_own [m, f], G_halo [h, f])."""
    lp = plan.lp
    H_own = _check_feat(plan, H_own, lp.m, "H_own")
    f = H_own.shape[1]
    dev = H_own.device
    if not transpose:
        if lp.h:
            H_halo = _check_feat(plan, H_halo, lp.h, "H_halo")
        Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        _call(plan, dev, "pgcn_spmm", 0, H_own.data_ptr(), H_halo.data_ptr() if lp.h else None, Z.data_ptr(), None, f)
        return Z
    G = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
    Gh = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
    _call(plan, dev, "pgcn_spmm", 1, H_own.data_ptr(), None, G.data_ptr(), Gh.data_ptr() if lp.h else None, f)
    return G, Gh


def spmm_split(plan, H_own, H_halo):
    """The overlapped forward's two kernels back to back: Z = A_own*H_own, then Z += A_halo*H_halo
    (Parallel-GCN/main.c:271,295). Same result as spmm_local up to fp32 summation order."""
    lp = plan.lp
    H_own = _check_feat(plan, H_own, lp.m, "H_own")
    H_halo = _check_feat(plan, H_halo, lp.h, "H_halo")
    f = H_own.shape[1]
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=H_own.device)
    _call(plan, H_own.device, "pgcn_spmm", 2, H_own.data_ptr(), None, Z.data_ptr(), None, f)
    _call(plan, H_own.device, "pgcn_spmm", 3, None, H_halo.data_ptr(), Z.data_ptr(), None, f)
    return Z


def pack_rows(plan, H_own):
    """send slab [S, f]: H[send_map[p]] for every peer p, concatenated in peer order (GPU/PGCN.py:104)."""
    H_own = _check_feat(plan, H_own, plan.lp.m, "H_own")
    f = H_own.shape[1]
    slab = torch.empty((plan.lp.S, f), dtype=torch.float32, device=H_own.device)
    _call(plan, H_own.device, "pgcn_pack", H_own.data_ptr(), slab.data_ptr(), f)
    return slab


def exchange_rows(plan, send_slab, backward=False):
    """The all-to-all-v of GPU/PGCN.py:99-115 (NCCL transport). Returns the received slab."""
    lp = plan.lp
    rows_out = lp.h if backward else lp.S
    rows_in = lp.S if backward else lp.h
    send_slab = _check_feat(plan, send_slab, rows_out, "send_slab")
    f = send_slab.shape[1]
    recv = torch.empty((rows_in, f), dtype=torch.float32, device=send_slab.device)
    _call(plan, send_slab.device, "pgcn_exchange", send_slab.data_ptr(), recv.data_ptr(), f, 1 if backward else 0,
          exchange=backward)
    return recv


def unpack_add(plan, recv_slab, G_own):
    """G_own[send_idx[j]] += recv_slab[j] for all j, fixed order (in place). Returns G_own."""
    recv_slab = _check_feat(plan, recv_slab, plan.lp.S, "recv_slab")
    if not G_own.is_contiguous():
        # in/out argument: a silent .contiguous() copy would accumulate into a temporary and leave G_own unchanged
        raise ValueError("G_own is updated in place and must be contiguous")
    G_own = _check_feat(plan, G_own, plan.lp.m, "G_own")
    _call(plan, G_own.device, "pgcn_unpack_add", recv_slab.data_ptr(), G_own.data_ptr(), G_own.shape[1])
    return G_own


def communicate_fgm(plan, H, backward=False):
    """The exchange of GPU/PGCN.py:85-119 in the compact layout.
    forward : H [m, f] -> halo rows [h, f] (what the reference scatters into X[recv_map]).
    backward: halo partials [h, f] -> contributions for my rows, summed, as a dense [m, f]."""
    if not backward:
        return exchange_rows(plan, pack_rows(plan, H), backward=False)
    recv = exchange_rows(plan, H, backward=True)
    G = torch.zeros((plan.lp.m, H.shape[1]), dtype=torch.float32, device=H.device)
    return unpack_add(plan, recv, G)
