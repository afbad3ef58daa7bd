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
"""
import torch

from . import cabi


def _stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def _check_feat(plan, H, rows, what):
    if not H.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the PGCN H100 path has no CPU fallback" % what)
    if H.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (what, H.dtype))
    if H.dim() != 2 or H.shape[0] != rows:
        raise ValueError("%s must be [%d, f], got %s" % (what, rows, tuple(H.shape)))
    if H.shape[1] > plan.f_max:
        raise ValueError("f=%d exceeds the plan's f_max=%d" % (H.shape[1], plan.f_max))
    return H.contiguous()


def aggregate_forward(plan, H_own, relu=False):
    """Z_own = (A * H)[owned rows]; H_own, Z_own are [m, f]. relu=True: Z_own = max(0, .), clamped inside the store of
    the launch that writes each row last (plan option "relu")."""
    H_own = _check_feat(plan, H_own, plan.m, "H")
    f = H_own.shape[1]
    Z = torch.empty((plan.m, f), dtype=torch.float32, device=H_own.device)
    lib = cabi.load()
    with torch.cuda.device(H_own.device):
        plan.use_values(None)             # PSpMM / PSpMMRelu aggregate with the plan's own values
        if relu:
            plan.set_option("relu", 1)
        try:
            cabi.check(lib.pgcn_forward(plan.handle, H_own.data_ptr(), Z.data_ptr(), f, _stream_ptr()), plan.handle)
        finally:
            if relu:
                plan.set_option("relu", 0)
    if plan.lp.k > 1:
        plan.count_exchange(backward=False)
    return Z


def aggregate_backward(plan, gZ_own):
    """G_own = (A^T * gZ)[owned rows] with every peer's contribution added; [m, f]."""
    gZ_own = _check_feat(plan, gZ_own, plan.m, "grad_output")
    f = gZ_own.shape[1]
    G = torch.empty((plan.m, f), dtype=torch.float32, device=gZ_own.device)
    lib = cabi.load()
    with torch.cuda.device(gZ_own.device):
        plan.use_values(None)
        cabi.check(lib.pgcn_backward(plan.handle, gZ_own.data_ptr(), G.data_ptr(), f, _stream_ptr()), plan.handle)
    if plan.lp.k > 1:
        plan.count_exchange(backward=True)
    return G


class PSpMM(torch.autograd.Function):
    """Same call shape as the reference operator: PSpMM.apply(A, H) (GPU/PGCN.py:145)."""

    @staticmethod
    def forward(ctx, A, H):
        ctx.plan = A
        if A.layout == "global":
            _check_feat(A, H, A.n, "H")
            Z_own = aggregate_forward(A, H.index_select(0, A.owned_index()))
            Z = torch.zeros((A.n, H.shape[1]), dtype=torch.float32, device=H.device)
            Z.index_copy_(0, A.owned_index(), Z_own)
            return Z
        return aggregate_forward(A, H)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        if A.layout == "global":
            g = _check_feat(A, grad_output, A.n, "grad_output")
            G_own = aggregate_backward(A, g.index_select(0, A.owned_index()))
            G = torch.zeros((A.n, g.shape[1]), dtype=torch.float32, device=g.device)
            G.index_copy_(0, A.owned_index(), G_own)
            return None, G
        return None, aggregate_backward(A, grad_output)


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
        ctx.glob = A.layout == "global"
        if ctx.glob:
            _check_feat(A, H, A.n, "H")
            H_own = H.index_select(0, A.owned_index())
        else:
            H_own = _check_feat(A, H, A.m, "H")
        lp = A.lp
        f = H_own.shape[1]
        want_dvals = ctx.needs_input_grad[1]
        keep = want_dvals and lp.k > 1 and lp.h > 0
        Z = torch.empty((lp.m, f), dtype=torch.float32, device=H_own.device)
        H_halo = torch.empty((lp.h, f), dtype=torch.float32, device=H_own.device) if keep else None
        lib = cabi.load()
        with torch.cuda.device(H_own.device):
            A.use_values(vals)
            if keep:
                cabi.check(lib.pgcn_forward_keep_halo(A.handle, H_own.data_ptr(), Z.data_ptr(), H_halo.data_ptr(), f,
                                                      _stream_ptr()), A.handle)
            else:
                cabi.check(lib.pgcn_forward(A.handle, H_own.data_ptr(), Z.data_ptr(), f, _stream_ptr()), A.handle)
        if lp.k > 1:
            A.count_exchange(backward=False)
        ctx.save_for_backward(vals, H_own if want_dvals else None, H_halo)
        if ctx.glob:
            Zg = torch.zeros((A.n, f), dtype=torch.float32, device=H.device)
            Zg.index_copy_(0, A.owned_index(), Z)
            return Zg
        return Z

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        vals, H_own, H_halo = ctx.saved_tensors
        if ctx.glob:
            g = _check_feat(A, grad_output, A.n, "grad_output").index_select(0, A.owned_index())
        else:
            g = _check_feat(A, grad_output, A.m, "grad_output")
        lp = A.lp
        f = g.shape[1]
        lib = cabi.load()
        dvals = dH = None
        with torch.cuda.device(g.device):
            if ctx.needs_input_grad[2]:
                A.use_values(vals)
                G = torch.empty((lp.m, f), dtype=torch.float32, device=g.device)
                cabi.check(lib.pgcn_backward(A.handle, g.data_ptr(), G.data_ptr(), f, _stream_ptr()), A.handle)
                if lp.k > 1:
                    A.count_exchange(backward=True)
                if ctx.glob:
                    dH = torch.zeros((A.n, f), dtype=torch.float32, device=g.device)
                    dH.index_copy_(0, A.owned_index(), G)
                else:
                    dH = G
            if ctx.needs_input_grad[1]:
                dvals = torch.empty((lp.nnz(),), dtype=torch.float32, device=g.device)
                cabi.check(lib.pgcn_sddmm(A.handle, g.data_ptr(), H_own.data_ptr(),
                                          H_halo.data_ptr() if H_halo is not None else None, dvals.data_ptr(), f,
                                          _stream_ptr()), A.handle)
        return None, dvals, dH


def _check_scores(plan, x, rows, what):
    if not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the PGCN H100 path has no CPU fallback" % what)
    if x.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (what, x.dtype))
    if x.dim() != 1 or x.shape[0] != rows:
        raise ValueError("%s must be [%d], got %s" % (what, rows, tuple(x.shape)))
    x = x.detach()
    return (x.index_select(0, plan.owned_index()) if plan.layout == "global" else x).contiguous()


def _to_layout(plan, x_own, rows):
    if plan.layout != "global":
        return x_own
    out = torch.zeros((rows,) + tuple(x_own.shape[1:]), dtype=torch.float32, device=x_own.device)
    out.index_copy_(0, plan.owned_index(), x_own)
    return out


class PGATAttention(torch.autograd.Function):
    """Single-head sparse graph attention over the plan's stored pattern (GPU/PGAT.py:139-148 without the dense n x n
    score matrix):

        PGATAttention.apply(A, Z, el, er, negative_slope)
        s_e = LeakyReLU(el[row(e)] + er[col(e)]),  alpha = softmax of s over each row's stored entries,  out = A(alpha) Z

    Z is [rows, f], el and er are [rows] fp32 CUDA tensors (rows = m in the "local" layout, n in the "global" one, whose
    non-owned rows are ignored and come back zero), out is [rows, f]. er of the halo columns comes from their owners
    (pgcn_halo_rows, padded to rows of 4 floats so that the peer transport carries it). Forward: the edge softmax kernel
    writes alpha, which becomes the resident values of A for pgcn_forward_keep_halo(Z). Backward: dZ = A(alpha)^T gOut
    with the exchange; dalpha = SDDMM(gOut, [Z_own; Z_halo]); the softmax backward kernel gives dpre and d_el; and
    d_er = A(dpre)^T 1, the column sums of dpre with the halo partials summed at their owners (pgcn_backward on an
    m x 4 matrix of ones). Everything is deterministic. Gradients to W and a flow through torch, since el and er are
    computed outside. The plan must be bound (PgcnPlan.bind_values); a later PSpMM on it restores the creation values."""

    @staticmethod
    def forward(ctx, A, Z, el, er, negative_slope=0.2):
        rows = A.n if A.layout == "global" else A.m
        Z_own = _check_feat(A, Z, rows, "Z")
        if A.layout == "global":
            Z_own = Z_own.index_select(0, A.owned_index())
        el_own = _check_scores(A, el, rows, "el")
        er_own = _check_scores(A, er, rows, "er")
        lp = A.lp
        f = Z_own.shape[1]
        dev = Z_own.device
        slope = float(negative_slope)
        lib = cabi.load()
        with torch.cuda.device(dev):
            if not A._bound:
                raise RuntimeError("PGATAttention sets the plan's edge values: call PgcnPlan.bind_values() once (set-up, "
                                   "before any CUDA-graph capture)")
            er_halo = torch.empty((lp.h,), dtype=torch.float32, device=dev)
            if lp.k > 1:
                er4 = torch.zeros((lp.m, 4), dtype=torch.float32, device=dev)
                er4[:, 0] = er_own
                er_halo4 = torch.empty((lp.h, 4), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_halo_rows(A.handle, er4.data_ptr(), er_halo4.data_ptr(), 4, _stream_ptr()),
                           A.handle)
                A.count_exchange(backward=False)
                er_halo = er_halo4[:, 0].contiguous()
            alpha = torch.empty((lp.nnz(),), dtype=torch.float32, device=dev)
            cabi.check(lib.pgcn_edge_softmax(A.handle, el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(), slope,
                                             alpha.data_ptr(), _stream_ptr()), A.handle)
            out = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            Z_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
            A.use_values(alpha)
            if lp.k > 1 and lp.h > 0:
                cabi.check(lib.pgcn_forward_keep_halo(A.handle, Z_own.data_ptr(), out.data_ptr(), Z_halo.data_ptr(), f,
                                                      _stream_ptr()), A.handle)
            else:
                cabi.check(lib.pgcn_forward(A.handle, Z_own.data_ptr(), out.data_ptr(), f, _stream_ptr()), A.handle)
            if lp.k > 1:
                A.count_exchange(backward=False)
        ctx.plan, ctx.rows, ctx.slope = A, rows, slope
        ctx.save_for_backward(alpha, Z_own, Z_halo, el_own, er_own, er_halo)
        return _to_layout(A, out, rows)

    @staticmethod
    def backward(ctx, grad_output):
        A, rows, slope = ctx.plan, ctx.rows, ctx.slope
        alpha, Z_own, Z_halo, el_own, er_own, er_halo = ctx.saved_tensors
        g = _check_feat(A, grad_output, rows, "grad_output")
        if A.layout == "global":
            g = g.index_select(0, A.owned_index())
        lp = A.lp
        f = g.shape[1]
        dev = g.device
        lib = cabi.load()
        dZ = d_el = d_er = None
        with torch.cuda.device(dev):
            if ctx.needs_input_grad[1]:
                A.use_values(alpha)
                G = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_backward(A.handle, g.data_ptr(), G.data_ptr(), f, _stream_ptr()), A.handle)
                if lp.k > 1:
                    A.count_exchange(backward=True)
                dZ = _to_layout(A, G, rows)
            if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
                dalpha = torch.empty_like(alpha)
                cabi.check(lib.pgcn_sddmm(A.handle, g.data_ptr(), Z_own.data_ptr(), Z_halo.data_ptr(),
                                          dalpha.data_ptr(), f, _stream_ptr()), A.handle)
                dpre = torch.empty_like(alpha)
                gel = torch.empty((lp.m,), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_edge_softmax_backward(A.handle, el_own.data_ptr(), er_own.data_ptr(),
                                                          er_halo.data_ptr(), alpha.data_ptr(), dalpha.data_ptr(),
                                                          slope, dpre.data_ptr(), gel.data_ptr(), _stream_ptr()),
                           A.handle)
                d_el = _to_layout(A, gel, rows) if ctx.needs_input_grad[2] else None
                if ctx.needs_input_grad[3]:
                    A.use_values(dpre)
                    ones = torch.ones((lp.m, 4), dtype=torch.float32, device=dev)
                    D = torch.empty((lp.m, 4), dtype=torch.float32, device=dev)
                    cabi.check(lib.pgcn_backward(A.handle, ones.data_ptr(), D.data_ptr(), 4, _stream_ptr()), A.handle)
                    if lp.k > 1:
                        A.count_exchange(backward=True)
                    d_er = _to_layout(A, D[:, 0].contiguous(), rows)
        return None, dZ, d_el, d_er, None


HEADS = (1, 2, 4, 8)


def _check_head_scores(plan, x, rows, heads, what):
    if not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the PGCN H100 path has no CPU fallback" % what)
    if x.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (what, x.dtype))
    if x.dim() != 2 or x.shape[0] != rows or x.shape[1] != heads:
        raise ValueError("%s must be [%d, %d], got %s" % (what, rows, heads, tuple(x.shape)))
    x = x.detach()
    return (x.index_select(0, plan.owned_index()) if plan.layout == "global" else x).contiguous()


class PGATMultiHeadAttention(torch.autograd.Function):
    """Multi-head sparse graph attention over the plan's stored pattern: K = el.shape[1] heads (1, 2, 4 or 8) of width
    d = f / K, concatenated.

        PGATMultiHeadAttention.apply(A, Z, el, er, negative_slope)
        s_eh = LeakyReLU(el[row(e), h] + er[col(e), h]),  alpha_.h = softmax of s_.h over each row's stored entries,
        out[:, h d:(h+1) d] = A(alpha[:, h]) Z[:, h d:(h+1) d]

    Z is [rows, f], el and er are [rows, K] fp32 CUDA tensors, out is [rows, f] (rows = m in the "local" layout, n in the
    "global" one, as PGATAttention). One exchange per layer carries the f-wide Z for every head, and er of the halo
    columns travels once for all heads (pgcn_halo_rows, rows padded to a multiple of 4 floats). The kernels take alpha
    ([nnz, K]) as an argument, so the plan's resident values are never rewritten: a PSpMM on the same plan needs no
    restore. Backward: dZ = A(alpha)^T gOut per head (pgcn_backward_heads), dalpha from pgcn_sddmm_heads, dpre and d_el
    from the softmax backward, d_er[:, h] = A(dpre[:, h])^T 1 (pgcn_backward_heads on an m x 4K matrix of ones, column
    4h), so the plan's f_max must be at least max(f, 4K). Deterministic. The exchange is the unsplit one (no per-source
    overlap). The plan must be bound (PgcnPlan.bind_values)."""

    @staticmethod
    def forward(ctx, A, Z, el, er, negative_slope=0.2):
        rows = A.n if A.layout == "global" else A.m
        if el.dim() != 2:
            raise ValueError("el must be [%d, heads], got %s" % (rows, tuple(el.shape)))
        K = el.shape[1]
        if K not in HEADS:
            raise ValueError("heads=%d: the multi-head kernels take 1, 2, 4 or 8 heads" % K)
        Z_own = _check_feat(A, Z, rows, "Z")
        f = Z_own.shape[1]
        if f % K:
            raise ValueError("f=%d is not a multiple of heads=%d" % (f, K))
        if A.f_max < 4 * K:
            raise ValueError("heads=%d: the backward aggregates rows of 4 x heads = %d floats, the plan's f_max is %d"
                             % (K, 4 * K, A.f_max))
        if A.layout == "global":
            Z_own = Z_own.index_select(0, A.owned_index())
        el_own = _check_head_scores(A, el, rows, K, "el")
        er_own = _check_head_scores(A, er, rows, K, "er")
        lp = A.lp
        dev = Z_own.device
        slope = float(negative_slope)
        lib = cabi.load()
        with torch.cuda.device(dev):
            if not A._bound:
                raise RuntimeError("PGATMultiHeadAttention reads the plan's value maps: call PgcnPlan.bind_values() once "
                                   "(set-up, before any CUDA-graph capture)")
            er_halo = torch.empty((lp.h, K), dtype=torch.float32, device=dev)
            if lp.k > 1:
                w = (K + 3) // 4 * 4
                erw = torch.zeros((lp.m, w), dtype=torch.float32, device=dev)
                erw[:, :K] = er_own
                er_halo_w = torch.empty((lp.h, w), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_halo_rows(A.handle, erw.data_ptr(), er_halo_w.data_ptr(), w, _stream_ptr()),
                           A.handle)
                A.count_exchange(backward=False)
                er_halo = er_halo_w[:, :K].contiguous()
            alpha = torch.empty((lp.nnz(), K), dtype=torch.float32, device=dev)
            cabi.check(lib.pgcn_edge_softmax_heads(A.handle, K, el_own.data_ptr(), er_own.data_ptr(), er_halo.data_ptr(),
                                                   slope, alpha.data_ptr(), _stream_ptr()), A.handle)
            out = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            Z_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
            keep = lp.k > 1 and lp.h > 0
            cabi.check(lib.pgcn_forward_heads(A.handle, K, alpha.data_ptr(), Z_own.data_ptr(), out.data_ptr(),
                                              Z_halo.data_ptr() if keep else None, f, _stream_ptr()), A.handle)
            if lp.k > 1:
                A.count_exchange(backward=False)
        ctx.plan, ctx.rows, ctx.slope, ctx.heads = A, rows, slope, K
        ctx.save_for_backward(alpha, Z_own, Z_halo, el_own, er_own, er_halo)
        return _to_layout(A, out, rows)

    @staticmethod
    def backward(ctx, grad_output):
        A, rows, slope, K = ctx.plan, ctx.rows, ctx.slope, ctx.heads
        alpha, Z_own, Z_halo, el_own, er_own, er_halo = ctx.saved_tensors
        g = _check_feat(A, grad_output, rows, "grad_output")
        if A.layout == "global":
            g = g.index_select(0, A.owned_index())
        lp = A.lp
        f = g.shape[1]
        dev = g.device
        lib = cabi.load()
        dZ = d_el = d_er = None
        with torch.cuda.device(dev):
            if ctx.needs_input_grad[1]:
                G = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_backward_heads(A.handle, K, alpha.data_ptr(), g.data_ptr(), G.data_ptr(), f,
                                                   _stream_ptr()), A.handle)
                if lp.k > 1:
                    A.count_exchange(backward=True)
                dZ = _to_layout(A, G, rows)
            if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
                dalpha = torch.empty_like(alpha)
                cabi.check(lib.pgcn_sddmm_heads(A.handle, K, g.data_ptr(), Z_own.data_ptr(), Z_halo.data_ptr(),
                                                dalpha.data_ptr(), f, _stream_ptr()), A.handle)
                dpre = torch.empty_like(alpha)
                gel = torch.empty((lp.m, K), dtype=torch.float32, device=dev)
                cabi.check(lib.pgcn_edge_softmax_backward_heads(A.handle, K, el_own.data_ptr(), er_own.data_ptr(),
                                                                er_halo.data_ptr(), alpha.data_ptr(), dalpha.data_ptr(),
                                                                slope, dpre.data_ptr(), gel.data_ptr(), _stream_ptr()),
                           A.handle)
                d_el = _to_layout(A, gel, rows) if ctx.needs_input_grad[2] else None
                if ctx.needs_input_grad[3]:
                    ones = torch.ones((lp.m, 4 * K), dtype=torch.float32, device=dev)
                    D = torch.empty((lp.m, 4 * K), dtype=torch.float32, device=dev)
                    cabi.check(lib.pgcn_backward_heads(A.handle, K, dpre.data_ptr(), ones.data_ptr(), D.data_ptr(),
                                                       4 * K, _stream_ptr()), A.handle)
                    if lp.k > 1:
                        A.count_exchange(backward=True)
                    d_er = _to_layout(A, D[:, 0::4].contiguous(), rows)
        return None, dZ, d_el, d_er, None


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
        rows = A.n if A.layout == "global" else A.m
        if att.dim() != 2:
            raise ValueError("att must be [heads, f / heads], got %s" % (tuple(att.shape),))
        K = att.shape[0]
        if K not in HEADS:
            raise ValueError("heads=%d: the GATv2 kernels take 1, 2, 4 or 8 heads" % K)
        XL_own = _check_feat(A, XL, rows, "XL")
        XR_own = _check_feat(A, XR, rows, "XR")
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
        if A.layout == "global":
            XL_own = XL_own.index_select(0, A.owned_index())
            XR_own = XR_own.index_select(0, A.owned_index())
        lp = A.lp
        dev = XL_own.device
        slope = float(negative_slope)
        lib = cabi.load()
        with torch.cuda.device(dev):
            if not A._bound:
                raise RuntimeError("PGATv2Attention reads the plan's value maps: call PgcnPlan.bind_values() once "
                                   "(set-up, before any CUDA-graph capture)")
            alpha = torch.empty((lp.nnz(), K), dtype=torch.float32, device=dev)
            out = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            XL_halo = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
            keep = lp.k > 1 and lp.h > 0
            cabi.check(lib.pgcn_forward_gatv2(A.handle, K, XL_own.data_ptr(), XR_own.data_ptr(), att_c.data_ptr(),
                                              slope, alpha.data_ptr(), out.data_ptr(),
                                              XL_halo.data_ptr() if keep else None, f, _stream_ptr()), A.handle)
            if lp.k > 1:
                A.count_exchange(backward=False)
        ctx.plan, ctx.rows, ctx.slope, ctx.heads = A, rows, slope, K
        ctx.save_for_backward(alpha, XL_own, XL_halo, XR_own, att_c)
        return _to_layout(A, out, rows)

    @staticmethod
    def backward(ctx, grad_output):
        A, rows, slope, K = ctx.plan, ctx.rows, ctx.slope, ctx.heads
        alpha, XL_own, XL_halo, XR_own, att = ctx.saved_tensors
        g = _check_feat(A, grad_output, rows, "grad_output")
        if A.layout == "global":
            g = g.index_select(0, A.owned_index())
        lp = A.lp
        f = g.shape[1]
        dev = g.device
        with torch.cuda.device(dev):
            work = torch.empty_like(alpha)
            dxl = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            dxr = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            datt = torch.empty_like(att)
            cabi.check(cabi.load().pgcn_backward_gatv2(
                A.handle, K, alpha.data_ptr(), g.data_ptr(), XL_own.data_ptr(), XL_halo.data_ptr() if lp.h else None,
                XR_own.data_ptr(), att.data_ptr(), slope, work.data_ptr(), dxl.data_ptr(), dxr.data_ptr(),
                datt.data_ptr(), f, _stream_ptr()), A.handle)
            if lp.k > 1:
                A.count_exchange(backward=True)
        return None, _to_layout(A, dxl, rows), _to_layout(A, dxr, rows), datt, None


# ---- max aggregation -------------------------------------------------------------------------------------------------

def _check_max_plan(plan, what):
    if not plan._bound:
        raise RuntimeError("%s walks the transposed records through the plan's value maps: call PgcnPlan.bind_values() "
                           "once (set-up, before any CUDA-graph capture)" % what)


def aggregate_max(plan, H_own):
    """(Z_own, arg): the element-wise maximum over each owned row's stored entries of [H_own ; H_halo] (pgcn_forward_max).
    Z_own is [m, f] fp32, arg [m, f] int32: the winning entry, the first in forward CSR order (lp.colidx's order) with
    the largest value, NaN above every number; lp.colidx[arg] is its local column. Rows without an entry give 0 / -1."""
    H_own = _check_feat(plan, H_own, plan.m, "H")
    _check_max_plan(plan, "aggregate_max")
    f = H_own.shape[1]
    Z = torch.empty((plan.m, f), dtype=torch.float32, device=H_own.device)
    arg = torch.empty((plan.m, f), dtype=torch.int32, device=H_own.device)
    with torch.cuda.device(H_own.device):
        cabi.check(cabi.load().pgcn_forward_max(plan.handle, H_own.data_ptr(), Z.data_ptr(), arg.data_ptr(), f,
                                                _stream_ptr()), plan.handle)
    if plan.lp.k > 1:
        plan.count_exchange(backward=False)
    return Z, arg


def aggregate_max_backward(plan, arg, gZ_own):
    """G_own [m, f]: gZ routed to the winning entries named by `arg` (aggregate_max's), summed per column on its owner
    (pgcn_backward_max)."""
    gZ_own = _check_feat(plan, gZ_own, plan.m, "grad_output")
    _check_max_plan(plan, "aggregate_max_backward")
    f = gZ_own.shape[1]
    if arg.dtype != torch.int32 or arg.device != gZ_own.device or tuple(arg.shape) != (plan.m, f):
        raise ValueError("arg must be int32 [%d, %d] on %s, got %s %s on %s"
                         % (plan.m, f, gZ_own.device, arg.dtype, tuple(arg.shape), arg.device))
    arg = arg.contiguous()
    G = torch.empty((plan.m, f), dtype=torch.float32, device=gZ_own.device)
    with torch.cuda.device(gZ_own.device):
        cabi.check(cabi.load().pgcn_backward_max(plan.handle, arg.data_ptr(), gZ_own.data_ptr(), G.data_ptr(), f,
                                                 _stream_ptr()), plan.handle)
    if plan.lp.k > 1:
        plan.count_exchange(backward=True)
    return G


class PSpMMMax(torch.autograd.Function):
    """Z = max over each row's neighbours, element-wise (the GraphSAGE "pool" aggregator, PyG aggr="max"), with the call
    shape of PSpMM: PSpMMMax.apply(A, H). The pattern of A is used, not its values. The gradient goes to the winning
    entry of every (row, feature), the first one on ties (aggregate_max), including winners in other ranks' rows.
    Layouts as PSpMM. The plan must be bound (PgcnPlan.bind_values)."""

    @staticmethod
    def forward(ctx, A, H):
        ctx.plan = A
        _check_max_plan(A, "PSpMMMax")
        if A.layout == "global":
            _check_feat(A, H, A.n, "H")
            Z_own, arg = aggregate_max(A, H.index_select(0, A.owned_index()))
        else:
            Z_own, arg = aggregate_max(A, H)
        ctx.save_for_backward(arg)
        return _to_layout(A, Z_own, A.n)

    @staticmethod
    def backward(ctx, grad_output):
        A = ctx.plan
        (arg,) = ctx.saved_tensors
        if A.layout == "global":
            g = _check_feat(A, grad_output, A.n, "grad_output").index_select(0, A.owned_index())
            return None, _to_layout(A, aggregate_max_backward(A, arg, g), A.n)
        return None, aggregate_max_backward(A, arg, grad_output)


# ---- the pieces, individually callable (NCCL transport), mirroring communicate_fgm ----------------

def spmm_local(plan, H_own, H_halo=None, transpose=False):
    """torch.sparse.mm(A, H) / torch.sparse.mm(A.t(), g) of GPU/PGCN.py:127,132 on the local matrix.
    transpose=False: returns Z [m, f].  transpose=True: returns (G_own [m, f], G_halo [h, f])."""
    lp = plan.lp
    H_own = _check_feat(plan, H_own, lp.m, "H_own")
    f = H_own.shape[1]
    dev = H_own.device
    lib = cabi.load()
    with torch.cuda.device(dev):
        if not transpose:
            if lp.h:
                H_halo = _check_feat(plan, H_halo, lp.h, "H_halo")
            Z = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
            cabi.check(lib.pgcn_spmm(plan.handle, 0, H_own.data_ptr(), H_halo.data_ptr() if lp.h else None,
                                     Z.data_ptr(), None, f, _stream_ptr()), plan.handle)
            return Z
        G = torch.empty((lp.m, f), dtype=torch.float32, device=dev)
        Gh = torch.empty((lp.h, f), dtype=torch.float32, device=dev)
        cabi.check(lib.pgcn_spmm(plan.handle, 1, H_own.data_ptr(), None, G.data_ptr(),
                                 Gh.data_ptr() if lp.h else None, f, _stream_ptr()), plan.handle)
        return G, Gh


def spmm_split(plan, H_own, H_halo):
    """The overlapped forward's two kernels back to back: Z = A_own*H_own, then Z += A_halo*H_halo
    (Parallel-GCN/main.c:271,295). Same result as spmm_local up to fp32 summation order."""
    lp = plan.lp
    H_own = _check_feat(plan, H_own, lp.m, "H_own")
    H_halo = _check_feat(plan, H_halo, lp.h, "H_halo")
    f = H_own.shape[1]
    Z = torch.empty((lp.m, f), dtype=torch.float32, device=H_own.device)
    lib = cabi.load()
    with torch.cuda.device(H_own.device):
        cabi.check(lib.pgcn_spmm(plan.handle, 2, H_own.data_ptr(), None, Z.data_ptr(), None, f, _stream_ptr()), plan.handle)
        cabi.check(lib.pgcn_spmm(plan.handle, 3, None, H_halo.data_ptr(), Z.data_ptr(), None, f, _stream_ptr()), plan.handle)
    return Z


def pack_rows(plan, H_own):
    """send slab [S, f]: H[send_map[p]] for every peer p, concatenated in peer order (GPU/PGCN.py:104)."""
    H_own = _check_feat(plan, H_own, plan.lp.m, "H_own")
    f = H_own.shape[1]
    slab = torch.empty((plan.lp.S, f), dtype=torch.float32, device=H_own.device)
    with torch.cuda.device(H_own.device):
        cabi.check(cabi.load().pgcn_pack(plan.handle, H_own.data_ptr(), slab.data_ptr(), f, _stream_ptr()), plan.handle)
    return slab


def exchange_rows(plan, send_slab, backward=False):
    """The all-to-all-v of GPU/PGCN.py:99-115 (NCCL transport). Returns the received slab."""
    lp = plan.lp
    rows_out = lp.h if backward else lp.S
    rows_in = lp.S if backward else lp.h
    send_slab = _check_feat(plan, send_slab, rows_out, "send_slab")
    f = send_slab.shape[1]
    recv = torch.empty((rows_in, f), dtype=torch.float32, device=send_slab.device)
    with torch.cuda.device(send_slab.device):
        cabi.check(cabi.load().pgcn_exchange(plan.handle, send_slab.data_ptr(), recv.data_ptr(), f,
                                             1 if backward else 0, _stream_ptr()), plan.handle)
    plan.count_exchange(backward=backward)
    return recv


def unpack_add(plan, recv_slab, G_own):
    """G_own[send_idx[j]] += recv_slab[j] for all j, fixed order (in place). Returns G_own."""
    recv_slab = _check_feat(plan, recv_slab, plan.lp.S, "recv_slab")
    if not G_own.is_contiguous():
        # in/out argument: a silent .contiguous() copy would accumulate into a temporary and leave G_own unchanged
        raise ValueError("G_own is updated in place and must be contiguous")
    G_own = _check_feat(plan, G_own, plan.lp.m, "G_own")
    with torch.cuda.device(G_own.device):
        cabi.check(cabi.load().pgcn_unpack_add(plan.handle, recv_slab.data_ptr(), G_own.data_ptr(),
                                               G_own.shape[1], _stream_ptr()), plan.handle)
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
