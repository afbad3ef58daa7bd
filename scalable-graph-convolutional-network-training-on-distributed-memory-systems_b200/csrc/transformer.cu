// Graph transformer attention (include/pgcn_transformer.h): the fused scaled dot-product attention of TransformerConv
// and its two backward walks, over the gated aggregation's work tables.
//
// One warp per work item, a row (or a chunk of a long row) of the forward CSR, or a column of the transposed one, in
// the lane layout of transformer_math.cuh. Per entry the warp gathers one 2f-wide row (k and v in the forward and the
// row walk; q and gZ in the column walk). The forward keeps an online softmax (running max m, running sum l,
// accumulator rescaled when m grows) and saves only L = m + log l. A row walked whole is finished in its warp; the
// chunks of a split row write their partials to the caller's work rows and a fixup warp per split row merges them in
// chunk order. Every output element is therefore reduced in one fixed order, without atomics.
#include "../../include/pgcn_transformer.h"
#include "transformer_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

template <int W, bool VEC>
__global__ void __launch_bounds__(kTrThreads) transformer_walk_kernel(TrArgs a)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f, K = a.heads;
    const Lanes ln = lanes(lane, f, K);
    const Drop dr = drop_state(a);
    const int gr = dr.on ? __ldg(a.gid + r) : 0;
    // the item's own row: q[r] (and gZ[r] in the row walk), or k[r] and v[r] in the column walk
    float x[8], y[8];
    if constexpr (W == kTrCols) {
        const float* kv = kv_row(a, r);
        load8<VEC>(kv, ln, x);
        load8<VEC>(kv + f, ln, y);
    } else {
        load8<VEC>(a.Q + (size_t)r * f, ln, x);
        if constexpr (W == kTrRows) load8<VEC>(a.gZ + (size_t)r * f, ln, y);
    }
    float Lr = 0.0f, Dr = 0.0f;
    if constexpr (W == kTrRows) {
        Lr = __ldg(a.L + (size_t)r * K + ln.h);
        if (slot < 0) {
            // a row walked whole computes its D here; a split row's D came from transformer_delta_kernel
            float z[8];
            load8<VEC>(a.Z + (size_t)r * f, ln, z);
            Dr = head_dot(y, z, ln);
            if (ln.g == 0) a.aux[(size_t)r * K + ln.h] = Dr;
        } else {
            Dr = a.aux[(size_t)r * K + ln.h];
        }
    }
    Soft st{-INFINITY, 0.0f};
    float acc[8] = {}, acc2[8] = {};
    for (int eb = e0; eb < e1; eb += 32) {
        const int nb = min(32, e1 - eb);
        const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
        const int mine_g = dr.on && lane < nb ? __ldg(a.gid + mine) : 0;
#pragma unroll 2
        for (int k = 0; k < nb; ++k) {
            const int j = __shfl_sync(0xffffffffu, mine, k);
            const int gj = __shfl_sync(0xffffffffu, mine_g, k);
            float u[8], v[8];                // k[j], v[j] (forward, row walk) or q[j], gZ[j] (column walk)
            if constexpr (W == kTrCols) {
                load8<VEC>(a.Q + (size_t)j * f, ln, u);
                load8<VEC>(a.gZ + (size_t)j * f, ln, v);
            } else {
                const float* kv = kv_row(a, j);
                load8<VEC>(kv, ln, u);
                load8<VEC>(kv + f, ln, v);
            }
            const float s = __fmul_rn(head_dot(x, u, ln), a.scale);
            const float mk = W == kTrCols ? mask(dr, gj, gr, ln.h) : mask(dr, gr, gj, ln.h);
            if constexpr (W == kTrForward) {
                soft_add(st, acc, s, mk, v);
            } else if constexpr (W == kTrRows) {
                const float p = expf(__fsub_rn(s, Lr));
                const float ds = __fmul_rn(p, __fsub_rn(__fmul_rn(mk, head_dot(y, v, ln)), Dr));
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] = __fmaf_rn(ds, u[q], acc[q]);
            } else {
                const float p = expf(__fsub_rn(s, __ldg(a.L + (size_t)j * K + ln.h)));
                const float ds = __fmul_rn(p, __fsub_rn(__fmul_rn(mk, head_dot(y, v, ln)),
                                                         __ldg(a.Dc + (size_t)j * K + ln.h)));
                const float pm = __fmul_rn(p, mk);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    acc[q] = __fmaf_rn(ds, u[q], acc[q]);
                    acc2[q] = __fmaf_rn(pm, v[q], acc2[q]);
                }
            }
        }
    }
    if constexpr (W == kTrForward) {
        if (slot < 0) {
            finish_forward<VEC>(a, r, ln, st, acc);
        } else {
            // a chunk of a split row: [acc | m | l], merged by transformer_forward_fixup_kernel
            float* w = a.work + (size_t)slot * (f + 2 * K);
            store8<false>(w, ln, acc);
            if (ln.g == 0) {
                w[f + ln.h] = st.m;
                w[f + K + ln.h] = st.l;
            }
        }
    } else if (slot < 0) {
        finish_grad<W, VEC>(a, r, ln, acc, acc2);
    } else {
        const int ow = W == kTrCols ? 2 * f : f;
        store8<false>(a.work + (size_t)slot * ow, ln, acc);
        if constexpr (W == kTrCols) store8<false>(a.work + (size_t)slot * ow + f, ln, acc2);
    }
}

// The split-row kernels (transformer_math.cuh): the forward's merge in chunk order, the gradients' sums in chunk order,
// and D of the split rows before the row walk's chunks read it.
__global__ void __launch_bounds__(kTrThreads) transformer_forward_fixup_kernel(TrArgs a) { forward_fixup(a); }

template <int W>
__global__ void __launch_bounds__(kTrThreads) transformer_sum_fixup_kernel(TrArgs a) { sum_fixup<W>(a); }

__global__ void __launch_bounds__(kTrThreads) transformer_delta_kernel(TrArgs a) { delta(a); }

}  // namespace pgcn

using namespace pgcn;

namespace {

std::string g_error = "";

int fail(int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_error = buf;
    return code;
}

int check_walk(const pgcn_gated_walk* w, int64_t rows, const char* what)
{
    if (!w) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows,
                    (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Everything but the walk and the walk-specific operands: sizes, width, heads, the shared operands and the device.
int check_call(const char* what, const pgcn_gated_walk* w, int32_t m, int32_t h, int32_t heads, int32_t f,
               const float* Q, const float* KV, const float* KVh, float scale, const int32_t* gid,
               const int64_t* drop, float keep_scale, const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (heads != 1 && heads != 2 && heads != 4 && heads != 8)
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: heads=%d: the kernels take 1, 2, 4 or 8 heads", what, heads);
    if (f < 1 || f > kTrMaxF)
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: f=%d outside [1, %d]: a row lives in registers", what, f,
                    kTrMaxF);
    if (f % heads) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: f=%d is not a multiple of heads=%d", what, f, heads);
    if (!std::isfinite(scale)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: scale is not finite", what);
    if (m > 0 && (!Q || !KV)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null Q_own/KV_own", what);
    if (h > 0 && !KVh) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: h=%d but KV_halo is null", what, h);
    if (drop && m + h > 0 && !gid) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: drop without gid", what);
    if (drop && !std::isfinite(keep_scale))
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: keep_scale is not finite", what);
    if (w->nslots > 0 && !work)
        return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    return 0;
}

int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_TRANSFORMER_ERR_NOGPU, "no CUDA device (%s): transformer attention has no CPU path",
                    cudaGetErrorString(e));
    }
    return 0;
}

bool aligned16(std::initializer_list<const void*> ops)
{
    for (const void* q : ops)
        if (q && (reinterpret_cast<uintptr_t>(q) & 15)) return false;
    return true;
}

TrArgs make_args(const pgcn_gated_walk* w, int32_t m, int32_t heads, int32_t f, const float* Q, const float* KV,
                 const float* KVh, float scale, const int32_t* gid, const int64_t* drop, uint32_t threshold,
                 float keep_scale, float* work)
{
    TrArgs a{};
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits; a.m = m; a.f = f; a.heads = heads;
    a.Q = Q; a.KV = KV; a.KVh = KVh; a.scale = scale;
    a.gid = gid; a.drop = drop; a.threshold = threshold; a.keep_scale = keep_scale;
    a.work = work;
    return a;
}

unsigned warps_grid(int n) { return (unsigned)((n + kTrWarps - 1) / kTrWarps); }

int launched(const char* what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_TRANSFORMER_ERR_CUDA, "%s launch: %s", what, cudaGetErrorString(e));
    return PGCN_TRANSFORMER_OK;
}

// The walk, its vector instance when the head width and every feature operand allow it, then its fixup.
template <int W>
int launch(const TrArgs& a, std::initializer_list<const void*> feats, void* stream)
{
    if (a.nitems == 0) return PGCN_TRANSFORMER_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc;
    if (W == kTrRows && a.nsplits > 0) {
        transformer_delta_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
        if ((rc = launched("transformer_delta_kernel"))) return rc;
    }
    const bool vec = (a.f / a.heads) % 4 == 0 && aligned16(feats);
    if (vec) transformer_walk_kernel<W, true><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a);
    else transformer_walk_kernel<W, false><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a);
    if ((rc = launched("transformer_walk_kernel"))) return rc;
    if (a.nsplits > 0) {
        if (W == kTrForward) {
            transformer_forward_fixup_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
            return launched("transformer_forward_fixup_kernel");
        }
        transformer_sum_fixup_kernel<W == kTrForward ? kTrRows : W><<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
        return launched("transformer_sum_fixup_kernel");
    }
    return PGCN_TRANSFORMER_OK;
}

}  // namespace

extern "C" {

const char* pgcn_transformer_version(void)
{
    return "pgcn_transformer 0.1 (sm_90a, fused scaled dot-product graph attention with recomputed gradients)";
}

const char* pgcn_transformer_last_error(void) { return g_error.c_str(); }

int pgcn_transformer_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* Q_own,
                             const float* KV_own, const float* KV_halo, float scale, const int32_t* gid,
                             const int64_t* drop, uint32_t threshold, float keep_scale, float* Z, float* L, float* work,
                             int32_t f, void* stream)
{
    const char* what = "pgcn_transformer_forward";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_call(what, fwd, m, h, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, keep_scale, work)))
        return rc;
    if (m > 0 && (!Z || !L)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null Z/L output", what);
    if ((rc = check_device())) return rc;
    KV_halo = h > 0 ? KV_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, work);
    a.out = Z;
    a.aux = L;
    return launch<kTrForward>(a, {Q_own, KV_own, KV_halo, Z}, stream);
}

int pgcn_transformer_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                   const float* Q_own, const float* KV_own, const float* KV_halo, float scale,
                                   const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                   const float* gZ, const float* Z, const float* L, float* dQ, float* D, float* work,
                                   int32_t f, void* stream)
{
    const char* what = "pgcn_transformer_backward_rows";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_call(what, fwd, m, h, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, keep_scale, work)))
        return rc;
    if (m > 0 && (!gZ || !Z || !L)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null gZ/Z/L", what);
    if (m > 0 && (!dQ || !D)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null dQ/D output", what);
    if ((rc = check_device())) return rc;
    KV_halo = h > 0 ? KV_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, work);
    a.gZ = gZ; a.Z = Z; a.L = L;
    a.out = dQ;
    a.aux = D;
    return launch<kTrRows>(a, {Q_own, KV_own, KV_halo, gZ, Z, dQ}, stream);
}

int pgcn_transformer_backward_cols(const pgcn_gated_walk* tr, int32_t m, int32_t h, int32_t heads,
                                   const float* Q_own, const float* KV_own, const float* KV_halo, float scale,
                                   const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                   const float* gZ, const float* L, const float* D, float* dKV, float* work, int32_t f,
                                   void* stream)
{
    const char* what = "pgcn_transformer_backward_cols";
    int rc = check_walk(tr, (int64_t)m + h, what);
    if (rc || (rc = check_call(what, tr, m, h, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, keep_scale, work)))
        return rc;
    if (m > 0 && (!gZ || !L || !D)) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null gZ/L/D", what);
    if ((int64_t)m + h > 0 && !dKV) return fail(PGCN_TRANSFORMER_ERR_INVALID, "%s: null dKV output", what);
    if ((rc = check_device())) return rc;
    KV_halo = h > 0 ? KV_halo : nullptr;
    TrArgs a = make_args(tr, m, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, work);
    a.gZ = gZ; a.L = L; a.Dc = D;
    a.out = dKV;
    return launch<kTrCols>(a, {Q_own, KV_own, KV_halo, gZ, dKV}, stream);
}

}  // extern "C"
