// Gated aggregation (include/pgcn_gated.h): the sigmoid-gated SpMM of ResGatedGraphConv and its two backward walks.
//
// One warp per work item, a row of at most kGatedChunk entries or one chunk of a longer row. The warp walks the item's
// entries in CSR order, 128 features per pass (4 per lane), and keeps per-feature sums in registers: per entry it
// gathers one 2 x 128-float slice (Q and V rows in the forward and row walks, K and gZ rows in the column walk) and
// recomputes the gate. Nothing is stored per entry. A row walked whole is finished in the same warp; the chunks of a
// split row write their partial sums to the caller's work rows, and a fixup warp per split row adds them in chunk order
// and finishes the row. Every output element is therefore one sum in a fixed order, without atomics.
#include "../../include/pgcn_gated.h"
#include "gated_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

constexpr int kGatedChunk = 512;         // entries per work item
constexpr int kGatedThreads = 256;
constexpr int kGatedWarps = kGatedThreads / 32;
constexpr int kTile = 128;               // features per pass of a warp

enum GatedWalk : int { kForward = 0, kRows = 1, kCols = 2 };

struct GatedArgs {
    const int4* items;
    const int32_t* splits;     // nsplits x 3
    const int32_t* idx;
    int nitems, nsplits, m, f;
    const float* K;            // m x f
    const float* QV;           // m x 2f
    const float* QVh;          // h x 2f
    const float* gZ;           // m x f (backward walks)
    float* out;                // m x f, or (m + h) x 2f for the column walk
    float* work;               // nslots x (f or 2f)
};

__device__ __forceinline__ const float* qv_row(const GatedArgs& a, int j)
{
    return j < a.m ? a.QV + (size_t)j * 2 * a.f : a.QVh + (size_t)(j - a.m) * 2 * a.f;
}

// Finish row r from its sums: forward Z = s0; row walk dK = gZ[r] * s0; column walk dQ = V[r] * s0, dV = s1.
template <int W, bool VEC>
__device__ __forceinline__ void finish(const GatedArgs& a, int r, int t0, int lane, float (&s)[2][4])
{
    const int f = a.f;
    if constexpr (W == kForward) {
        store4<VEC>(a.out + (size_t)r * f, t0, lane, f, s[0]);
    } else {
        float g[4], o[4];
        load4<VEC>(W == kRows ? a.gZ + (size_t)r * f : qv_row(a, r) + f, t0, lane, f, g);
#pragma unroll
        for (int u = 0; u < 4; ++u) o[u] = __fmul_rn(g[u], s[0][u]);
        if constexpr (W == kRows) {
            store4<VEC>(a.out + (size_t)r * f, t0, lane, f, o);
        } else {
            store4<VEC>(a.out + (size_t)r * 2 * f, t0, lane, f, o);
            store4<VEC>(a.out + (size_t)r * 2 * f + f, t0, lane, f, s[1]);
        }
    }
}

template <int W, bool VEC>
__global__ void __launch_bounds__(kGatedThreads) gated_walk_kernel(GatedArgs a)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kGatedWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f;
    // the row's own operand: K[r] (forward, row walk) or Q[r] (column walk)
    const float* fixed = W == kCols ? qv_row(a, r) : a.K + (size_t)r * f;
    for (int t0 = 0; t0 < f; t0 += kTile) {
        float fx[4], s[2][4] = {};
        load4<VEC>(fixed, t0, lane, f, fx);
        for (int eb = e0; eb < e1; eb += 32) {
            const int nb = min(32, e1 - eb);
            const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
#pragma unroll 4
            for (int k = 0; k < nb; ++k) {
                const int j = __shfl_sync(0xffffffffu, mine, k);
                float x[4], y[4];            // Q[j], V[j] (forward, row walk) or K[j], gZ[j] (column walk)
                if constexpr (W == kCols) {
                    load4<VEC>(a.K + (size_t)j * f, t0, lane, f, x);
                    load4<VEC>(a.gZ + (size_t)j * f, t0, lane, f, y);
                } else {
                    const float* q = qv_row(a, j);
                    load4<VEC>(q, t0, lane, f, x);
                    load4<VEC>(q + f, t0, lane, f, y);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float ds;
                    const float eta = gate(__fadd_rn(fx[u], x[u]), ds);
                    if constexpr (W == kForward) {
                        s[0][u] = __fmaf_rn(eta, y[u], s[0][u]);
                    } else {
                        s[0][u] = __fmaf_rn(y[u], ds, s[0][u]);
                        if constexpr (W == kCols) s[1][u] = __fmaf_rn(eta, y[u], s[1][u]);
                    }
                }
            }
        }
        if (slot < 0) {
            finish<W, VEC>(a, r, t0, lane, s);
        } else {
            // a chunk of a split row: its raw sums, [s0] or [s0 | s1], finished by the fixup
            const int ow = W == kCols ? 2 * f : f;
            store4<VEC>(a.work + (size_t)slot * ow, t0, lane, f, s[0]);
            if constexpr (W == kCols) store4<VEC>(a.work + (size_t)slot * ow + f, t0, lane, f, s[1]);
        }
    }
}

// One warp per split row (row, slot0, count): the chunks' partial sums added in chunk order, then the row finished.
template <int W>
__global__ void __launch_bounds__(kGatedThreads) gated_fixup_kernel(GatedArgs a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kGatedWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f, ow = W == kCols ? 2 * f : f;
    for (int t0 = 0; t0 < f; t0 += kTile) {
        float s[2][4] = {};
        for (int q = 0; q < n; ++q) {
            const float* p = a.work + (size_t)(slot0 + q) * ow;
            float v[4];
            load4<false>(p, t0, lane, f, v);
#pragma unroll
            for (int u = 0; u < 4; ++u) s[0][u] = __fadd_rn(s[0][u], v[u]);
            if constexpr (W == kCols) {
                load4<false>(p + f, t0, lane, f, v);
#pragma unroll
                for (int u = 0; u < 4; ++u) s[1][u] = __fadd_rn(s[1][u], v[u]);
            }
        }
        finish<W, false>(a, row, t0, lane, s);
    }
}

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
    if (!w) return fail(PGCN_GATED_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_GATED_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows, (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_GATED_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && !w->items) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_GATED_ERR_INVALID, "%s: null items/splits", what);
    return 0;
}

// Everything but the walk: sizes, width and operand pointers. `out_rows` rows of the output.
int check_call(const char* what, int32_t m, int32_t h, int32_t f, const float* K, const float* QV, const float* QVh,
               bool need_g, const float* gZ, const float* out, int64_t out_rows, const pgcn_gated_walk* w,
               const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_GATED_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (f < 1 || f > (1 << 24)) return fail(PGCN_GATED_ERR_INVALID, "%s: f=%d outside [1, 2^24]", what, f);
    if (m > 0 && (!K || !QV || (need_g && !gZ)))
        return fail(PGCN_GATED_ERR_INVALID, "%s: null K_own/QV_own%s", what, need_g ? "/gZ" : "");
    if (h > 0 && !QVh) return fail(PGCN_GATED_ERR_INVALID, "%s: h=%d but QV_halo is null", what, h);
    if (out_rows > 0 && !out) return fail(PGCN_GATED_ERR_INVALID, "%s: null output", what);
    if (w->nslots > 0 && !work) return fail(PGCN_GATED_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_GATED_ERR_NOGPU, "no CUDA device (%s): gated aggregation has no CPU path", cudaGetErrorString(e));
    }
    return 0;
}

bool aligned16(std::initializer_list<const void*> ops)
{
    for (const void* q : ops)
        if (q && (reinterpret_cast<uintptr_t>(q) & 15)) return false;
    return true;
}

template <int W>
int launch(const pgcn_gated_walk* w, int32_t m, int32_t f, const float* K, const float* QV, const float* QVh,
           const float* gZ, float* out, float* work, void* stream)
{
    if (w->nitems == 0) return PGCN_GATED_OK;
    GatedArgs a;
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits; a.m = m; a.f = f;
    a.K = K; a.QV = QV; a.QVh = QVh; a.gZ = gZ; a.out = out; a.work = work;
    const bool vec = f % 4 == 0 && aligned16({K, QV, QVh, gZ, out, work});
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((w->nitems + kGatedWarps - 1) / kGatedWarps);
    if (vec) gated_walk_kernel<W, true><<<grid, kGatedThreads, 0, s>>>(a);
    else gated_walk_kernel<W, false><<<grid, kGatedThreads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_GATED_ERR_CUDA, "gated_walk_kernel launch: %s", cudaGetErrorString(e));
    if (w->nsplits > 0) {
        gated_fixup_kernel<W><<<(unsigned)((w->nsplits + kGatedWarps - 1) / kGatedWarps), kGatedThreads, 0, s>>>(a);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail(PGCN_GATED_ERR_CUDA, "gated_fixup_kernel launch: %s", cudaGetErrorString(e));
    }
    return PGCN_GATED_OK;
}

}  // namespace

extern "C" {

const char* pgcn_gated_version(void) { return "pgcn_gated 0.1 (sm_90a, sigmoid-gated SpMM with recomputed gradients)"; }

const char* pgcn_gated_last_error(void) { return g_error.c_str(); }

int32_t pgcn_gated_chunk(void) { return kGatedChunk; }

int pgcn_gated_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* K_own, const float* QV_own,
                       const float* QV_halo, float* Z, float* work, int32_t f, void* stream)
{
    int rc = check_walk(fwd, m, "pgcn_gated_forward");
    if (rc || (rc = check_call("pgcn_gated_forward", m, h, f, K_own, QV_own, QV_halo, false, nullptr, Z, m, fwd, work)))
        return rc;
    return launch<kForward>(fwd, m, f, K_own, QV_own, h > 0 ? QV_halo : nullptr, nullptr, Z, work, stream);
}

int pgcn_gated_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* K_own,
                             const float* QV_own, const float* QV_halo, const float* gZ, float* dK, float* work,
                             int32_t f, void* stream)
{
    int rc = check_walk(fwd, m, "pgcn_gated_backward_rows");
    if (rc || (rc = check_call("pgcn_gated_backward_rows", m, h, f, K_own, QV_own, QV_halo, true, gZ, dK, m, fwd,
                               work)))
        return rc;
    return launch<kRows>(fwd, m, f, K_own, QV_own, h > 0 ? QV_halo : nullptr, gZ, dK, work, stream);
}

int pgcn_gated_backward_cols(const pgcn_gated_walk* tr, int32_t m, int32_t h, const float* K_own,
                             const float* QV_own, const float* QV_halo, const float* gZ, float* dQV, float* work,
                             int32_t f, void* stream)
{
    int rc = check_walk(tr, (int64_t)m + h, "pgcn_gated_backward_cols");
    if (rc || (rc = check_call("pgcn_gated_backward_cols", m, h, f, K_own, QV_own, QV_halo, true, gZ, dQV,
                               (int64_t)m + h, tr, work)))
        return rc;
    return launch<kCols>(tr, m, f, K_own, QV_own, h > 0 ? QV_halo : nullptr, gZ, dQV, work, stream);
}

}  // extern "C"
