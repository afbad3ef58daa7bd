// Relational aggregation (include/pgcn_rgcn.h): R-GCN's per-relation weighted sum, forward and backward by one walk.
//
// The relations are virtual rows: Z [m, R, f] is a plain [m R, f] output over a CSR whose rows are v = i R + r, and the
// backward's column walk reads gZ [m R, f] at t_colidx R + rel. The caller's walks carry R in their indices, so one
// kernel serves both directions:
//   out[v] = sum_{e in item of v} w[perm[e]] * src[idx[e]]        src = own rows [0, split), then halo rows
// with the gated aggregation's structure (gated.cu, gine.cu): one warp per work item, a row of at most
// pgcn_gated_chunk() entries or one chunk of a longer row, walked in CSR order 128 features per pass (4 per lane) with
// per-feature sums in registers. Per entry the warp gathers one 128-float slice of src; the entry's index (and, with
// weights, its weight through perm) is loaded once per 32 entries by one lane and broadcast. A row walked whole is
// finished in the same warp; the chunks of a split row write their partial sums to the caller's work rows, and a
// fixup warp per split row adds them in chunk order. No atomics.
#include "../../include/pgcn_rgcn.h"
#include "gated_math.cuh"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

constexpr int kRgcnThreads = 256;
constexpr int kRgcnWarps = kRgcnThreads / 32;
constexpr int kRgcnTile = 128;           // features per pass of a warp

struct RgcnArgs {
    const int4* items;
    const int32_t* splits;     // nsplits x 3
    const int32_t* idx;        // source row of every entry: X column (forward) or virtual row of gZ (backward)
    const int32_t* perm;       // forward entry of every walked entry (read only with weights)
    const float* w;            // nnz, forward entry order, or NULL
    int nitems, nsplits, split, f;
    const float* src;          // split x f: X_own (forward) or gZ (backward)
    const float* srch;         // halo rows of X (forward), NULL (backward)
    float* out;                // Z (forward, m R x f) or dX (backward, (m + h) x f)
    float* work;               // nslots x f
};

__device__ __forceinline__ const float* src_row(const RgcnArgs& a, int j)
{
    return j < a.split ? a.src + (size_t)j * a.f : a.srch + (size_t)(j - a.split) * a.f;
}

template <bool VEC, bool WEIGHTED>
__global__ void __launch_bounds__(kRgcnThreads) rgcn_walk_kernel(RgcnArgs a)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kRgcnWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f;
    for (int t0 = 0; t0 < f; t0 += kRgcnTile) {
        float s[4] = {};
        for (int eb = e0; eb < e1; eb += 32) {
            const int nb = min(32, e1 - eb);
            const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
            float mw = 0.0f;
            if constexpr (WEIGHTED) mw = lane < nb ? __ldg(a.w + __ldg(a.perm + eb + lane)) : 0.0f;
#pragma unroll 4
            for (int k = 0; k < nb; ++k) {
                const int j = __shfl_sync(0xffffffffu, mine, k);
                float x[4];
                load4<VEC>(src_row(a, j), t0, lane, f, x);
                if constexpr (WEIGHTED) {
                    const float wk = __shfl_sync(0xffffffffu, mw, k);
#pragma unroll
                    for (int u = 0; u < 4; ++u) s[u] = __fadd_rn(s[u], __fmul_rn(wk, x[u]));
                } else {
#pragma unroll
                    for (int u = 0; u < 4; ++u) s[u] = __fadd_rn(s[u], x[u]);
                }
            }
        }
        // a row walked whole is finished here; a chunk of a split row leaves its raw sum to the fixup
        if (slot < 0) store4<VEC>(a.out + (size_t)r * f, t0, lane, f, s);
        else store4<VEC>(a.work + (size_t)slot * f, t0, lane, f, s);
    }
}

// One warp per split row (row, slot0, count): the chunks' partial sums added in chunk order, then the row written.
__global__ void __launch_bounds__(kRgcnThreads) rgcn_fixup_kernel(RgcnArgs a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kRgcnWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f;
    for (int t0 = 0; t0 < f; t0 += kRgcnTile) {
        float s[4] = {};
        for (int q = 0; q < n; ++q) {
            float v[4];
            load4<false>(a.work + (size_t)(slot0 + q) * f, t0, lane, f, v);
#pragma unroll
            for (int u = 0; u < 4; ++u) s[u] = __fadd_rn(s[u], v[u]);
        }
        store4<false>(a.out + (size_t)row * f, t0, lane, f, s);
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
    if (!w) return fail(PGCN_RGCN_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_RGCN_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows, (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_RGCN_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_RGCN_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Sizes, relation count, width, work and weights, before the walk; the other pointers are checked by each entry point,
// the device last.
int check_sizes(const char* what, int32_t m, int32_t h, int32_t R, int32_t f)
{
    if (m < 0 || h < 0) return fail(PGCN_RGCN_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (R < 1) return fail(PGCN_RGCN_ERR_INVALID, "%s: R=%d relations, need at least 1", what, R);
    if ((int64_t)m * R > INT32_MAX)
        return fail(PGCN_RGCN_ERR_INVALID, "%s: m R = %lld virtual rows exceed 2^31 - 1", what, (long long)m * R);
    if (f < 1 || f > (1 << 24)) return fail(PGCN_RGCN_ERR_INVALID, "%s: f=%d outside [1, 2^24]", what, f);
    return 0;
}

int check_operands(const char* what, const pgcn_gated_walk* w, const int32_t* perm, const float* wt,
                   const float* work)
{
    if (w->nslots > 0 && !work) return fail(PGCN_RGCN_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    if (wt && w->rows > 0 && !perm) return fail(PGCN_RGCN_ERR_INVALID, "%s: weights given but perm is null", what);
    return 0;
}

// Last of the checks: a device to run on.
int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_RGCN_ERR_NOGPU, "no CUDA device (%s): R-GCN has no CPU path", cudaGetErrorString(e));
    }
    return 0;
}

bool aligned16(std::initializer_list<const void*> ops)
{
    for (const void* q : ops)
        if (q && (reinterpret_cast<uintptr_t>(q) & 15)) return false;
    return true;
}

template <bool VEC>
void launch_walk(RgcnArgs a, unsigned grid, cudaStream_t s)
{
    if (a.w) rgcn_walk_kernel<VEC, true><<<grid, kRgcnThreads, 0, s>>>(a);
    else rgcn_walk_kernel<VEC, false><<<grid, kRgcnThreads, 0, s>>>(a);
}

int launch(const pgcn_gated_walk* w, RgcnArgs a, void* stream)
{
    if (w->nitems == 0) return PGCN_RGCN_OK;
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits;
    const bool vec = a.f % 4 == 0 && aligned16({a.src, a.srch, a.out, a.work});
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((w->nitems + kRgcnWarps - 1) / kRgcnWarps);
    if (vec) launch_walk<true>(a, grid, s);
    else launch_walk<false>(a, grid, s);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_RGCN_ERR_CUDA, "rgcn_walk_kernel launch: %s", cudaGetErrorString(e));
    if (w->nsplits > 0) {
        rgcn_fixup_kernel<<<(unsigned)((w->nsplits + kRgcnWarps - 1) / kRgcnWarps), kRgcnThreads, 0, s>>>(a);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail(PGCN_RGCN_ERR_CUDA, "rgcn_fixup_kernel launch: %s", cudaGetErrorString(e));
    }
    return PGCN_RGCN_OK;
}

}  // namespace

extern "C" {

const char* pgcn_rgcn_version(void) { return "pgcn_rgcn 0.1 (sm_90a, R-GCN relational aggregation)"; }

const char* pgcn_rgcn_last_error(void) { return g_error.c_str(); }

int pgcn_rgcn_load(void)
{
    static bool loaded[256] = {};
    int rc = check_device();
    if (rc) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && loaded[dev]) return PGCN_RGCN_OK;
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)rgcn_walk_kernel<true, true>),
                          cudaFuncGetAttributes(&fa, (const void*)rgcn_walk_kernel<true, false>),
                          cudaFuncGetAttributes(&fa, (const void*)rgcn_walk_kernel<false, true>),
                          cudaFuncGetAttributes(&fa, (const void*)rgcn_walk_kernel<false, false>),
                          cudaFuncGetAttributes(&fa, (const void*)rgcn_fixup_kernel)})
        if (e != cudaSuccess && !rc) rc = fail(PGCN_RGCN_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
    if (!rc && dev >= 0 && dev < 256) loaded[dev] = true;
    return rc;
}

int pgcn_rgcn_forward(const pgcn_gated_walk* fwd, const int32_t* perm, int32_t m, int32_t h, int32_t R,
                      const float* X_own, const float* X_halo, const float* w, float* Z, float* work, int32_t f,
                      void* stream)
{
    const char* what = "pgcn_rgcn_forward";
    int rc = check_sizes(what, m, h, R, f);
    if (rc || (rc = check_walk(fwd, (int64_t)m * R, what)) || (rc = check_operands(what, fwd, perm, w, work)))
        return rc;
    if (m > 0 && !X_own) return fail(PGCN_RGCN_ERR_INVALID, "%s: null X_own", what);
    if (h > 0 && !X_halo) return fail(PGCN_RGCN_ERR_INVALID, "%s: h=%d but X_halo is null", what, h);
    if (fwd->rows > 0 && !Z) return fail(PGCN_RGCN_ERR_INVALID, "%s: null output Z", what);
    if ((rc = check_device())) return rc;
    RgcnArgs a = {};
    a.split = m; a.f = f;
    a.perm = perm; a.w = w; a.src = X_own; a.srch = h > 0 ? X_halo : nullptr; a.out = Z; a.work = work;
    return launch(fwd, a, stream);
}

int pgcn_rgcn_backward(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, int32_t R,
                       const float* gZ, const float* w, float* dX, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_rgcn_backward";
    int rc = check_sizes(what, m, h, R, f);
    if (rc || (rc = check_walk(tr, (int64_t)m + h, what)) || (rc = check_operands(what, tr, perm, w, work)))
        return rc;
    if (m > 0 && !gZ) return fail(PGCN_RGCN_ERR_INVALID, "%s: null gZ", what);
    if (tr->rows > 0 && !dX) return fail(PGCN_RGCN_ERR_INVALID, "%s: null output dX", what);
    if ((rc = check_device())) return rc;
    RgcnArgs a = {};
    a.split = m * R; a.f = f;
    a.perm = perm; a.w = w; a.src = gZ; a.srch = nullptr; a.out = dX; a.work = work;
    return launch(tr, a, stream);
}

}  // extern "C"
