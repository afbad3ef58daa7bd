// GINE (include/pgcn_gine.h): the edge-feature sum aggregation with ReLU messages and its one backward walk.
//
// The gated aggregation's structure (gated.cu, gatedgcn.cu): one warp per work item, a row of at most
// pgcn_gated_chunk() entries or one chunk of a longer row, walked in CSR order 128 features per pass (4 per lane) with
// per-feature sums in registers. Per entry the warp streams one 128-float slice of E (nnz x f, 64-bit offsets) and
// gathers one 128-float slice of a node operand:
//   forward   E_e, X[j]             -> msg_e;                  per row     sum msg            -> Z
//   backward  E_p, gZ[i]  (p = perm[t], X[j] once per item)    per column  sum dE_p           -> dX; dE_p written
// A row walked whole is finished in the same warp; the chunks of a split row write their partial sums to the caller's
// work rows, and a fixup warp per split row adds them in chunk order and finishes the row. No atomics.
#include "../../include/pgcn_gine.h"
#include "gated_math.cuh"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

constexpr int kGineThreads = 256;
constexpr int kGineWarps = kGineThreads / 32;
constexpr int kGineTile = 128;           // features per pass of a warp

enum GineWalk : int { kGineForward = 0, kGineBackward = 1 };

struct GineArgs {
    const int4* items;
    const int32_t* splits;     // nsplits x 3
    const int32_t* idx;        // columns (forward CSR) or rows (transposed CSR)
    const int32_t* perm;       // backward: forward entry of each transposed entry
    int nitems, nsplits, m, f;
    const float* X;            // m x f
    const float* Xh;           // h x f
    const float* E;            // nnz x f
    const float* gZ;           // m x f (backward)
    float* dE;                 // nnz x f or NULL (backward)
    float* out;                // Z (forward, m x f) or dX (backward, (m + h) x f)
    float* work;               // nslots x f
};

__device__ __forceinline__ const float* x_row(const GineArgs& a, int j)
{
    return j < a.m ? a.X + (size_t)j * a.f : a.Xh + (size_t)(j - a.m) * a.f;
}

template <int W, bool VEC>
__global__ void __launch_bounds__(kGineThreads) gine_walk_kernel(GineArgs a)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kGineWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f;
    for (int t0 = 0; t0 < f; t0 += kGineTile) {
        float s[4] = {};
        float xr[4] = {};                  // X[r], the column's own features (backward)
        if constexpr (W == kGineBackward) load4<VEC>(x_row(a, r), t0, lane, f, xr);
        for (int eb = e0; eb < e1; eb += 32) {
            const int nb = min(32, e1 - eb);
            const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
            const int mperm = W == kGineBackward && lane < nb ? __ldg(a.perm + eb + lane) : 0;
#pragma unroll 4
            for (int k = 0; k < nb; ++k) {
                const int j = __shfl_sync(0xffffffffu, mine, k);      // column (forward) or row (backward)
                if constexpr (W == kGineForward) {
                    const size_t pe = (size_t)(eb + k) * f;
                    float x[4], e[4];
                    load4<VEC>(x_row(a, j), t0, lane, f, x);
                    load4<VEC>(a.E + pe, t0, lane, f, e);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const float pre = __fadd_rn(x[u], e[u]);
                        s[u] = __fadd_rn(s[u], pre < 0.0f ? 0.0f : pre);
                    }
                } else {
                    const size_t pe = (size_t)__shfl_sync(0xffffffffu, mperm, k) * f;
                    float e[4], g[4], d[4];
                    load4<VEC>(a.E + pe, t0, lane, f, e);
                    load4<VEC>(a.gZ + (size_t)j * f, t0, lane, f, g);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        d[u] = !(__fadd_rn(xr[u], e[u]) <= 0.0f) ? g[u] : 0.0f;
                        s[u] = __fadd_rn(s[u], d[u]);
                    }
                    if (a.dE) store4<VEC>(a.dE + pe, t0, lane, f, d);
                }
            }
        }
        // a row walked whole is finished here; a chunk of a split row leaves its raw sum to the fixup
        if (slot < 0) store4<VEC>(a.out + (size_t)r * f, t0, lane, f, s);
        else store4<VEC>(a.work + (size_t)slot * f, t0, lane, f, s);
    }
}

// One warp per split row (row, slot0, count): the chunks' partial sums added in chunk order, then the row written.
template <int W>
__global__ void __launch_bounds__(kGineThreads) gine_fixup_kernel(GineArgs a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kGineWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f;
    for (int t0 = 0; t0 < f; t0 += kGineTile) {
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
    if (!w) return fail(PGCN_GINE_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_GINE_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows, (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_GINE_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_GINE_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Sizes, width, work and the X operands; the other pointers are checked by each entry point, the device last.
int check_call(const char* what, int32_t m, int32_t h, int32_t f, const pgcn_gated_walk* w, const float* X_own,
               const float* X_halo, const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_GINE_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (f < 1 || f > (1 << 24)) return fail(PGCN_GINE_ERR_INVALID, "%s: f=%d outside [1, 2^24]", what, f);
    if (w->nslots > 0 && !work) return fail(PGCN_GINE_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    if (m > 0 && !X_own) return fail(PGCN_GINE_ERR_INVALID, "%s: null X_own", what);
    if (h > 0 && !X_halo) return fail(PGCN_GINE_ERR_INVALID, "%s: h=%d but X_halo is null", what, h);
    return 0;
}

// Last of the checks: a device to run on.
int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_GINE_ERR_NOGPU, "no CUDA device (%s): GINE has no CPU path", cudaGetErrorString(e));
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
int launch(const pgcn_gated_walk* w, GineArgs a, void* stream)
{
    if (w->nitems == 0) return PGCN_GINE_OK;
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits;
    const bool vec = a.f % 4 == 0 && aligned16({a.X, a.Xh, a.E, a.gZ, a.dE, a.out, a.work});
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((w->nitems + kGineWarps - 1) / kGineWarps);
    if (vec) gine_walk_kernel<W, true><<<grid, kGineThreads, 0, s>>>(a);
    else gine_walk_kernel<W, false><<<grid, kGineThreads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_GINE_ERR_CUDA, "gine_walk_kernel launch: %s", cudaGetErrorString(e));
    if (w->nsplits > 0) {
        gine_fixup_kernel<W><<<(unsigned)((w->nsplits + kGineWarps - 1) / kGineWarps), kGineThreads, 0, s>>>(a);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail(PGCN_GINE_ERR_CUDA, "gine_fixup_kernel launch: %s", cudaGetErrorString(e));
    }
    return PGCN_GINE_OK;
}

template <int W>
void touch(int& rc)
{
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)gine_walk_kernel<W, true>),
                          cudaFuncGetAttributes(&fa, (const void*)gine_walk_kernel<W, false>),
                          cudaFuncGetAttributes(&fa, (const void*)gine_fixup_kernel<W>)})
        if (e != cudaSuccess && !rc) rc = fail(PGCN_GINE_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
}

}  // namespace

extern "C" {

const char* pgcn_gine_version(void) { return "pgcn_gine 0.1 (sm_90a, GINE edge-feature sum aggregation)"; }

const char* pgcn_gine_last_error(void) { return g_error.c_str(); }

int pgcn_gine_load(void)
{
    static bool loaded[256] = {};
    int rc = check_device();
    if (rc) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && loaded[dev]) return PGCN_GINE_OK;
    touch<kGineForward>(rc);
    touch<kGineBackward>(rc);
    if (!rc && dev >= 0 && dev < 256) loaded[dev] = true;
    return rc;
}

int pgcn_gine_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* X_own, const float* X_halo,
                      const float* E, float* Z, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_gine_forward";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_call(what, m, h, f, fwd, X_own, X_halo, work))) return rc;
    if (m > 0 && !E) return fail(PGCN_GINE_ERR_INVALID, "%s: null E", what);
    if (m > 0 && !Z) return fail(PGCN_GINE_ERR_INVALID, "%s: null output Z", what);
    if ((rc = check_device())) return rc;
    GineArgs a = {};
    a.m = m; a.f = f;
    a.X = X_own; a.Xh = h > 0 ? X_halo : nullptr; a.E = E; a.out = Z; a.work = work;
    return launch<kGineForward>(fwd, a, stream);
}

int pgcn_gine_backward(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, const float* X_own,
                       const float* X_halo, const float* E, const float* gZ, float* dE, float* dX, float* work,
                       int32_t f, void* stream)
{
    const char* what = "pgcn_gine_backward";
    int rc = check_walk(tr, (int64_t)m + h, what);
    if (rc || (rc = check_call(what, m, h, f, tr, X_own, X_halo, work))) return rc;
    if (tr->rows > 0 && !perm) return fail(PGCN_GINE_ERR_INVALID, "%s: null perm", what);
    if (m > 0 && (!E || !gZ)) return fail(PGCN_GINE_ERR_INVALID, "%s: null E/gZ", what);
    if (tr->rows > 0 && !dX) return fail(PGCN_GINE_ERR_INVALID, "%s: null output dX", what);
    if ((rc = check_device())) return rc;
    GineArgs a = {};
    a.m = m; a.f = f;
    a.perm = perm; a.X = X_own; a.Xh = h > 0 ? X_halo : nullptr; a.E = E; a.gZ = gZ; a.dE = dE; a.out = dX;
    a.work = work;
    return launch<kGineBackward>(tr, a, stream);
}

}  // extern "C"
