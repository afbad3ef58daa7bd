// GatedGCN (include/pgcn_gatedgcn.h): the edge-gated aggregation with an edge-feature stream and its two backward walks.
//
// The gated aggregation's structure (gated.cu): one warp per work item, a row of at most pgcn_gated_chunk() entries or
// one chunk of a longer row, walked in CSR order 128 features per pass (4 per lane) with per-feature sums in registers.
// Per entry the warp streams one 128-float slice of each per-entry tensor (Ce, ehat, gEhat, dCe: nnz x f, 64-bit
// offsets) and gathers at most one 128-float slice of a node operand:
//   forward     Ce_e, [Ex | Bx][j]      -> ehat_e;      per row  num, den             -> Z, den
//   row walk    ehat_e, gEhat_e, Bx[j]  -> dCe_e;       per row  dDx (U, Z fixed)     -> dDx, U
//   column walk ehat_p, dCe_p, U[i]     (p = perm[t]);  per column  dEx, dBx          -> [dEx | dBx]
// A row walked whole is finished in the same warp; the chunks of a split row write their partial sums to the caller's
// work rows, and a fixup warp per split row adds them in chunk order and finishes the row. No atomics.
#include "../../include/pgcn_gatedgcn.h"
#include "gated_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

constexpr int kGcnThreads = 256;
constexpr int kGcnWarps = kGcnThreads / 32;
constexpr int kGcnTile = 128;            // features per pass of a warp

enum GatedGcnWalk : int { kGcnForward = 0, kGcnRows = 1, kGcnCols = 2 };

struct GatedGcnArgs {
    const int4* items;
    const int32_t* splits;     // nsplits x 3
    const int32_t* idx;        // columns (forward CSR) or rows (transposed CSR)
    const int32_t* perm;       // column walk: forward entry of each transposed entry
    int nitems, nsplits, m, f;
    float eps;
    const float* Dx;           // m x f (forward)
    const float* EB;           // m x 2f
    const float* EBh;          // h x 2f
    const float* Ce;           // nnz x f (forward)
    const float* Ehat;         // nnz x f (backward walks)
    const float* gEhat;        // nnz x f or NULL (row walk)
    const float* Z;            // m x f (row walk)
    const float* den;          // m x f (row walk)
    const float* gZ;           // m x f (row walk)
    const float* U;            // m x f (column walk)
    float* out;                // Z (forward), dDx (row walk), or (m + h) x 2f [dEx | dBx] (column walk)
    float* out2;               // den (forward), U (row walk)
    float* pe;                 // per-entry output: ehat (forward), dCe (row walk)
    const float* pe_in;        // dCe (column walk)
    float* work;               // nslots x (2f or f)
};

__device__ __forceinline__ const float* eb_row(const GatedGcnArgs& a, int j)
{
    return j < a.m ? a.EB + (size_t)j * 2 * a.f : a.EBh + (size_t)(j - a.m) * 2 * a.f;
}

// U = gZ / (den + eps) and Z of row r: the row walk's fixed operands, formed the same way wherever they are needed.
template <bool VEC>
__device__ __forceinline__ void row_u(const GatedGcnArgs& a, int r, int t0, int lane, float (&u)[4], float (&z)[4])
{
    const int f = a.f;
    float g[4], d[4];
    load4<VEC>(a.gZ + (size_t)r * f, t0, lane, f, g);
    load4<VEC>(a.den + (size_t)r * f, t0, lane, f, d);
    load4<VEC>(a.Z + (size_t)r * f, t0, lane, f, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = __fdiv_rn(g[k], __fadd_rn(d[k], a.eps));
}

// Finish row r from its sums: forward Z = s0 / (s1 + eps), den = s1; row walk dDx = s0 and U; column walk
// [dEx | dBx] = [s0 | s1].
template <int W, bool VEC>
__device__ __forceinline__ void finish(const GatedGcnArgs& a, int r, int t0, int lane, float (&s)[2][4])
{
    const int f = a.f;
    if constexpr (W == kGcnForward) {
        float z[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = __fdiv_rn(s[0][k], __fadd_rn(s[1][k], a.eps));
        store4<VEC>(a.out + (size_t)r * f, t0, lane, f, z);
        store4<VEC>(a.out2 + (size_t)r * f, t0, lane, f, s[1]);
    } else if constexpr (W == kGcnRows) {
        float u[4], z[4];
        row_u<VEC>(a, r, t0, lane, u, z);
        store4<VEC>(a.out + (size_t)r * f, t0, lane, f, s[0]);
        store4<VEC>(a.out2 + (size_t)r * f, t0, lane, f, u);
    } else {
        store4<VEC>(a.out + (size_t)r * 2 * f, t0, lane, f, s[0]);
        store4<VEC>(a.out + (size_t)r * 2 * f + f, t0, lane, f, s[1]);
    }
}

template <int W, bool VEC>
__global__ void __launch_bounds__(kGcnThreads) gatedgcn_walk_kernel(GatedGcnArgs a)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kGcnWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f;
    for (int t0 = 0; t0 < f; t0 += kGcnTile) {
        float s[2][4] = {};
        float fx[4] = {}, fz[4] = {};      // Dx[r] (forward); U[r], Z[r] (row walk)
        if constexpr (W == kGcnForward) load4<VEC>(a.Dx + (size_t)r * f, t0, lane, f, fx);
        if constexpr (W == kGcnRows) row_u<VEC>(a, r, t0, lane, fx, fz);
        for (int eb = e0; eb < e1; eb += 32) {
            const int nb = min(32, e1 - eb);
            const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
            const int mperm = W == kGcnCols && lane < nb ? __ldg(a.perm + eb + lane) : 0;
#pragma unroll 4
            for (int k = 0; k < nb; ++k) {
                const int j = __shfl_sync(0xffffffffu, mine, k);      // column (forward, row walk) or row
                if constexpr (W == kGcnForward) {
                    const size_t pe = (size_t)(eb + k) * f;
                    const float* q = eb_row(a, j);
                    float x[4], y[4], c[4], e[4];
                    load4<VEC>(q, t0, lane, f, x);
                    load4<VEC>(q + f, t0, lane, f, y);
                    load4<VEC>(a.Ce + pe, t0, lane, f, c);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        float ds;
                        e[u] = __fadd_rn(__fadd_rn(fx[u], x[u]), c[u]);
                        const float eta = gate(e[u], ds);
                        s[0][u] = __fmaf_rn(eta, y[u], s[0][u]);
                        s[1][u] = __fadd_rn(s[1][u], eta);
                    }
                    store4<VEC>(a.pe + pe, t0, lane, f, e);
                } else if constexpr (W == kGcnRows) {
                    const size_t pe = (size_t)(eb + k) * f;
                    float y[4], e[4], g[4] = {}, d[4];
                    load4<VEC>(eb_row(a, j) + f, t0, lane, f, y);
                    load4<VEC>(a.Ehat + pe, t0, lane, f, e);
                    if (a.gEhat) load4<VEC>(a.gEhat + pe, t0, lane, f, g);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        float ds;
                        gate(e[u], ds);
                        const float dsig = __fmul_rn(fx[u], __fsub_rn(y[u], fz[u]));
                        d[u] = __fmaf_rn(dsig, ds, g[u]);
                        s[0][u] = __fadd_rn(s[0][u], d[u]);
                    }
                    store4<VEC>(a.pe + pe, t0, lane, f, d);
                } else {
                    const size_t pe = (size_t)__shfl_sync(0xffffffffu, mperm, k) * f;
                    float e[4], d[4], u4[4];
                    load4<VEC>(a.Ehat + pe, t0, lane, f, e);
                    load4<VEC>(a.pe_in + pe, t0, lane, f, d);
                    load4<VEC>(a.U + (size_t)j * f, t0, lane, f, u4);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        float ds;
                        const float eta = gate(e[u], ds);
                        s[0][u] = __fadd_rn(s[0][u], d[u]);
                        s[1][u] = __fmaf_rn(eta, u4[u], s[1][u]);
                    }
                }
            }
        }
        if (slot < 0) {
            finish<W, VEC>(a, r, t0, lane, s);
        } else {
            // a chunk of a split row: its raw sums, [s0 | s1] or [s0], finished by the fixup
            const int ow = W == kGcnRows ? f : 2 * f;
            store4<VEC>(a.work + (size_t)slot * ow, t0, lane, f, s[0]);
            if constexpr (W != kGcnRows) store4<VEC>(a.work + (size_t)slot * ow + f, t0, lane, f, s[1]);
        }
    }
}

// One warp per split row (row, slot0, count): the chunks' partial sums added in chunk order, then the row finished.
template <int W>
__global__ void __launch_bounds__(kGcnThreads) gatedgcn_fixup_kernel(GatedGcnArgs a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kGcnWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f, ow = W == kGcnRows ? f : 2 * f;
    for (int t0 = 0; t0 < f; t0 += kGcnTile) {
        float s[2][4] = {};
        for (int q = 0; q < n; ++q) {
            const float* p = a.work + (size_t)(slot0 + q) * ow;
            float v[4];
            load4<false>(p, t0, lane, f, v);
#pragma unroll
            for (int u = 0; u < 4; ++u) s[0][u] = __fadd_rn(s[0][u], v[u]);
            if constexpr (W != kGcnRows) {
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
    if (!w) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows,
                    (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Sizes, width, eps and work; the operand pointers are checked by each entry point, the device last.
int check_call(const char* what, int32_t m, int32_t h, int32_t f, float eps, const pgcn_gated_walk* w,
               const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (f < 1 || f > (1 << 24)) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: f=%d outside [1, 2^24]", what, f);
    if (!(eps >= 0.0f) || std::isinf(eps))
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: eps=%g must be finite and >= 0", what, (double)eps);
    if (w->nslots > 0 && !work)
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    return 0;
}

// Last of the checks: a device to run on.
int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_GATEDGCN_ERR_NOGPU, "no CUDA device (%s): GatedGCN has no CPU path", cudaGetErrorString(e));
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
int launch(const pgcn_gated_walk* w, GatedGcnArgs a, void* stream)
{
    if (w->nitems == 0) return PGCN_GATEDGCN_OK;
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits;
    const bool vec = a.f % 4 == 0 && aligned16({a.Dx, a.EB, a.EBh, a.Ce, a.Ehat, a.gEhat, a.Z, a.den, a.gZ, a.U, a.out,
                                                a.out2, a.pe, a.pe_in, a.work});
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((w->nitems + kGcnWarps - 1) / kGcnWarps);
    if (vec) gatedgcn_walk_kernel<W, true><<<grid, kGcnThreads, 0, s>>>(a);
    else gatedgcn_walk_kernel<W, false><<<grid, kGcnThreads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_GATEDGCN_ERR_CUDA, "gatedgcn_walk_kernel launch: %s", cudaGetErrorString(e));
    if (w->nsplits > 0) {
        gatedgcn_fixup_kernel<W><<<(unsigned)((w->nsplits + kGcnWarps - 1) / kGcnWarps), kGcnThreads, 0, s>>>(a);
        e = cudaGetLastError();
        if (e != cudaSuccess)
            return fail(PGCN_GATEDGCN_ERR_CUDA, "gatedgcn_fixup_kernel launch: %s", cudaGetErrorString(e));
    }
    return PGCN_GATEDGCN_OK;
}

template <int W>
void touch(int& rc)
{
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)gatedgcn_walk_kernel<W, true>),
                          cudaFuncGetAttributes(&fa, (const void*)gatedgcn_walk_kernel<W, false>),
                          cudaFuncGetAttributes(&fa, (const void*)gatedgcn_fixup_kernel<W>)})
        if (e != cudaSuccess && !rc) rc = fail(PGCN_GATEDGCN_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
}

GatedGcnArgs blank(int32_t m, int32_t f, float eps)
{
    GatedGcnArgs a = {};
    a.m = m; a.f = f; a.eps = eps;
    return a;
}

}  // namespace

extern "C" {

const char* pgcn_gatedgcn_version(void) { return "pgcn_gatedgcn 0.1 (sm_90a, GatedGCN edge-gated aggregation)"; }

const char* pgcn_gatedgcn_last_error(void) { return g_error.c_str(); }

int pgcn_gatedgcn_load(void)
{
    static bool loaded[256] = {};
    int rc = check_device();
    if (rc) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && loaded[dev]) return PGCN_GATEDGCN_OK;
    touch<kGcnForward>(rc);
    touch<kGcnRows>(rc);
    touch<kGcnCols>(rc);
    if (!rc && dev >= 0 && dev < 256) loaded[dev] = true;
    return rc;
}

int pgcn_gatedgcn_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* Dx_own, const float* EB_own,
                          const float* EB_halo, const float* Ce, float eps, float* Z, float* den, float* Ehat,
                          float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_gatedgcn_forward";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_call(what, m, h, f, eps, fwd, work))) return rc;
    if (m > 0 && (!Dx_own || !EB_own || !Ce))
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null Dx_own/EB_own/Ce", what);
    if (h > 0 && !EB_halo) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: h=%d but EB_halo is null", what, h);
    if (m > 0 && (!Z || !den || !Ehat)) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null output Z/den/Ehat", what);
    if ((rc = check_device())) return rc;
    GatedGcnArgs a = blank(m, f, eps);
    a.Dx = Dx_own; a.EB = EB_own; a.EBh = h > 0 ? EB_halo : nullptr; a.Ce = Ce;
    a.out = Z; a.out2 = den; a.pe = Ehat; a.work = work;
    return launch<kGcnForward>(fwd, a, stream);
}

int pgcn_gatedgcn_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* EB_own,
                                const float* EB_halo, const float* Ehat, const float* gEhat, const float* Z,
                                const float* den, const float* gZ, float eps, float* U, float* dCe, float* dDx,
                                float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_gatedgcn_backward_rows";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_call(what, m, h, f, eps, fwd, work))) return rc;
    if (m > 0 && (!EB_own || !Ehat || !Z || !den || !gZ))
        return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null EB_own/Ehat/Z/den/gZ", what);
    if (h > 0 && !EB_halo) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: h=%d but EB_halo is null", what, h);
    if (m > 0 && (!U || !dCe || !dDx)) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null output U/dCe/dDx", what);
    if ((rc = check_device())) return rc;
    GatedGcnArgs a = blank(m, f, eps);
    a.EB = EB_own; a.EBh = h > 0 ? EB_halo : nullptr; a.Ehat = Ehat; a.gEhat = gEhat; a.Z = Z; a.den = den; a.gZ = gZ;
    a.out = dDx; a.out2 = U; a.pe = dCe; a.work = work;
    return launch<kGcnRows>(fwd, a, stream);
}

int pgcn_gatedgcn_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h,
                                const float* Ehat, const float* dCe, const float* U, float* dEB, float* work,
                                int32_t f, void* stream)
{
    const char* what = "pgcn_gatedgcn_backward_cols";
    int rc = check_walk(tr, (int64_t)m + h, what);
    if (rc || (rc = check_call(what, m, h, f, 0.0f, tr, work))) return rc;
    if (tr->rows > 0 && !perm) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null perm", what);
    if (m > 0 && (!Ehat || !dCe || !U)) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null Ehat/dCe/U", what);
    if (tr->rows > 0 && !dEB) return fail(PGCN_GATEDGCN_ERR_INVALID, "%s: null output dEB", what);
    if ((rc = check_device())) return rc;
    GatedGcnArgs a = blank(m, f, 0.0f);
    a.perm = perm; a.Ehat = Ehat; a.pe_in = dCe; a.U = U; a.out = dEB; a.work = work;
    return launch<kGcnCols>(tr, a, stream);
}

}  // extern "C"
