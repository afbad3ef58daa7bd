// GATv2 attention with edge features (include/pgcn_gatv2_edge.h): GATv2Conv's dynamic attention with an edge term in
// the score, attention dropout, and its two backward walks, over the gated aggregation's work tables.
//
// The lane layout, online softmax, dropout mask and split-row fixups are the transformer's (transformer_math.cuh), with
// XL in the place of [k | v] (rows of f floats, not 2f: xl_row) and XR in the place of q. Per entry:
//   forward     XL[j] gathered, E_e streamed (64-bit offsets), t = (XR[i] + XL[j]) + E_e    -> online softmax  -> Z, L
//   row walk    the same gather and stream, p = expf(s - L)          -> G_e = g_e, PS_e = [P | ds], datt partial -> dXR
//   column walk gZ[i] gathered, PS_p and G_p read (p = perm[t])                                                -> dXL
// The column walk recomputes no score: the row walk has stored each entry's P = M p and g (f floats), which it needs
// anyway as dE, where a recomputation would need the entry's f-wide E through the same scattered permutation. A row
// walked whole is finished in its warp; the chunks of a split row write their partials to the caller's work rows and a
// fixup warp per split row merges them in chunk order. datt is summed per CTA of the row walk (its warps in warp order)
// and the CTA partials in CTA order by gatv2_edge_datt_kernel. Every output element is reduced in one fixed order,
// without atomics.
#include "../../include/pgcn_gatv2_edge.h"
#include "transformer_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

// The operands beside the transformer's (TrArgs: Q = XR, KV = XL_own, KVh = XL_halo, both f wide).
struct G2Args {
    const float* att;          // f: att[h, c] is feature h d + c
    float slope;
    const float* E;            // nnz x f (forward, row walk)
    float* G;                  // nnz x f: g_e, written by the row walk (dE or scratch)
    float* PS;                 // nnz x 2K: written by the row walk
    const float* Gc;           // the same two, read by the column walk
    const float* PSc;
    const int32_t* perm;       // column walk: forward entry of each transposed entry
    float* part;               // row walk: one datt partial of f floats per CTA
};

__device__ __forceinline__ const float* xl_row(const TrArgs& a, int j)
{
    return j < a.m ? a.KV + (size_t)j * a.f : a.KVh + (size_t)(j - a.m) * a.f;
}

__device__ __forceinline__ float leaky(float t, float slope) { return t > 0.0f ? t : __fmul_rn(t, slope); }

// xl = XL[j] and lt = LeakyReLU(t), t = (XR[i] + XL[j]) + E_e, on this lane's slots (unused slots stay 0). Returns
// bit u set where t > 0, all the row walk keeps of t.
template <bool VEC>
__device__ __forceinline__ unsigned edge_t(const TrArgs& a, const G2Args& b, int j, size_t pe, const Lanes& ln,
                                           const float (&xr)[8], float (&xl)[8], float (&lt)[8])
{
    float e[8];
    load8<VEC>(xl_row(a, j), ln, xl);
    load8<VEC>(b.E + pe, ln, e);
    unsigned pos = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const float t = __fadd_rn(__fadd_rn(xr[u], xl[u]), e[u]);
        pos |= (t > 0.0f ? 1u : 0u) << u;
        lt[u] = leaky(t, b.slope);
    }
    return pos;
}

template <int W, bool VEC>
__global__ void __launch_bounds__(kTrThreads, W == kTrRows ? 2 : 1) gatv2_edge_walk_kernel(TrArgs a, G2Args b)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    const int f = a.f, K = a.heads;
    const Lanes ln = lanes(lane, f, K);
    float acc[8] = {}, acc2[8] = {};         // Z, dXR or dXL; the row walk's datt
    if (item < a.nitems) {
        const int4 it = __ldg(a.items + item);           // (row, e0, e1, slot)
        const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
        if constexpr (W == kTrCols) {
            for (int eb = e0; eb < e1; eb += 32) {
                const int nb = min(32, e1 - eb);
                const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
                const int mperm = lane < nb ? __ldg(b.perm + eb + lane) : 0;
#pragma unroll 2
                for (int k = 0; k < nb; ++k) {
                    const int i = __shfl_sync(0xffffffffu, mine, k);
                    const size_t pe = (size_t)__shfl_sync(0xffffffffu, mperm, k);
                    const float P = __ldg(b.PSc + pe * 2 * K + ln.h);
                    float y[8], g[8];            // gZ[i], g_e
                    load8<VEC>(a.gZ + (size_t)i * f, ln, y);
                    load8<VEC>(b.Gc + pe * f, ln, g);
#pragma unroll
                    for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], __fmaf_rn(P, y[q], g[q]));
                }
            }
        } else {
            const Drop dr = drop_state(a);
            const int gr = dr.on ? __ldg(a.gid + r) : 0;
            float xr[8], at[8], y[8];            // XR[r], att; gZ[r] in the row walk
            load8<VEC>(a.Q + (size_t)r * f, ln, xr);
            load8<VEC>(b.att, ln, at);
            float Lr = 0.0f, Dr = 0.0f;
            if constexpr (W == kTrRows) {
                load8<VEC>(a.gZ + (size_t)r * f, ln, y);
                Lr = __ldg(a.L + (size_t)r * K + ln.h);
                if (slot < 0) {
                    // a row walked whole computes its D here; a split row's D came from gatv2_edge_delta_kernel
                    float z[8];
                    load8<VEC>(a.Z + (size_t)r * f, ln, z);
                    Dr = head_dot(y, z, ln);
                    if (ln.g == 0) a.aux[(size_t)r * K + ln.h] = Dr;
                } else {
                    Dr = a.aux[(size_t)r * K + ln.h];
                }
            }
            Soft st{-INFINITY, 0.0f};
            for (int eb = e0; eb < e1; eb += 32) {
                const int nb = min(32, e1 - eb);
                const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
                const int mine_g = dr.on && lane < nb ? __ldg(a.gid + mine) : 0;
#pragma unroll(W == kTrRows ? 1 : 2)
                for (int k = 0; k < nb; ++k) {
                    const int j = __shfl_sync(0xffffffffu, mine, k);
                    const int gj = __shfl_sync(0xffffffffu, mine_g, k);
                    const size_t e = (size_t)(eb + k);
                    float xl[8], lt[8];
                    const unsigned pos = edge_t<VEC>(a, b, j, e * f, ln, xr, xl, lt);
                    const float s = head_dot(at, lt, ln);
                    const float mk = mask(dr, gr, gj, ln.h);
                    if constexpr (W == kTrForward) {
                        soft_add(st, acc, s, mk, xl);
                    } else {
                        const float p = expf(__fsub_rn(s, Lr));
                        const float ds = __fmul_rn(p, __fsub_rn(__fmul_rn(mk, head_dot(y, xl, ln)), Dr));
                        const float P = __fmul_rn(p, mk);
                        float g[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float da = __fmul_rn(ds, at[q]);
                            g[q] = (pos >> q) & 1u ? da : __fmul_rn(da, b.slope);
                            acc[q] = __fadd_rn(acc[q], g[q]);
                            acc2[q] = __fmaf_rn(ds, lt[q], acc2[q]);
                        }
                        store8<VEC>(b.G + e * f, ln, g);
                        if (ln.g == 0) {
                            b.PS[e * 2 * K + ln.h] = P;
                            b.PS[e * 2 * K + K + ln.h] = ds;
                        }
                    }
                }
            }
            if constexpr (W == kTrForward) {
                if (slot < 0) {
                    finish_forward<VEC>(a, r, ln, st, acc);
                } else {
                    // a chunk of a split row: [acc | m | l], merged by gatv2_edge_forward_fixup_kernel
                    float* w = a.work + (size_t)slot * (f + 2 * K);
                    store8<false>(w, ln, acc);
                    if (ln.g == 0) {
                        w[f + ln.h] = st.m;
                        w[f + K + ln.h] = st.l;
                    }
                }
            }
        }
        if constexpr (W != kTrForward) {
            // a.scale is 1: finish_grad stores acc unchanged
            if (slot < 0) finish_grad<kTrRows, VEC>(a, r, ln, acc, acc2);
            else store8<false>(a.work + (size_t)slot * f, ln, acc);
        }
    }
    if constexpr (W == kTrRows) {
        // the CTA's datt partial: its warps' sums (0 for a warp without an item) added in warp order
        __shared__ float s_att[kTrWarps][kTrMaxF];
        store8<false>(s_att[threadIdx.x >> 5], ln, acc2);
        __syncthreads();
        for (int c = threadIdx.x; c < f; c += kTrThreads) {
            float s = s_att[0][c];
#pragma unroll
            for (int w = 1; w < kTrWarps; ++w) s = __fadd_rn(s, s_att[w][c]);
            b.part[(size_t)blockIdx.x * f + c] = s;
        }
    }
}

// datt[c] = the row walk's CTA partials summed in CTA order: one CTA per 32 features, kG2RedWarps warps each take
// every kG2RedWarps-th partial in increasing order, then warp 0 adds the warps' sums in warp order.
constexpr int kG2RedWarps = 32;

__global__ void __launch_bounds__(32 * kG2RedWarps)
gatv2_edge_datt_kernel(const float* __restrict__ part, int nparts, int f, float* __restrict__ datt)
{
    __shared__ float s[kG2RedWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    float acc = 0.0f;
    if (c < f)
        for (int i = w; i < nparts; i += kG2RedWarps) acc = __fadd_rn(acc, part[(size_t)i * f + c]);
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0 && c < f) {
        float t = s[0][lane];
#pragma unroll
        for (int k = 1; k < kG2RedWarps; ++k) t = __fadd_rn(t, s[k][lane]);
        datt[c] = t;
    }
}

// The split-row kernels (transformer_math.cuh), under this library's names.
__global__ void __launch_bounds__(kTrThreads) gatv2_edge_forward_fixup_kernel(TrArgs a) { forward_fixup(a); }

__global__ void __launch_bounds__(kTrThreads) gatv2_edge_sum_fixup_kernel(TrArgs a) { sum_fixup<kTrRows>(a); }

__global__ void __launch_bounds__(kTrThreads) gatv2_edge_delta_kernel(TrArgs a) { delta(a); }

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
    if (!w) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows,
                    (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)", what,
                    w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Sizes, width, heads and work: what every call takes.
int check_shape(const char* what, const pgcn_gated_walk* w, int32_t m, int32_t h, int32_t heads, int32_t f,
                const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (heads != 1 && heads != 2 && heads != 4 && heads != 8)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: heads=%d: the kernels take 1, 2, 4 or 8 heads", what, heads);
    if (f < 1 || f > kTrMaxF)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: f=%d outside [1, %d]: a row lives in registers", what, f,
                    kTrMaxF);
    if (f % heads)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: f=%d is not a multiple of heads=%d", what, f, heads);
    if (w->nslots > 0 && !work)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    return 0;
}

// The operands of the walks over the forward CSR: XL, XR, att, slope, E and the dropout.
int check_rows_operands(const char* what, const pgcn_gated_walk* w, int32_t m, int32_t h, const float* XL,
                        const float* XLh, const float* XR, const float* att, float slope, const float* E,
                        const int32_t* gid, const int64_t* drop, float keep_scale)
{
    if (m > 0 && (!XL || !XR)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null XL_own/XR", what);
    if (h > 0 && !XLh) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: h=%d but XL_halo is null", what, h);
    if (!att) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null att", what);
    if (!std::isfinite(slope)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: negative_slope is not finite", what);
    if (w->nitems > 0 && !E) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null E", what);
    if (drop && m + h > 0 && !gid) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: drop without gid", what);
    if (drop && !std::isfinite(keep_scale))
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: keep_scale is not finite", what);
    return 0;
}

// Last of the checks: a device to run on.
int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_GATV2_EDGE_ERR_NOGPU, "no CUDA device (%s): GATv2 attention with edge features has no CPU path",
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

TrArgs make_args(const pgcn_gated_walk* w, int32_t m, int32_t heads, int32_t f, const float* XR, const float* XL,
                 const float* XLh, const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                 float* work)
{
    TrArgs a{};
    a.items = reinterpret_cast<const int4*>(w->items);
    a.splits = w->splits;
    a.idx = w->idx;
    a.nitems = w->nitems; a.nsplits = w->nsplits; a.m = m; a.f = f; a.heads = heads;
    a.Q = XR; a.KV = XL; a.KVh = XLh; a.scale = 1.0f;
    a.gid = gid; a.drop = drop; a.threshold = threshold; a.keep_scale = keep_scale;
    a.work = work;
    return a;
}

unsigned warps_grid(int n) { return (unsigned)((n + kTrWarps - 1) / kTrWarps); }

int launched(const char* what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_GATV2_EDGE_ERR_CUDA, "%s launch: %s", what, cudaGetErrorString(e));
    return PGCN_GATV2_EDGE_OK;
}

// The walk, its vector instance when the head width and every feature operand allow it, then its fixup; the row
// walk ends with the datt reduction (datt = 0 when there is no item).
template <int W>
int launch(const TrArgs& a, const G2Args& b, float* datt, std::initializer_list<const void*> feats, void* stream)
{
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc;
    if (a.nitems == 0) {
        if (W == kTrRows && cudaMemsetAsync(datt, 0, (size_t)a.f * sizeof(float), s) != cudaSuccess)
            return launched("datt memset");
        return PGCN_GATV2_EDGE_OK;
    }
    if (W == kTrRows && a.nsplits > 0) {
        gatv2_edge_delta_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
        if ((rc = launched("gatv2_edge_delta_kernel"))) return rc;
    }
    const bool vec = (a.f / a.heads) % 4 == 0 && aligned16(feats);
    if (vec) gatv2_edge_walk_kernel<W, true><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a, b);
    else gatv2_edge_walk_kernel<W, false><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a, b);
    if ((rc = launched("gatv2_edge_walk_kernel"))) return rc;
    if (a.nsplits > 0) {
        if (W == kTrForward) {
            gatv2_edge_forward_fixup_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
            if ((rc = launched("gatv2_edge_forward_fixup_kernel"))) return rc;
        } else {
            gatv2_edge_sum_fixup_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
            if ((rc = launched("gatv2_edge_sum_fixup_kernel"))) return rc;
        }
    }
    if (W == kTrRows) {
        gatv2_edge_datt_kernel<<<(unsigned)((a.f + 31) / 32), 32 * kG2RedWarps, 0, s>>>(b.part, (int)warps_grid(a.nitems),
                                                                                          a.f, datt);
        return launched("gatv2_edge_datt_kernel");
    }
    return PGCN_GATV2_EDGE_OK;
}

template <int W>
void touch(int& rc)
{
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_walk_kernel<W, true>),
                          cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_walk_kernel<W, false>)})
        if (e != cudaSuccess && !rc)
            rc = fail(PGCN_GATV2_EDGE_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
}

}  // namespace

extern "C" {

const char* pgcn_gatv2_edge_version(void)
{
    return "pgcn_gatv2_edge 0.1 (sm_90a, fused GATv2 graph attention with edge features and attention dropout)";
}

const char* pgcn_gatv2_edge_last_error(void) { return g_error.c_str(); }

int64_t pgcn_gatv2_edge_work_rows(const pgcn_gated_walk* fwd)
{
    return fwd ? (int64_t)fwd->nslots + warps_grid(fwd->nitems) : -1;
}

int pgcn_gatv2_edge_load(void)
{
    static bool loaded[256] = {};
    int rc = check_device();
    if (rc) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && loaded[dev]) return PGCN_GATV2_EDGE_OK;
    touch<kTrForward>(rc);
    touch<kTrRows>(rc);
    touch<kTrCols>(rc);
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_forward_fixup_kernel),
                          cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_sum_fixup_kernel),
                          cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_delta_kernel),
                          cudaFuncGetAttributes(&fa, (const void*)gatv2_edge_datt_kernel)})
        if (e != cudaSuccess && !rc)
            rc = fail(PGCN_GATV2_EDGE_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
    if (!rc && dev >= 0 && dev < 256) loaded[dev] = true;
    return rc;
}

int pgcn_gatv2_edge_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* XL_own,
                            const float* XL_halo, const float* XR, const float* att, const float* E,
                            float negative_slope, const int32_t* gid, const int64_t* drop, uint32_t threshold,
                            float keep_scale, float* Z, float* L, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_gatv2_edge_forward";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_shape(what, fwd, m, h, heads, f, work)) ||
        (rc = check_rows_operands(what, fwd, m, h, XL_own, XL_halo, XR, att, negative_slope, E, gid, drop,
                                  keep_scale)))
        return rc;
    if (m > 0 && (!Z || !L)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null Z/L output", what);
    if ((rc = check_device())) return rc;
    XL_halo = h > 0 ? XL_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, XR, XL_own, XL_halo, gid, drop, threshold, keep_scale, work);
    a.out = Z;
    a.aux = L;
    G2Args b{};
    b.att = att; b.slope = negative_slope; b.E = E;
    return launch<kTrForward>(a, b, nullptr, {XL_own, XL_halo, XR, att, E, Z}, stream);
}

int pgcn_gatv2_edge_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                  const float* XL_own, const float* XL_halo, const float* XR, const float* att,
                                  const float* E, float negative_slope, const int32_t* gid, const int64_t* drop,
                                  uint32_t threshold, float keep_scale, const float* gZ, const float* Z,
                                  const float* L, float* dXR, float* D, float* PS, float* G, float* datt, float* work,
                                  int32_t f, void* stream)
{
    const char* what = "pgcn_gatv2_edge_backward_rows";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_shape(what, fwd, m, h, heads, f, work)) ||
        (rc = check_rows_operands(what, fwd, m, h, XL_own, XL_halo, XR, att, negative_slope, E, gid, drop,
                                  keep_scale)))
        return rc;
    if (m > 0 && (!gZ || !Z || !L)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null gZ/Z/L", what);
    if (m > 0 && (!dXR || !D)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null dXR/D output", what);
    if (fwd->nitems > 0 && (!PS || !G)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null PS/G output", what);
    if (!datt) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null datt output", what);
    if (fwd->nitems > 0 && !work)
        return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null work (it holds the datt partials)", what);
    if ((rc = check_device())) return rc;
    XL_halo = h > 0 ? XL_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, XR, XL_own, XL_halo, gid, drop, threshold, keep_scale, work);
    a.gZ = gZ; a.Z = Z; a.L = L;
    a.out = dXR;
    a.aux = D;
    G2Args b{};
    b.att = att; b.slope = negative_slope; b.E = E; b.G = G; b.PS = PS;
    b.part = work ? work + (size_t)fwd->nslots * f : nullptr;
    return launch<kTrRows>(a, b, datt, {XL_own, XL_halo, XR, att, E, gZ, Z, dXR, G}, stream);
}

int pgcn_gatv2_edge_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, int32_t heads,
                                  const float* gZ, const float* PS, const float* G, float* dXL, float* work, int32_t f,
                                  void* stream)
{
    const char* what = "pgcn_gatv2_edge_backward_cols";
    int rc = check_walk(tr, (int64_t)m + h, what);
    if (rc || (rc = check_shape(what, tr, m, h, heads, f, work))) return rc;
    if (tr->rows > 0 && !perm) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null perm", what);
    if (m > 0 && !gZ) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null gZ", what);
    if (tr->nitems > 0 && (!PS || !G)) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null PS/G", what);
    if ((int64_t)m + h > 0 && !dXL) return fail(PGCN_GATV2_EDGE_ERR_INVALID, "%s: null dXL output", what);
    if ((rc = check_device())) return rc;
    TrArgs a = make_args(tr, m, heads, f, nullptr, nullptr, nullptr, nullptr, nullptr, 0u, 1.0f, work);
    a.gZ = gZ;
    a.out = dXL;
    G2Args b{};
    b.Gc = G; b.PSc = PS; b.perm = perm;
    return launch<kTrCols>(a, b, nullptr, {gZ, G, dXL}, stream);
}

}  // extern "C"
