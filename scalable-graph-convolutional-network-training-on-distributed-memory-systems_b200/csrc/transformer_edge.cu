// Graph transformer attention with edge features (include/pgcn_transformer_edge.h): TransformerConv's attention with
// an edge term added to the keys and values, and its two backward walks, over the gated aggregation's work tables.
//
// The lane layout, online softmax and split-row fixups are the transformer's (transformer_math.cuh). Per entry:
//   forward     [k | v][j] gathered, E_e streamed (64-bit offsets)           -> online softmax on kk, vv  -> Z, L
//   row walk    [k | v][j] gathered, E_e streamed, p = expf(s - L)           -> dE_e, PS_e = [P | ds]     -> dQ, D
//   column walk q[i], gZ[i] gathered, PS_p read (p = perm[t], 8K bytes)      -> [dK | dV]
// The column walk recomputes no score: the row walk has stored each entry's P = M p and ds, 2K floats, where a
// recomputation would need the entry's f-wide E through the same scattered permutation. A row walked whole is finished
// in its warp; the chunks of a split row write their partials to the caller's work rows and a fixup warp per split row
// merges them in chunk order. Every output element is reduced in one fixed order, without atomics.
#include "../../include/pgcn_transformer_edge.h"
#include "transformer_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <initializer_list>
#include <string>

namespace pgcn {

// The per-entry operands beside the transformer's.
struct EdgeArgs {
    const float* E;            // nnz x f (forward, row walk)
    float* dE;                 // nnz x f or null (row walk)
    float* PS;                 // nnz x 2K: written by the row walk
    const float* PSc;          // the same, read by the column walk
    const int32_t* perm;       // column walk: forward entry of each transposed entry
};

// kk = k[j] + E_e and vv = v[j] + E_e on this lane's slots (unused slots stay 0 + 0).
template <bool VEC>
__device__ __forceinline__ void edge_kv(const TrArgs& a, const EdgeArgs& b, int j, size_t pe, const Lanes& ln,
                                        float (&kk)[8], float (&vv)[8])
{
    const float* kv = kv_row(a, j);
    float e[8];
    load8<VEC>(kv, ln, kk);
    load8<VEC>(kv + a.f, ln, vv);
    load8<VEC>(b.E + pe, ln, e);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        kk[u] = __fadd_rn(kk[u], e[u]);
        vv[u] = __fadd_rn(vv[u], e[u]);
    }
}

template <int W, bool VEC>
__global__ void __launch_bounds__(kTrThreads) transformer_edge_walk_kernel(TrArgs a, EdgeArgs b)
{
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    if (item >= a.nitems) return;
    const int4 it = __ldg(a.items + item);               // (row, e0, e1, slot)
    const int r = it.x, e0 = it.y, e1 = it.z, slot = it.w;
    const int f = a.f, K = a.heads;
    const Lanes ln = lanes(lane, f, K);
    float acc[8] = {}, acc2[8] = {};
    if constexpr (W == kTrCols) {
        for (int eb = e0; eb < e1; eb += 32) {
            const int nb = min(32, e1 - eb);
            const int mine = lane < nb ? __ldg(a.idx + eb + lane) : 0;
            const int mperm = lane < nb ? __ldg(b.perm + eb + lane) : 0;
#pragma unroll 2
            for (int k = 0; k < nb; ++k) {
                const int i = __shfl_sync(0xffffffffu, mine, k);
                const size_t pe = (size_t)__shfl_sync(0xffffffffu, mperm, k) * 2 * K;
                const float P = __ldg(b.PSc + pe + ln.h), ds = __ldg(b.PSc + pe + K + ln.h);
                float u[8], v[8];                // q[i], gZ[i]
                load8<VEC>(a.Q + (size_t)i * f, ln, u);
                load8<VEC>(a.gZ + (size_t)i * f, ln, v);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    acc[q] = __fmaf_rn(ds, u[q], acc[q]);
                    acc2[q] = __fmaf_rn(P, v[q], acc2[q]);
                }
            }
        }
    } else {
        const Drop dr = drop_state(a);
        const int gr = dr.on ? __ldg(a.gid + r) : 0;
        float x[8], y[8];                    // q[r]; gZ[r] in the row walk
        load8<VEC>(a.Q + (size_t)r * f, ln, x);
        float Lr = 0.0f, Dr = 0.0f;
        if constexpr (W == kTrRows) {
            load8<VEC>(a.gZ + (size_t)r * f, ln, y);
            Lr = __ldg(a.L + (size_t)r * K + ln.h);
            if (slot < 0) {
                // a row walked whole computes its D here; a split row's D came from transformer_edge_delta_kernel
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
#pragma unroll 2
            for (int k = 0; k < nb; ++k) {
                const int j = __shfl_sync(0xffffffffu, mine, k);
                const int gj = __shfl_sync(0xffffffffu, mine_g, k);
                const size_t e = (size_t)(eb + k);
                float u[8], v[8];                // kk_e, vv_e
                edge_kv<VEC>(a, b, j, e * f, ln, u, v);
                const float s = __fmul_rn(head_dot(x, u, ln), a.scale);
                const float mk = mask(dr, gr, gj, ln.h);
                if constexpr (W == kTrForward) {
                    soft_add(st, acc, s, mk, v);
                } else {
                    const float p = expf(__fsub_rn(s, Lr));
                    const float ds = __fmul_rn(p, __fsub_rn(__fmul_rn(mk, head_dot(y, v, ln)), Dr));
                    const float P = __fmul_rn(p, mk);
#pragma unroll
                    for (int q = 0; q < 8; ++q) acc[q] = __fmaf_rn(ds, u[q], acc[q]);
                    if (b.dE) {
                        const float sds = __fmul_rn(a.scale, ds);
                        float d[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) d[q] = __fmaf_rn(sds, x[q], __fmul_rn(P, y[q]));
                        store8<VEC>(b.dE + e * f, ln, d);
                    }
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
                // a chunk of a split row: [acc | m | l], merged by transformer_edge_forward_fixup_kernel
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
        if (slot < 0) {
            finish_grad<W, VEC>(a, r, ln, acc, acc2);
        } else {
            const int ow = W == kTrCols ? 2 * f : f;
            store8<false>(a.work + (size_t)slot * ow, ln, acc);
            if constexpr (W == kTrCols) store8<false>(a.work + (size_t)slot * ow + f, ln, acc2);
        }
    }
}

// The split-row kernels (transformer_math.cuh), under this library's names.
__global__ void __launch_bounds__(kTrThreads) transformer_edge_forward_fixup_kernel(TrArgs a) { forward_fixup(a); }

template <int W>
__global__ void __launch_bounds__(kTrThreads) transformer_edge_sum_fixup_kernel(TrArgs a) { sum_fixup<W>(a); }

__global__ void __launch_bounds__(kTrThreads) transformer_edge_delta_kernel(TrArgs a) { delta(a); }

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
    if (!w) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null walk", what);
    if (w->rows != rows)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: the walk has %d rows, expected %lld", what, w->rows,
                    (long long)rows);
    if (w->nitems < w->rows || w->nsplits < 0 || w->nslots < 0)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: bad work table (rows=%d nitems=%d nsplits=%d nslots=%d)",
                    what, w->rows, w->nitems, w->nsplits, w->nslots);
    if ((w->nitems > 0 && (!w->items || !w->idx)) || (w->nsplits > 0 && !w->splits))
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null idx/items/splits", what);
    return 0;
}

// Sizes, width, heads, scale and work: what every call takes.
int check_shape(const char* what, const pgcn_gated_walk* w, int32_t m, int32_t h, int32_t heads, int32_t f,
                float scale, const float* work)
{
    if (m < 0 || h < 0) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: bad sizes m=%d h=%d", what, m, h);
    if (heads != 1 && heads != 2 && heads != 4 && heads != 8)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: heads=%d: the kernels take 1, 2, 4 or 8 heads", what,
                    heads);
    if (f < 1 || f > kTrMaxF)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: f=%d outside [1, %d]: a row lives in registers", what, f,
                    kTrMaxF);
    if (f % heads)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: f=%d is not a multiple of heads=%d", what, f, heads);
    if (!std::isfinite(scale)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: scale is not finite", what);
    if (w->nslots > 0 && !work)
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: nslots=%d but work is null", what, w->nslots);
    return 0;
}

// The operands of the walks over the forward CSR: q, [k | v], E and the dropout.
int check_rows_operands(const char* what, const pgcn_gated_walk* w, int32_t m, int32_t h, const float* Q,
                        const float* KV, const float* KVh, const float* E, const int32_t* gid, const int64_t* drop,
                        float keep_scale)
{
    if (m > 0 && (!Q || !KV)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null Q_own/KV_own", what);
    if (h > 0 && !KVh) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: h=%d but KV_halo is null", what, h);
    if (w->nitems > 0 && !E) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null E", what);
    if (drop && m + h > 0 && !gid) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: drop without gid", what);
    if (drop && !std::isfinite(keep_scale))
        return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: keep_scale is not finite", what);
    return 0;
}

// Last of the checks: a device to run on.
int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_TRANSFORMER_EDGE_ERR_NOGPU,
                    "no CUDA device (%s): transformer attention with edge features has no CPU path",
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
    if (e != cudaSuccess) return fail(PGCN_TRANSFORMER_EDGE_ERR_CUDA, "%s launch: %s", what, cudaGetErrorString(e));
    return PGCN_TRANSFORMER_EDGE_OK;
}

// The walk, its vector instance when the head width and every feature operand allow it, then its fixup.
template <int W>
int launch(const TrArgs& a, const EdgeArgs& b, std::initializer_list<const void*> feats, void* stream)
{
    if (a.nitems == 0) return PGCN_TRANSFORMER_EDGE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc;
    if (W == kTrRows && a.nsplits > 0) {
        transformer_edge_delta_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
        if ((rc = launched("transformer_edge_delta_kernel"))) return rc;
    }
    const bool vec = (a.f / a.heads) % 4 == 0 && aligned16(feats);
    if (vec) transformer_edge_walk_kernel<W, true><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a, b);
    else transformer_edge_walk_kernel<W, false><<<warps_grid(a.nitems), kTrThreads, 0, s>>>(a, b);
    if ((rc = launched("transformer_edge_walk_kernel"))) return rc;
    if (a.nsplits > 0) {
        if (W == kTrForward) {
            transformer_edge_forward_fixup_kernel<<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
            return launched("transformer_edge_forward_fixup_kernel");
        }
        transformer_edge_sum_fixup_kernel<W == kTrForward ? kTrRows : W>
            <<<warps_grid(a.nsplits), kTrThreads, 0, s>>>(a);
        return launched("transformer_edge_sum_fixup_kernel");
    }
    return PGCN_TRANSFORMER_EDGE_OK;
}

template <int W>
void touch(int& rc)
{
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)transformer_edge_walk_kernel<W, true>),
                          cudaFuncGetAttributes(&fa, (const void*)transformer_edge_walk_kernel<W, false>)})
        if (e != cudaSuccess && !rc)
            rc = fail(PGCN_TRANSFORMER_EDGE_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
}

}  // namespace

extern "C" {

const char* pgcn_transformer_edge_version(void)
{
    return "pgcn_transformer_edge 0.1 (sm_90a, fused scaled dot-product graph attention with edge features)";
}

const char* pgcn_transformer_edge_last_error(void) { return g_error.c_str(); }

int pgcn_transformer_edge_load(void)
{
    static bool loaded[256] = {};
    int rc = check_device();
    if (rc) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && loaded[dev]) return PGCN_TRANSFORMER_EDGE_OK;
    touch<kTrForward>(rc);
    touch<kTrRows>(rc);
    touch<kTrCols>(rc);
    cudaFuncAttributes fa;
    for (cudaError_t e : {cudaFuncGetAttributes(&fa, (const void*)transformer_edge_forward_fixup_kernel),
                          cudaFuncGetAttributes(&fa, (const void*)transformer_edge_sum_fixup_kernel<kTrRows>),
                          cudaFuncGetAttributes(&fa, (const void*)transformer_edge_sum_fixup_kernel<kTrCols>),
                          cudaFuncGetAttributes(&fa, (const void*)transformer_edge_delta_kernel)})
        if (e != cudaSuccess && !rc)
            rc = fail(PGCN_TRANSFORMER_EDGE_ERR_CUDA, "loading the kernels: %s", cudaGetErrorString(e));
    if (!rc && dev >= 0 && dev < 256) loaded[dev] = true;
    return rc;
}

int pgcn_transformer_edge_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* Q_own,
                                  const float* KV_own, const float* KV_halo, const float* E, float scale,
                                  const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                  float* Z, float* L, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_transformer_edge_forward";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_shape(what, fwd, m, h, heads, f, scale, work)) ||
        (rc = check_rows_operands(what, fwd, m, h, Q_own, KV_own, KV_halo, E, gid, drop, keep_scale)))
        return rc;
    if (m > 0 && (!Z || !L)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null Z/L output", what);
    if ((rc = check_device())) return rc;
    KV_halo = h > 0 ? KV_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, work);
    a.out = Z;
    a.aux = L;
    EdgeArgs b{};
    b.E = E;
    return launch<kTrForward>(a, b, {Q_own, KV_own, KV_halo, E, Z}, stream);
}

int pgcn_transformer_edge_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                        const float* Q_own, const float* KV_own, const float* KV_halo, const float* E,
                                        float scale, const int32_t* gid, const int64_t* drop, uint32_t threshold,
                                        float keep_scale, const float* gZ, const float* Z, const float* L, float* dQ,
                                        float* D, float* PS, float* dE, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_transformer_edge_backward_rows";
    int rc = check_walk(fwd, m, what);
    if (rc || (rc = check_shape(what, fwd, m, h, heads, f, scale, work)) ||
        (rc = check_rows_operands(what, fwd, m, h, Q_own, KV_own, KV_halo, E, gid, drop, keep_scale)))
        return rc;
    if (m > 0 && (!gZ || !Z || !L)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null gZ/Z/L", what);
    if (m > 0 && (!dQ || !D)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null dQ/D output", what);
    if (fwd->nitems > 0 && !PS) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null PS output", what);
    if ((rc = check_device())) return rc;
    KV_halo = h > 0 ? KV_halo : nullptr;
    TrArgs a = make_args(fwd, m, heads, f, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, work);
    a.gZ = gZ; a.Z = Z; a.L = L;
    a.out = dQ;
    a.aux = D;
    EdgeArgs b{};
    b.E = E; b.dE = dE; b.PS = PS;
    return launch<kTrRows>(a, b, {Q_own, KV_own, KV_halo, E, gZ, Z, dQ, dE}, stream);
}

int pgcn_transformer_edge_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h,
                                        int32_t heads, const float* Q_own, const float* gZ, const float* PS,
                                        float scale, float* dKV, float* work, int32_t f, void* stream)
{
    const char* what = "pgcn_transformer_edge_backward_cols";
    int rc = check_walk(tr, (int64_t)m + h, what);
    if (rc || (rc = check_shape(what, tr, m, h, heads, f, scale, work))) return rc;
    if (tr->rows > 0 && !perm) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null perm", what);
    if (m > 0 && (!Q_own || !gZ || !PS)) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null Q_own/gZ/PS", what);
    if ((int64_t)m + h > 0 && !dKV) return fail(PGCN_TRANSFORMER_EDGE_ERR_INVALID, "%s: null dKV output", what);
    if ((rc = check_device())) return rc;
    TrArgs a = make_args(tr, m, heads, f, Q_own, nullptr, nullptr, scale, nullptr, nullptr, 0u, 1.0f, work);
    a.gZ = gZ;
    a.out = dKV;
    EdgeArgs b{};
    b.PSc = PS; b.perm = perm;
    return launch<kTrCols>(a, b, {Q_own, gZ, dKV}, stream);
}

}  // extern "C"
