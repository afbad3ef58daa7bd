// attention.cuh — sm_90a kernels of the edge softmax of sparse graph attention (GPU/PGAT.py:139-148 over the stored
// pattern of the local matrix instead of a dense n x n score matrix), with K = 1, 2, 4 or 8 heads.
//
// With el (destination side, one per owned row and head) and er (source side, one per column and head: owned rows,
// then the halo rows), for every head h
//     s_eh     = LeakyReLU(el[row(e), h] + er[col(e), h], slope)
//     alpha_eh = exp(s_eh - max_row s_.h) / sum_row exp(s_.h - max_row s_.h)          over the stored entries of row(e)
// and, given dalpha (the SDDMM of the output gradient against the aggregated rows, per head),
//     c_ih     = sum_row(i) alpha_.h * dalpha_.h
//     dpre_eh  = alpha_eh (dalpha_eh - c_row(e)h) * (s_eh > 0 ? 1 : slope)
//     d_el[i, h] = sum_row(i) dpre_.h
// Every array is row-major and head-minor ([m, K], [h, K], [nnz, K]); entries are in forward CSR order, the order
// pgcn_plan_set_values takes. Columns come from the forward records (entry e is word (e >> 5) * kPieceInts + (e & 31)),
// rows from the device rowptr pgcn_plan_bind_values keeps. K = 1 is the single-head layer.
//
//   edge_softmax_kernel<K, VEC>   / edge_softmax_backward_kernel<K, VEC>
//   edge_softmax_raw_kernel<K, VEC> / edge_softmax_raw_backward_kernel<K, VEC>   the same rows over scores already stored
//                                 in `out` (GATv2), in place; the backward has no slope factor and no d_el
// One launch serves every row. Blocks [0, nlong) take one long row each (more than kAttnLongRow entries: the hub rows
// of R-MAT graphs, which would set the launch time if one warp walked them); every later block gives one warp to each
// of 8 consecutive rows and skips the long ones. Lanes stride over their row's entries; one gather of a column brings
// its K er values (VEC: one 4- to 32-byte vector load, when every [., K] operand is aligned to it), and a lane keeps K
// partials. The per-lane partials are merged by an xor butterfly (every lane ends with the same bits) and, in a long
// row, the warps' results by every thread in warp order. The forward takes the row maximum in a pass of its own and
// sums the exponentials in a second one: a running (max, sum) pair would chain every entry's exponential to the
// previous one and keep the er gathers of a lane from overlapping (0.50 ms on C2 at 700 W, against 0.2 ms aimed at).
// No atomics: two runs are bit-identical. expf is the full-precision one, and the row maximum is always subtracted, so
// rows of any length and scores of any size stay finite.
#pragma once
#include "spmm_kernels.cuh"

namespace pgcn {

constexpr int kAttnThreads = 256;
constexpr int kAttnWarps = kAttnThreads / 32;
constexpr int kAttnLongRow = 1024;           // rows with more entries get a whole CTA

struct AttnArgs {
    const int* rowptr;       // m + 1, forward CSR
    const int* long_rows;    // rows with more than kAttnLongRow entries, ascending
    int nlong;
    int m;
    const int* pieces;       // the forward matrix's records
    const float* el;         // m x K
    const float* er_own;     // m x K
    const float* er_halo;    // h x K (null when h == 0)
    float slope;
    const float* alpha;      // backward: nnz x K
    const float* dalpha;     // backward: nnz x K
    float* out;              // forward: alpha; backward: dpre (nnz x K)
    float* d_el;             // backward: m x K
};

// K consecutive floats: VEC reads them as float2 / float4 vectors (the caller checked the alignment), else one by one.
// RO: read-only for the whole launch (the non-coherent path); the forward reads back its own scores without it.
template <int K, bool VEC, bool RO>
__device__ __forceinline__ void ld_heads(float (&x)[K], const float* p)
{
    if constexpr (VEC && K == 2) {
        const float2 v = RO ? __ldg(reinterpret_cast<const float2*>(p)) : *reinterpret_cast<const float2*>(p);
        x[0] = v.x; x[1] = v.y;
    } else if constexpr (VEC && K >= 4) {
#pragma unroll
        for (int q = 0; q < K / 4; ++q) {
            const float4 v = RO ? __ldg(reinterpret_cast<const float4*>(p) + q) : reinterpret_cast<const float4*>(p)[q];
            x[4 * q] = v.x; x[4 * q + 1] = v.y; x[4 * q + 2] = v.z; x[4 * q + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int h = 0; h < K; ++h) x[h] = RO ? __ldg(p + h) : p[h];
    }
}

template <int K, bool VEC>
__device__ __forceinline__ void st_heads(float* p, const float (&x)[K])
{
    if constexpr (VEC && K == 2) {
        *reinterpret_cast<float2*>(p) = make_float2(x[0], x[1]);
    } else if constexpr (VEC && K >= 4) {
#pragma unroll
        for (int q = 0; q < K / 4; ++q)
            reinterpret_cast<float4*>(p)[q] = make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]);
    } else {
#pragma unroll
        for (int h = 0; h < K; ++h) p[h] = x[h];
    }
}

// the K scores of entry e of a row whose el values are eli
template <int K, bool VEC>
__device__ __forceinline__ void attn_score(const AttnArgs& a, const float (&eli)[K], int e, float (&x)[K])
{
    const int col = __ldg(a.pieces + (size_t)(e >> 5) * kPieceInts + (e & 31));
    if constexpr (K == 1) {
        x[0] = eli[0] + (col < a.m ? __ldg(a.er_own + col) : __ldg(a.er_halo + (col - a.m)));
    } else {
        ld_heads<K, VEC, true>(x, col < a.m ? a.er_own + (size_t)col * K : a.er_halo + (size_t)(col - a.m) * K);
#pragma unroll
        for (int h = 0; h < K; ++h) x[h] = eli[h] + x[h];
    }
#pragma unroll
    for (int h = 0; h < K; ++h) x[h] = x[h] > 0.f ? x[h] : x[h] * a.slope;
}

__device__ __forceinline__ float sum_warp(float x)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// the per-head partials of a row's NT threads: butterfly within each warp, then (NT = a CTA) the warps in warp order
template <int NT, int K>
__device__ __forceinline__ void sum_row(float (&x)[K], float (&sm)[kAttnWarps][K], int t)
{
#pragma unroll
    for (int h = 0; h < K; ++h) x[h] = sum_warp(x[h]);
    if (NT > 32) {
        if ((t & 31) == 0) {
#pragma unroll
            for (int h = 0; h < K; ++h) sm[t >> 5][h] = x[h];
        }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < K; ++h) {
            x[h] = sm[0][h];
            for (int w = 1; w < NT / 32; ++w) x[h] += sm[w][h];
        }
    }
}

// One row, walked by NT threads (t = this thread's index among them). Long rows (NT = a CTA) combine the warps'
// results through shared memory in warp order. RAW: `out` already holds the scores (GATv2), el / er are not read.
template <int NT, int K, bool VEC, bool RAW = false>
__device__ __forceinline__ void softmax_row(const AttnArgs& a, int i, int t)
{
    __shared__ float sm_m[kAttnWarps][K], sm_s[kAttnWarps][K];
    const int b = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
    float eli[K];
    if constexpr (!RAW) ld_heads<K, VEC, true>(eli, a.el + (size_t)i * K);
    float* __restrict__ out = a.out;
    // pass 1: the scores (kept in `out`, read back by this thread) and the row maxima. No exponential here, so the
    // gathers of consecutive entries do not wait for each other.
    float m[K];
#pragma unroll
    for (int h = 0; h < K; ++h) m[h] = -INFINITY;
#pragma unroll 4
    for (int e = b + t; e < end; e += NT) {
        float x[K];
        if constexpr (RAW) {
            ld_heads<K, VEC, false>(x, out + (size_t)e * K);
        } else {
            attn_score<K, VEC>(a, eli, e, x);
            st_heads<K, VEC>(out + (size_t)e * K, x);
        }
#pragma unroll
        for (int h = 0; h < K; ++h) m[h] = fmaxf(m[h], x[h]);
    }
#pragma unroll
    for (int h = 0; h < K; ++h)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], o));
    if (NT > 32) {
        if ((t & 31) == 0) {
#pragma unroll
            for (int h = 0; h < K; ++h) sm_m[t >> 5][h] = m[h];
        }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < K; ++h) {
            m[h] = sm_m[0][h];
            for (int w = 1; w < NT / 32; ++w) m[h] = fmaxf(m[h], sm_m[w][h]);
        }
    }
    // pass 2: the sums of exp(s - max), per lane in entry order, then in one fixed butterfly / warp order
    float s[K];
#pragma unroll
    for (int h = 0; h < K; ++h) s[h] = 0.f;
#pragma unroll 4
    for (int e = b + t; e < end; e += NT) {
        float x[K];
        ld_heads<K, VEC, false>(x, out + (size_t)e * K);
#pragma unroll
        for (int h = 0; h < K; ++h) s[h] += expf(x[h] - m[h]);
    }
    sum_row<NT, K>(s, sm_s, t);
    for (int e = b + t; e < end; e += NT) {
        float x[K];
        ld_heads<K, VEC, false>(x, out + (size_t)e * K);
#pragma unroll
        for (int h = 0; h < K; ++h) x[h] = expf(x[h] - m[h]) / s[h];
        st_heads<K, VEC>(out + (size_t)e * K, x);
    }
}

// RAW: dscore = alpha (dalpha - c) without the slope factor and d_el, written over dalpha (out == dalpha is allowed:
// each entry is read and rewritten by one thread, so dalpha takes the coherent path).
template <int NT, int K, bool VEC, bool RAW = false>
__device__ __forceinline__ void softmax_backward_row(const AttnArgs& a, int i, int t)
{
    __shared__ float sm_x[kAttnWarps][K];
    const int b = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
    float c[K];
#pragma unroll
    for (int h = 0; h < K; ++h) c[h] = 0.f;
    for (int e = b + t; e < end; e += NT) {
        float al[K], da[K];
        ld_heads<K, VEC, true>(al, a.alpha + (size_t)e * K);
        ld_heads<K, VEC, !RAW>(da, a.dalpha + (size_t)e * K);
#pragma unroll
        for (int h = 0; h < K; ++h) c[h] = fmaf(al[h], da[h], c[h]);
    }
    sum_row<NT, K>(c, sm_x, t);
    if constexpr (RAW) {
        for (int e = b + t; e < end; e += NT) {
            float al[K], da[K];
            ld_heads<K, VEC, true>(al, a.alpha + (size_t)e * K);
            ld_heads<K, VEC, false>(da, a.dalpha + (size_t)e * K);
#pragma unroll
            for (int h = 0; h < K; ++h) da[h] = al[h] * (da[h] - c[h]);
            st_heads<K, VEC>(a.out + (size_t)e * K, da);
        }
        return;
    }
    if (NT > 32) __syncthreads();                           // sm_x is reused below
    float eli[K];
    ld_heads<K, VEC, true>(eli, a.el + (size_t)i * K);
    float d[K];
#pragma unroll
    for (int h = 0; h < K; ++h) d[h] = 0.f;
    for (int e = b + t; e < end; e += NT) {
        float x[K], al[K], da[K], g[K];
        attn_score<K, VEC>(a, eli, e, x);
        ld_heads<K, VEC, true>(al, a.alpha + (size_t)e * K);
        ld_heads<K, VEC, true>(da, a.dalpha + (size_t)e * K);
#pragma unroll
        for (int h = 0; h < K; ++h) {
            g[h] = al[h] * (da[h] - c[h]) * (x[h] > 0.f ? 1.f : a.slope);
            d[h] += g[h];
        }
        st_heads<K, VEC>(a.out + (size_t)e * K, g);
    }
    sum_row<NT, K>(d, sm_x, t);
    if (t == 0) {
#pragma unroll
        for (int h = 0; h < K; ++h) a.d_el[(size_t)i * K + h] = d[h];
    }
}

__device__ __forceinline__ bool attn_short_row(const AttnArgs& a, int& i)
{
    i = (int)(blockIdx.x - (unsigned)a.nlong) * kAttnWarps + (int)(threadIdx.x >> 5);
    return i < a.m && __ldg(a.rowptr + i + 1) - __ldg(a.rowptr + i) <= kAttnLongRow;
}

template <int K, bool VEC>
__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_row<kAttnThreads, K, VEC>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_row<32, K, VEC>(a, i, threadIdx.x & 31);
}

template <int K, bool VEC>
__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_backward_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_backward_row<kAttnThreads, K, VEC>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_backward_row<32, K, VEC>(a, i, threadIdx.x & 31);
}

// The edge softmax of stored scores (GATv2: the score kernel wrote them into `out`), in place: the same rows, passes,
// orders and bits as edge_softmax_kernel once the scores are there.
template <int K, bool VEC>
__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_raw_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_row<kAttnThreads, K, VEC, true>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_row<32, K, VEC, true>(a, i, threadIdx.x & 31);
}

// dscore = alpha (dalpha - sum_row alpha dalpha) per head, in place over dalpha (out == dalpha).
template <int K, bool VEC>
__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_raw_backward_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_backward_row<kAttnThreads, K, VEC, true>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_backward_row<32, K, VEC, true>(a, i, threadIdx.x & 31);
}

}  // namespace pgcn
