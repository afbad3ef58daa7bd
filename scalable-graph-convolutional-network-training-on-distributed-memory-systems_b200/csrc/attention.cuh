// attention.cuh — sm_90a kernels of the edge softmax of sparse graph attention (GPU/PGAT.py:139-148 over the stored
// pattern of the local matrix instead of a dense n x n score matrix).
//
// With el (destination side, one per owned row) and er (source side, one per column: owned rows, then the halo rows)
//     s_e     = LeakyReLU(el[row(e)] + er[col(e)], slope)
//     alpha_e = exp(s_e - max_row s) / sum_row exp(s - max_row s)          over the stored entries of row(e)
// and, given dalpha (the SDDMM of the output gradient against the aggregated rows),
//     c_i     = sum_row(i) alpha * dalpha
//     dpre_e  = alpha_e (dalpha_e - c_row(e)) * (s_e > 0 ? 1 : slope)
//     d_el[i] = sum_row(i) dpre
// Both outputs are in forward CSR order, the order pgcn_plan_set_values takes. Columns come from the forward records
// (entry e is word (e >> 5) * kPieceInts + (e & 31)), rows from the device rowptr pgcn_plan_bind_values keeps.
//
//   edge_softmax_kernel           / edge_softmax_backward_kernel
// One launch serves every row. Blocks [0, nlong) take one long row each (more than kAttnLongRow entries: the hub rows
// of R-MAT graphs, which would set the launch time if one warp walked them); every later block gives one warp to each
// of 8 consecutive rows and skips the long ones. Lanes stride over their row's entries; the per-lane partials are
// merged by an xor butterfly (every lane ends with the same bits) and, in a long row, the warps' results by every
// thread in warp order. The forward takes the row maximum in a pass of its own and sums the exponentials in a second
// one: a running (max, sum) pair would chain every entry's exponential to the previous one and keep the er gathers
// of a lane from overlapping (0.50 ms on C2 at 700 W, against 0.2 ms aimed at). No atomics: two runs are
// bit-identical. expf is the full-precision one, and the row maximum is always subtracted, so rows of any length and
// scores of any size stay finite.
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
    const float* el;         // m
    const float* er_own;     // m
    const float* er_halo;    // h (null when h == 0)
    float slope;
    const float* alpha;      // backward: nnz
    const float* dalpha;     // backward: nnz
    float* out;              // forward: alpha; backward: dpre (nnz)
    float* d_el;             // backward: m
};

__device__ __forceinline__ float attn_score(const AttnArgs& a, float eli, int e)
{
    const int col = __ldg(a.pieces + (size_t)(e >> 5) * kPieceInts + (e & 31));
    const float x = eli + (col < a.m ? __ldg(a.er_own + col) : __ldg(a.er_halo + (col - a.m)));
    return x > 0.f ? x : x * a.slope;
}

__device__ __forceinline__ float sum_warp(float x)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// One row, walked by NT threads (t = this thread's index among them). Long rows (NT = a CTA) combine the warps'
// results through shared memory in warp order.
template <int NT>
__device__ __forceinline__ void softmax_row(const AttnArgs& a, int i, int t)
{
    __shared__ float sm_m[kAttnWarps], sm_s[kAttnWarps];
    const int b = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
    const float eli = __ldg(a.el + i);
    float* __restrict__ out = a.out;
    // pass 1: the scores (kept in `out`, read back by this thread) and the row maximum. No exponential here, so the
    // gathers of consecutive entries do not wait for each other.
    float m = -INFINITY;
#pragma unroll 4
    for (int e = b + t; e < end; e += NT) {
        const float x = attn_score(a, eli, e);
        out[e] = x;
        m = fmaxf(m, x);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (NT > 32) {
        if ((t & 31) == 0) sm_m[t >> 5] = m;
        __syncthreads();
        m = sm_m[0];
        for (int w = 1; w < NT / 32; ++w) m = fmaxf(m, sm_m[w]);
    }
    // pass 2: the sum of exp(s - max), per lane in entry order, then in one fixed butterfly / warp order
    float s = 0.f;
#pragma unroll 4
    for (int e = b + t; e < end; e += NT) s += expf(out[e] - m);
    s = sum_warp(s);
    if (NT > 32) {
        if ((t & 31) == 0) sm_s[t >> 5] = s;
        __syncthreads();
        s = sm_s[0];
        for (int w = 1; w < NT / 32; ++w) s += sm_s[w];
    }
    for (int e = b + t; e < end; e += NT) out[e] = expf(out[e] - m) / s;
}

template <int NT>
__device__ __forceinline__ void softmax_backward_row(const AttnArgs& a, int i, int t)
{
    __shared__ float sm_x[kAttnWarps];
    const int b = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
    float c = 0.f;
    for (int e = b + t; e < end; e += NT) c = fmaf(__ldg(a.alpha + e), __ldg(a.dalpha + e), c);
    c = sum_warp(c);
    if (NT > 32) {
        if ((t & 31) == 0) sm_x[t >> 5] = c;
        __syncthreads();
        c = sm_x[0];
        for (int w = 1; w < NT / 32; ++w) c += sm_x[w];
        __syncthreads();                                    // sm_x is reused below
    }
    const float eli = __ldg(a.el + i);
    float d = 0.f;
    for (int e = b + t; e < end; e += NT) {
        const float x = attn_score(a, eli, e);
        const float g = __ldg(a.alpha + e) * (__ldg(a.dalpha + e) - c) * (x > 0.f ? 1.f : a.slope);
        a.out[e] = g;
        d += g;
    }
    d = sum_warp(d);
    if (NT > 32) {
        if ((t & 31) == 0) sm_x[t >> 5] = d;
        __syncthreads();
        d = sm_x[0];
        for (int w = 1; w < NT / 32; ++w) d += sm_x[w];
    }
    if (t == 0) a.d_el[i] = d;
}

__device__ __forceinline__ bool attn_short_row(const AttnArgs& a, int& i)
{
    i = (int)(blockIdx.x - (unsigned)a.nlong) * kAttnWarps + (int)(threadIdx.x >> 5);
    return i < a.m && __ldg(a.rowptr + i + 1) - __ldg(a.rowptr + i) <= kAttnLongRow;
}

__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_row<kAttnThreads>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_row<32>(a, i, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kAttnThreads)
edge_softmax_backward_kernel(const AttnArgs a)
{
    int i;
    if ((int)blockIdx.x < a.nlong) softmax_backward_row<kAttnThreads>(a, __ldg(a.long_rows + blockIdx.x), threadIdx.x);
    else if (attn_short_row(a, i)) softmax_backward_row<32>(a, i, threadIdx.x & 31);
}

}  // namespace pgcn
