// The lane layout, loads, dot products, dropout mask, online softmax and split-row fixups shared by the graph
// transformer attention (transformer.cu) and its edge-feature variant (transformer_edge.cu): one definition of each, so
// that both libraries reduce every head in the same order and give the same bits where their formulas agree.
//
// One warp per work item. The warp's lanes are split into K groups of G = 32 / K lanes, one group per head; lane g of
// head h holds the head's features 4 (g + G w) + u, u < 4, of pass w < 2, so a row of f <= 256 floats sits in 8
// registers per lane. A per-head dot product is each lane's sum over its slots in (w, u) order, then a butterfly over
// the group's lanes; all lanes of the group end with the same bits.
#pragma once

#include "philox.cuh"

#include <cuda_runtime.h>

#include <cstdint>

namespace pgcn {

constexpr int kTrThreads = 256;
constexpr int kTrWarps = kTrThreads / 32;
constexpr int kTrMaxF = 256;             // 2 passes x 32 lanes x 4 features

enum TrWalk : int { kTrForward = 0, kTrRows = 1, kTrCols = 2 };

struct TrArgs {
    const int4* items;
    const int32_t* splits;     // nsplits x 3
    const int32_t* idx;
    int nitems, nsplits, m, f, heads;
    const float* Q;            // m x f
    const float* KV;           // m x 2f
    const float* KVh;          // h x 2f
    float scale;
    const int32_t* gid;        // m + h
    const int64_t* drop;       // [key, c] or null
    uint32_t threshold;
    float keep_scale;
    const float* gZ;           // m x f (backward walks)
    const float* Z;            // m x f (row walk)
    const float* L;            // m x K (backward walks)
    float* out;                // Z (m x f), dQ (m x f) or [dK | dV] ((m + h) x 2f)
    float* aux;                // L (forward) or D (row walk), m x K; D is read by the column walk through `Dc`
    const float* Dc;           // m x K (column walk)
    float* work;               // nslots x (f + 2K), f or 2f
};

// This lane's place: head h, rank g in the head's group of G lanes, head width C, passes nw (1 when 4 G >= C).
struct Lanes {
    int h, g, G, C, nw;
};

__device__ __forceinline__ Lanes lanes(int lane, int f, int K)
{
    Lanes ln;
    ln.G = 32 / K;
    ln.h = lane / ln.G;
    ln.g = lane % ln.G;
    ln.C = f / K;
    ln.nw = 4 * ln.G < ln.C ? 2 : 1;
    return ln;
}

__device__ __forceinline__ const float* kv_row(const TrArgs& a, int j)
{
    return j < a.m ? a.KV + (size_t)j * 2 * a.f : a.KVh + (size_t)(j - a.m) * 2 * a.f;
}

// The lane's 8 slots of `row` (a row of f floats): VEC loads each pass's 4 consecutive features as one float4 (the host
// checked C % 4 == 0 and 16-byte alignment), the scalar instance loads the same features one by one. Unused slots 0.
template <bool VEC>
__device__ __forceinline__ void load8(const float* row, const Lanes& ln, float (&v)[8])
{
#pragma unroll
    for (int w = 0; w < 2; ++w) {
        const int cl = 4 * (ln.g + ln.G * w);
        const float* p = row + ln.h * ln.C + cl;
        if constexpr (VEC) {
            if (w < ln.nw && cl < ln.C) {
                const float4 u = __ldg(reinterpret_cast<const float4*>(p));
                v[4 * w] = u.x; v[4 * w + 1] = u.y; v[4 * w + 2] = u.z; v[4 * w + 3] = u.w;
            } else {
                v[4 * w] = v[4 * w + 1] = v[4 * w + 2] = v[4 * w + 3] = 0.0f;
            }
        } else {
#pragma unroll
            for (int u = 0; u < 4; ++u) v[4 * w + u] = w < ln.nw && cl + u < ln.C ? __ldg(p + u) : 0.0f;
        }
    }
}

// Plain (not read-only-path) loads: for work rows and for arrays the same launch writes elsewhere.
__device__ __forceinline__ void load8_plain(const float* row, const Lanes& ln, float (&v)[8])
{
#pragma unroll
    for (int w = 0; w < 2; ++w) {
        const int cl = 4 * (ln.g + ln.G * w);
#pragma unroll
        for (int u = 0; u < 4; ++u) v[4 * w + u] = w < ln.nw && cl + u < ln.C ? row[ln.h * ln.C + cl + u] : 0.0f;
    }
}

template <bool VEC>
__device__ __forceinline__ void store8(float* row, const Lanes& ln, const float (&v)[8])
{
#pragma unroll
    for (int w = 0; w < 2; ++w) {
        const int cl = 4 * (ln.g + ln.G * w);
        float* p = row + ln.h * ln.C + cl;
        if constexpr (VEC) {
            if (w < ln.nw && cl < ln.C)
                *reinterpret_cast<float4*>(p) = make_float4(v[4 * w], v[4 * w + 1], v[4 * w + 2], v[4 * w + 3]);
        } else {
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (w < ln.nw && cl + u < ln.C) p[u] = v[4 * w + u];
        }
    }
}

// < a, b > over this lane's head: the lane's slots in (w, u) order, then a butterfly over the head's G lanes. The
// unused slots hold 0 in both operands and add nothing.
__device__ __forceinline__ float head_dot(const float (&a)[8], const float (&b)[8], const Lanes& ln)
{
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s = __fmaf_rn(a[k], b[k], s);
    for (int o = 1; o < ln.G; o <<= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    return s;
}

struct Drop {
    bool on;
    uint32_t k0, k1, c, threshold;
    float keep_scale;
};

__device__ __forceinline__ Drop drop_state(const TrArgs& a)
{
    Drop d{a.drop != nullptr, 0u, 0u, 0u, a.threshold, a.keep_scale};
    if (d.on) {
        const uint64_t key = (uint64_t)__ldg(a.drop);
        d.k0 = (uint32_t)key;
        d.k1 = (uint32_t)(key >> 32);
        d.c = (uint32_t)__ldg(a.drop + 1);
    }
    return d;
}

// M of entry (gi, gj), head h: keep_scale when word h & 3 of Philox(gi, gj, c, h >> 2) >= threshold, else 0; 1 without
// dropout.
__device__ __forceinline__ float mask(const Drop& d, int gi, int gj, int h)
{
    if (!d.on) return 1.0f;
    uint32_t w[4];
    philox4x32_10((uint32_t)gi, (uint32_t)gj, d.c, (uint32_t)(h >> 2), d.k0, d.k1, w);
    const int q = h & 3;
    const uint32_t x = q == 0 ? w[0] : q == 1 ? w[1] : q == 2 ? w[2] : w[3];
    return x >= d.threshold ? d.keep_scale : 0.0f;
}

// Online-softmax state of one head on this lane.
struct Soft {
    float m, l;
};

// Take entry score s with aggregated row y, weighted p M: rescale when the max grows, then add.
__device__ __forceinline__ void soft_add(Soft& st, float (&acc)[8], float s, float mk, const float (&y)[8])
{
    if (s > st.m) {
        const float cr = expf(__fsub_rn(st.m, s));
        st.l = __fmul_rn(st.l, cr);
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] = __fmul_rn(acc[u], cr);
        st.m = s;
    }
    const float p = expf(__fsub_rn(s, st.m));
    st.l = __fadd_rn(st.l, p);
    const float pm = __fmul_rn(p, mk);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = __fmaf_rn(pm, y[u], acc[u]);
}

// Merge a chunk's (mc, lc, ac) into the state, in the same form.
__device__ __forceinline__ void soft_merge(Soft& st, float (&acc)[8], float mc, float lc, const float (&ac)[8])
{
    if (mc > st.m) {
        const float cr = expf(__fsub_rn(st.m, mc));
        st.l = __fmul_rn(st.l, cr);
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] = __fmul_rn(acc[u], cr);
        st.m = mc;
    }
    const float b = expf(__fsub_rn(mc, st.m));
    st.l = __fmaf_rn(lc, b, st.l);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = __fmaf_rn(ac[u], b, acc[u]);
}

// Z[r] = acc / l (0 for a row without entries, l == 0) and L[r, h] = m + log l.
template <bool VEC>
__device__ __forceinline__ void finish_forward(const TrArgs& a, int r, const Lanes& ln, const Soft& st,
                                               const float (&acc)[8])
{
    float z[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) z[u] = st.l == 0.0f ? 0.0f : __fdiv_rn(acc[u], st.l);
    store8<VEC>(a.out + (size_t)r * a.f, ln, z);
    if (ln.g == 0) a.aux[(size_t)r * a.heads + ln.h] = __fadd_rn(st.m, logf(st.l));
}

// dQ[r] = scale acc (row walk); [dK | dV][r] = [scale acc | acc2] (column walk).
template <int W, bool VEC>
__device__ __forceinline__ void finish_grad(const TrArgs& a, int r, const Lanes& ln, const float (&acc)[8],
                                            const float (&acc2)[8])
{
    float o[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) o[u] = __fmul_rn(acc[u], a.scale);
    if constexpr (W == kTrRows) {
        store8<VEC>(a.out + (size_t)r * a.f, ln, o);
    } else {
        store8<VEC>(a.out + (size_t)r * 2 * a.f, ln, o);
        store8<VEC>(a.out + (size_t)r * 2 * a.f + a.f, ln, acc2);
    }
}

// The bodies of the split-row kernels. Each library launches them through __global__ kernels of its own name.

// One warp per split row (row, slot0, count): the chunks' (acc, m, l) merged in chunk order, then the row finished.
__device__ __forceinline__ void forward_fixup(const TrArgs& a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f, K = a.heads, ow = f + 2 * K;
    const Lanes ln = lanes(lane, f, K);
    const float* w = a.work + (size_t)slot0 * ow;
    Soft st{w[f + ln.h], w[f + K + ln.h]};
    float acc[8];
    load8_plain(w, ln, acc);
    for (int q = 1; q < n; ++q) {
        w = a.work + (size_t)(slot0 + q) * ow;
        float ac[8];
        load8_plain(w, ln, ac);
        soft_merge(st, acc, w[f + ln.h], w[f + K + ln.h], ac);
    }
    finish_forward<false>(a, row, ln, st, acc);
}

// One warp per split row: the chunks' partial sums added in chunk order, then the row finished (row or column walk).
template <int W>
__device__ __forceinline__ void sum_fixup(const TrArgs& a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int row = __ldg(a.splits + 3 * sp), slot0 = __ldg(a.splits + 3 * sp + 1), n = __ldg(a.splits + 3 * sp + 2);
    const int f = a.f, ow = W == kTrCols ? 2 * f : f;
    const Lanes ln = lanes(lane, f, a.heads);
    float s[8] = {}, s2[8] = {};
    for (int q = 0; q < n; ++q) {
        const float* p = a.work + (size_t)(slot0 + q) * ow;
        float v[8];
        load8_plain(p, ln, v);
#pragma unroll
        for (int u = 0; u < 8; ++u) s[u] = __fadd_rn(s[u], v[u]);
        if constexpr (W == kTrCols) {
            load8_plain(p + f, ln, v);
#pragma unroll
            for (int u = 0; u < 8; ++u) s2[u] = __fadd_rn(s2[u], v[u]);
        }
    }
    finish_grad<W, false>(a, row, ln, s, s2);
}

// D[r, h] = < gZ[r, h], Z[r, h] > of the split rows, before the row walk's chunks read it: once per row.
__device__ __forceinline__ void delta(const TrArgs& a)
{
    const int lane = threadIdx.x & 31;
    const int sp = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
    if (sp >= a.nsplits) return;
    const int r = __ldg(a.splits + 3 * sp);
    const Lanes ln = lanes(lane, a.f, a.heads);
    float g[8], z[8];
    load8<false>(a.gZ + (size_t)r * a.f, ln, g);
    load8<false>(a.Z + (size_t)r * a.f, ln, z);
    const float D = head_dot(g, z, ln);
    if (ln.g == 0) a.aux[(size_t)r * a.heads + ln.h] = D;
}

}  // namespace pgcn
