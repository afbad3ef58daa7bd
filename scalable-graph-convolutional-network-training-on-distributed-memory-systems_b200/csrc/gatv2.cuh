// gatv2.cuh — sm_90a kernels of GATv2 attention (Brody et al., PyG / DGL GATv2Conv) over the stored pattern.
//
// With xl (source side, one row per column: owned rows, then the halo rows), xr (destination side, one row per owned
// row), att [K, d] (d = f / K; flat, att[h, c] is feature h d + c) and t_e = xl[col(e)] + xr[row(e)]:
//     s_eh     = sum_c att[h d + c] * LeakyReLU(t_e[h d + c])                       the score kernels
//     alpha    = the edge softmax of s per row and head                             edge_softmax_raw_kernel
//     Z        = A(alpha) xl, head h on its slice                                   spmm_heads_kernel
// and, with dscore (edge_softmax_raw_backward_kernel over dalpha = sddmm_heads(gZ, xl)) and
// g_ec = dscore_e,h(c) * att_c * LeakyReLU'(t_ec):
//     dxr[i]    = sum_{e in row i} g_e                                              gatv2_row_backward_kernel
//     datt[c]   = sum_e dscore_e,h(c) * LeakyReLU(t_ec)                             per-chunk partials + gatv2_datt_kernel
//     dxl[j]    = sum_{e in col j} alpha_e,h(c) gZ[row(e), c] + g_ec                gatv2_col_backward_kernel
//
//   gatv2_score_ring_kernel<NV, K>  f = 128 NV (NV = 1, 2), 16-byte aligned operands: sddmm_heads_ring_walk with xr's
//                                   row in registers where the SDDMM holds gZ and att_c * LeakyReLU(xl_c + xr_c) as the
//                                   per-element term
//   gatv2_score_plain_kernel        any f and alignment, the same bits: lanes and reduction tree of the ring (below)
//
// The summation order of a score. Head h's d features are dealt to L = min(32, 2^floor(log2(max(1, d / 4)))) lanes,
// feature o (0 <= o < d) to lane (o / 4) % L; a lane sums its features in increasing o with fmaf, starting from 0, and
// the L lane sums are added by an xor butterfly over lane masks L/2, L/4, .., 1. For f = 128 and 256 this is exactly
// what the ring kernel's lanes, chains and transposing butterfly compute (fp32 addition commutes, so only the pairing
// of the tree matters), so both instances give the same bits.
#pragma once
#include "sddmm.cuh"

namespace pgcn {

// ---- scores ---------------------------------------------------------------------------------------------------------

__device__ __forceinline__ float leaky(float t, float slope) { return t > 0.f ? t : t * slope; }

// att_c * LeakyReLU(xl_c + xr_c): g = xr (the register row), r = xl (the gathered row), att = this lane's slices of att
template <int NV>
struct Gatv2Score {
    float4 att[NV];
    float slope;
    __device__ __forceinline__ void operator()(float& s, const float4& g, const float4& r, int v) const
    {
        s = fmaf(att[v].x, leaky(r.x + g.x, slope), s); s = fmaf(att[v].y, leaky(r.y + g.y, slope), s);
        s = fmaf(att[v].z, leaky(r.z + g.z, slope), s); s = fmaf(att[v].w, leaky(r.w + g.w, slope), s);
    }
};

// The halo rows of a forward: the exchange's slab, or its odd-epoch twin on the peer transport.
struct Gatv2Halo {
    const float* odd;                       // null: a.H1 is the only slab
    const unsigned long long* epoch;
};

// a: SddmmArgs with gZ = xr, H0 = xl_own, H1 = the halo slab, dvals = the scores (nnz x K)
template <int NV, int K>
__global__ void __maxnreg__(232)         // launched with kSddmmWarps * 32 threads, as sddmm_heads_ring_kernel
gatv2_score_ring_kernel(SddmmArgs a, const Gatv2Halo hl, const float* __restrict__ att, float slope)
{
    if (hl.odd && epoch_odd(hl.epoch)) a.H1 = hl.odd;
    Gatv2Score<NV> c;
    const float4* ap = reinterpret_cast<const float4*>(att) + (threadIdx.x & 31);
#pragma unroll
    for (int v = 0; v < NV; ++v) c.att[v] = __ldg(ap + v * 32);
    c.slope = slope;
    sddmm_heads_ring_walk<NV, K>(a, c);
}

// One warp per row block, one edge at a time: in each round the warp's lanes take (head, lane of the head) pairs, each
// lane sums its features, and the butterfly over the head's lanes finishes the score.
__global__ void __launch_bounds__(256)
gatv2_score_plain_kernel(SddmmArgs a, const Gatv2Halo hl, const float* __restrict__ att, float slope, int K)
{
    const int lane = threadIdx.x & 31;
    const int w = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    if (w >= a.nblocks) return;
    if (hl.odd && epoch_odd(hl.epoch)) a.H1 = hl.odd;
    const int4 b = __ldg(a.blocks + w);
    const bool seg = b.y < 0;
    const int d = a.f / K;
    int L = 1;
    while (L < 32 && 8 * L <= d) L *= 2;                     // min(32, 2^floor(log2(d / 4))), 1 when d < 8
    const int hpr = 32 / L;                                  // heads per round
    const int li = lane % L;
    int row = b.x;
    for (int e = b.z; e < b.w; ++e) {
        const int* pc = a.pieces + (size_t)(e >> 5) * kPieceInts;
        const int col = __ldg(pc + (e & 31));
        const bool end = !seg && ((__ldg(reinterpret_cast<const unsigned*>(pc + 64)) >> (e & 31)) & 1u);
        const int orow = a.rowids ? __ldg(a.rowids + row) : row;
        const float* xr = a.gZ + (size_t)(unsigned)orow * a.f;
        const float* xl = (a.H1 && col >= a.split) ? a.H1 + (size_t)(col - a.split) * a.f : a.H0 + (size_t)col * a.f;
        for (int h0 = 0; h0 < K; h0 += hpr) {
            const int h = h0 + lane / L;
            float s = 0.f;
            if (h < K) {
                for (int o0 = 4 * li; o0 < d; o0 += 4 * L)
                    for (int o = o0; o < o0 + 4 && o < d; ++o) {
                        const int c = h * d + o;
                        s = fmaf(__ldg(att + c), leaky(__ldg(xl + c) + __ldg(xr + c), slope), s);
                    }
            }
            for (int m = L >> 1; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
            if (h < K && li == 0) a.dvals[(size_t)e * K + h] = s;
        }
        if (end) ++row;
    }
}

// ---- backward -------------------------------------------------------------------------------------------------------

struct Gatv2BwdArgs {
    const float* alpha;      // nnz x NH, forward CSR order
    const float* dscore;     // nnz x NH
    const float* att;        // f
    float slope;
    int hd;                  // f / NH
    const int* amap;         // launched entry -> forward entry (null: the forward records)
    const float* xv;         // row kernel: xr (m x f, by output row); column kernel: xl_own (m x f)
    const float* xv_halo;    // column kernel: xl_halo (h x f, rows m ..)
    float* datt_part;        // row kernel: f floats per chunk of kGatv2Chunk row blocks
};

constexpr int kGatv2Chunk = 8;          // row blocks per datt partial: every CTA holds whole chunks (8 .. 64 lane groups)

// The staged per-entry head values of a chunk (alpha, dscore): two chunks of NH floats per thread each.
template <int NH>
__device__ __forceinline__ float* gatv2_head_smem()
{
    __shared__ float s_hv[2 * 2 * kSpmmThreads * NH];
    return s_hv;
}

// vector helpers of the backward: per float, the same operations at VW = 4 and 1
__device__ __forceinline__ void g2_add(float4& r, const float4& a, const float4& b) { r = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ void g2_add(float& r, const float& a, const float& b) { r = a + b; }
// acc += ds * att * LeakyReLU'(t)
__device__ __forceinline__ void g2_score_grad(float& acc, float ds, float at, float t, float slope)
{
    acc = fmaf(ds, t > 0.f ? at : at * slope, acc);
}
__device__ __forceinline__ void g2_score_grad(float4& acc, float ds, const float4& at, const float4& t, float slope)
{
    g2_score_grad(acc.x, ds, at.x, t.x, slope); g2_score_grad(acc.y, ds, at.y, t.y, slope);
    g2_score_grad(acc.z, ds, at.z, t.z, slope); g2_score_grad(acc.w, ds, at.w, t.w, slope);
}
// datt += ds * LeakyReLU(t)
__device__ __forceinline__ void g2_att_grad(float& acc, float ds, float t, float slope) { acc = fmaf(ds, leaky(t, slope), acc); }
__device__ __forceinline__ void g2_att_grad(float4& acc, float ds, const float4& t, float slope)
{
    g2_att_grad(acc.x, ds, t.x, slope); g2_att_grad(acc.y, ds, t.y, slope);
    g2_att_grad(acc.z, ds, t.z, slope); g2_att_grad(acc.w, ds, t.w, slope);
}

// The register walk both backward kernels share: spmm_heads_kernel's lane groups, blocks, segments, chunks of LPE
// entries staged in shared memory with their NH alpha / dscore values, two gathers in flight and flushes at row ends.
// COL = false (the row kernel, forward records): gathers xl[col]; the row's xr is resident; accumulates dxr and datt.
// COL = true (the column kernel, transposed records through amap): gathers gZ[i] and xr[i]; the row's xl is resident;
// accumulates dxl. Rows [0, zsplit) go to Z0, the rest to Z1; split rows write partials that spmm_fixup_kernel sums.
template <int LPE, int VW, bool HALO, int NH, bool COL>
__device__ __forceinline__ void gatv2_backward_walk(const SpmmArgs& a, const Gatv2BwdArgs& g)
{
    typedef typename Vec<VW>::type vec_t;
    __shared__ int2 s_cw[2][kSpmmThreads];
    __shared__ vec_t s_datt[kSpmmThreads];

    const int lane_w = threadIdx.x & 31;
    const int gl = threadIdx.x & (LPE - 1);
    const int gbase = threadIdx.x & ~(LPE - 1);
    const unsigned gmask = (LPE == 32) ? 0xffffffffu
                                       : (((1u << (LPE & 31)) - 1u) << (lane_w & ~(LPE - 1)));
    const int group = (int)((blockIdx.x * (unsigned)kSpmmThreads + threadIdx.x) / LPE);
    const unsigned pitch = (unsigned)a.f * 4u;
    const int f0 = blockIdx.y * (LPE * VW) + gl * VW;
    const bool fok = f0 < a.f;                                        // f % VW == 0 (launcher)
    vec_t datt = vzero((vec_t*)nullptr);

    if (group < a.nblocks) {                                          // whole lane groups are in or out
        const int4 b = a.blocks[group];
        const bool seg = b.y < 0;
        const int lastmask = seg ? 0 : kLastFlag;
        const int e_end = b.w;
        int e = b.z;
        int row = b.x;

        const char* hb0 = reinterpret_cast<const char*>(a.H0) + (size_t)f0 * 4;     // row: xl_own; column: gZ
        const char* hb1 = HALO ? reinterpret_cast<const char*>(a.H1) + (size_t)f0 * 4 - (size_t)a.split * pitch : hb0;
        const char* rb = reinterpret_cast<const char*>(a.H1) + (size_t)f0 * 4;      // column kernel: xr (H1)
        const int hv = fok ? f0 / g.hd : 0;
        const vec_t at = fok ? *reinterpret_cast<const vec_t*>(g.att + f0) : vzero((vec_t*)nullptr);
        float* s_hv = gatv2_head_smem<NH>();
        auto sidx = [&](int k, int bf, int t) { return ((size_t)(k * 2 + bf) * kSpmmThreads + t) * NH; };
        float al_next[NH], ds_next[NH];
        auto ld_hv = [&](float (&al)[NH], float (&ds)[NH], int ee) {
            const bool ok = ee < e_end;
            const int me = !ok ? 0 : (g.amap ? __ldg(g.amap + ee) : ee);
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                al[h] = (COL && ok) ? __ldg(g.alpha + (size_t)me * NH + h) : 0.f;
                ds[h] = ok ? __ldg(g.dscore + (size_t)me * NH + h) : 0.f;
            }
        };
        auto st_hv = [&](int bf, const float (&al)[NH], const float (&ds)[NH]) {
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                if (COL) s_hv[sidx(0, bf, threadIdx.x) + h] = al[h];
                s_hv[sidx(1, bf, threadIdx.x) + h] = ds[h];
            }
        };

        const unsigned long long pol_hot = l2_policy_evict_last();
        const unsigned long long pol_cold = l2_policy_evict_first();

        // the resident row: row kernel xr[orow], column kernel xl[orow] (own or halo)
        vec_t xres = vzero((vec_t*)nullptr);
        auto load_res = [&]() {
            if (!fok) return;
            const int orow = (a.rowids != nullptr) ? __ldg(a.rowids + row) : row;
            const float* base = COL ? (orow < a.zsplit ? g.xv + (size_t)(unsigned)orow * a.f
                                                       : g.xv_halo + (size_t)(unsigned)(orow - a.zsplit) * a.f)
                                    : g.xv + (size_t)(unsigned)orow * a.f;
            xres = ld_feat(reinterpret_cast<const vec_t*>(base + f0));
        };
        vec_t acc = vzero((vec_t*)nullptr);
        auto flush_row = [&]() {
            const int orow = (a.rowids != nullptr) ? __ldg(a.rowids + row) : row;
            char* zb = (orow < a.zsplit)
                           ? reinterpret_cast<char*>(a.Z0) + (size_t)(unsigned)orow * pitch
                           : reinterpret_cast<char*>(a.Z1) + (size_t)(unsigned)(orow - a.zsplit) * pitch;
            if (fok) st_out(reinterpret_cast<vec_t*>(zb + (size_t)f0 * 4), acc);
            acc = vzero((vec_t*)nullptr);
            ++row;
        };
        // row kernel: r0 = xl[col]; column kernel: r0 = gZ[i], r1 = xr[i]
        auto gather = [&](vec_t& r0, vec_t& r1, int craw) {
            const unsigned cj = (unsigned)(craw & kColMask);
            const unsigned long long pol = (craw & kColdFlag) ? pol_cold : pol_hot;
            if (!fok) return;
            const char* hb = (HALO && cj >= (unsigned)a.split) ? hb1 : hb0;
            r0 = ld_feat_hint(reinterpret_cast<const vec_t*>(hb + (size_t)cj * pitch), pol);
            if (COL) r1 = ld_feat_hint(reinterpret_cast<const vec_t*>(rb + (size_t)cj * pitch), pol);
        };
        auto consume = [&](const vec_t& r0, const vec_t& r1, int2 cw, int j, int bf) {
            if (fok) {
                const float ds = s_hv[sidx(1, bf, gbase + j) + hv];
                vec_t t;
                if (COL) {
                    g2_add(t, xres, r1);                                  // xl[j] + xr[i]
                    vfma(acc, s_hv[sidx(0, bf, gbase + j) + hv], r0);     // alpha gZ[i]
                } else {
                    g2_add(t, r0, xres);                                  // xl[j] + xr[i]
                    g2_att_grad(datt, ds, t, g.slope);
                }
                g2_score_grad(acc, ds, at, t, g.slope);
            }
            if (cw.x & lastmask) {
                flush_row();
                if (e + j + 1 < e_end) load_res();
            }
        };

        load_res();
        int buf = 0;
        {
            int2 cw = make_int2(0, 0);
            if (e + gl < e_end) cw = ld_entry(a.pieces, e + gl);
            s_cw[0][threadIdx.x] = cw;
            float al[NH], ds[NH];
            ld_hv(al, ds, e + gl);
            st_hv(0, al, ds);
        }
        int2 cw_next = make_int2(0, 0);
        if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
        ld_hv(al_next, ds_next, e + LPE + gl);
        __syncwarp(gmask);

        while (e < e_end) {
            const int n = min(LPE, e_end - e);
            const int2* cwp = &s_cw[buf][gbase];
            vec_t rA0, rA1, rB0, rB1;
            int2 cwA = cwp[0], cwB;
            gather(rA0, rA1, cwA.x);
#pragma unroll 1
            for (int j = 0; j < n; j += 2) {
                const bool hasB = j + 1 < n;
                if (hasB) { cwB = cwp[j + 1]; gather(rB0, rB1, cwB.x); }
                consume(rA0, rA1, cwA, j, buf);
                if (j + 2 < n) { cwA = cwp[j + 2]; gather(rA0, rA1, cwA.x); }
                if (hasB) consume(rB0, rB1, cwB, j + 1, buf);
            }
            e += n;
            buf ^= 1;
            s_cw[buf][threadIdx.x] = cw_next;
            cw_next = make_int2(0, 0);
            if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
            st_hv(buf, al_next, ds_next);
            ld_hv(al_next, ds_next, e + LPE + gl);
            __syncwarp(gmask);
        }

        if (seg && fok) {
            char* pb = reinterpret_cast<char*>(a.partial) + (size_t)(unsigned)(-b.y - 1) * pitch + (size_t)f0 * 4;
            *reinterpret_cast<vec_t*>(pb) = acc;
        }
    }

    if (!COL) {
        // datt: the lane groups of each chunk of kGatv2Chunk consecutive row blocks, added in group order. The chunks do
        // not depend on LPE or VW, so neither does any bit of datt.
        s_datt[threadIdx.x] = datt;
        __syncthreads();
        const int gi = threadIdx.x / LPE;                                   // lane group within the CTA
        if (gi % kGatv2Chunk == 0 && group < a.nblocks && fok) {
            vec_t s = s_datt[threadIdx.x];
#pragma unroll 1
            for (int k = 1; k < kGatv2Chunk; ++k) vadd(s, s_datt[threadIdx.x + k * LPE]);
            *reinterpret_cast<vec_t*>(g.datt_part + (size_t)(group / kGatv2Chunk) * a.f + f0) = s;
        }
    }
}

// dxr and the datt partials: the forward records of the register schedule. H0 = xl_own, H1 = xl_halo (HALO),
// Z0 = dxr, g.xv = xr. 3 CTAs of 256 threads per SM: with the next chunk's staged values and the resident row in
// registers, the 4-CTA budget of spmm_heads_kernel spills.
template <int LPE, int VW, bool HALO, int NH>
__global__ void __launch_bounds__(kSpmmThreads, 3)
gatv2_row_backward_kernel(const SpmmArgs a, const Gatv2BwdArgs g)
{
    gatv2_backward_walk<LPE, VW, HALO, NH, false>(a, g);
}

// dxl: the transposed records of the register schedule. H0 = gZ, H1 = xr (both m x f, at the record's column),
// Z0 = dxl (rows < m), Z1 = the reverse send slab (halo rows), g.xv / g.xv_halo = xl_own / xl_halo.
template <int LPE, int VW, int NH>
__global__ void __launch_bounds__(kSpmmThreads, NH == 8 ? 2 : 3)     // NH = 8: 16 staged values in flight, no spills
gatv2_col_backward_kernel(const SpmmArgs a, const Gatv2BwdArgs g)
{
    gatv2_backward_walk<LPE, VW, false, NH, true>(a, g);
}

// datt[c] = sum of the chunk partials in chunk order: one CTA per 32 features, kGatv2RedWarps warps each take every
// kGatv2RedWarps-th chunk, then warp 0 adds the warps' sums in warp order.
constexpr int kGatv2RedWarps = 32;

__global__ void __launch_bounds__(32 * kGatv2RedWarps)
gatv2_datt_kernel(const float* __restrict__ part, int nchunks, int f, float* __restrict__ datt)
{
    __shared__ float s[kGatv2RedWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    float acc = 0.f;
    if (c < f) {
        int i = w;
        for (; i + 3 * kGatv2RedWarps < nchunks; i += 4 * kGatv2RedWarps) {
            const float x0 = __ldcs(part + (size_t)i * f + c);
            const float x1 = __ldcs(part + (size_t)(i + kGatv2RedWarps) * f + c);
            const float x2 = __ldcs(part + (size_t)(i + 2 * kGatv2RedWarps) * f + c);
            const float x3 = __ldcs(part + (size_t)(i + 3 * kGatv2RedWarps) * f + c);
            acc += x0; acc += x1; acc += x2; acc += x3;
        }
        for (; i < nchunks; i += kGatv2RedWarps) acc += __ldcs(part + (size_t)i * f + c);
    }
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0 && c < f) {
        float t = s[0][lane];
#pragma unroll
        for (int k = 1; k < kGatv2RedWarps; ++k) t += s[k][lane];
        datt[c] = t;
    }
}

}  // namespace pgcn
