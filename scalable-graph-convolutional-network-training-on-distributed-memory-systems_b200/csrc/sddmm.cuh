// sddmm.cuh — sm_90a kernels of the differentiable edge values of the aggregation.
//
// With Z = A H and the values of A set per call (pgcn_plan_set_values), the gradient of the values is the sampled
// dense-dense product
//     dvals[e] = < gZ[row(e), :], [H_own ; H_halo][col(e), :] >        for every stored entry e of A,
// what torch.sparse.mm(A, H) returns as dA.values when A's values require grad (GPU/PGCN.py:127 with a learned A).
//
//   set_values_kernel   rewrites the value words of every record set of a plan (forward, transposed, own-column and
//                       per-peer blocks) from one array in forward CSR order, through the maps pgcn_plan_bind_values
//                       built: a gather, so the record writes coalesce (32 consecutive value words per piece)
//   sddmm_ring_kernel   the SDDMM for f = 128 .. 512 (multiples of 128) with 16-byte aligned operands: it gathers the
//                       same rows of H as the forward SpMM, so it is built like spmm_ring_kernel — per-warp rings of
//                       row slots filled by 1-D TMA bulk copies with mbarrier completion, row blocks of the forward
//                       schedule, persistent CTAs — but it writes 4 bytes per edge instead of a row per row
//   sddmm_plain_kernel  every other width or alignment: one lane per edge, a sequential dot product
//   sddmm_heads_ring_kernel / sddmm_plain_heads_kernel   the same with K heads: one dot product per (edge, head)
//   copy_halo_kernel    the halo rows a forward received, copied out of the slab of the call's exchange parity
#pragma once
#include "spmm_ring.cuh"

namespace pgcn {

// ---- value rewrite -------------------------------------------------------------------------------------------------

// One record set of a plan: entry e of `cw` takes vals[map[e]] (map == nullptr: vals[e], the forward matrix itself).
// `start` = entries of all earlier sets (the sets are walked as one concatenated index space).
struct ValueSet {
    int* cw;
    const int* map;
    long long nnz;
    long long start;
};

__global__ void __launch_bounds__(256)
set_values_kernel(const ValueSet* sets, int nsets, long long total, const float* vals)
{
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = nsets - 1;                       // last set whose start <= t
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (__ldg(&sets[mid].start) <= t) lo = mid; else hi = mid - 1;
        }
        const ValueSet& s = sets[lo];
        const long long e = t - s.start;
        const long long src = s.map ? (long long)__ldg(s.map + e) : e;
        s.cw[(size_t)(e >> 5) * kPieceInts + 32 + (e & 31)] = __float_as_int(__ldg(vals + src));
    }
}

// ---- halo rows of the last forward ------------------------------------------------------------------------------

// dst[0 .. n) = the halo slab of the call: src_odd while the exchange epoch is odd (peer transport), else src.
__global__ void __launch_bounds__(256)
copy_halo_kernel(const float* src, const float* src_odd, const unsigned long long* epoch, float* dst, long long n)
{
    const float* s = epoch_odd(epoch) ? src_odd : src;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        dst[t] = s[t];
}

// ---- SDDMM ----------------------------------------------------------------------------------------------------------

struct SddmmArgs {
    const int4* blocks;      // the forward matrix's row blocks {first row, nrows | -(slot+1), e_begin, e_end}
    int nblocks;
    const int* pieces;       // the forward matrix's records (forward CSR order: entry e is dvals[e])
    const float* gZ;         // m x f, indexed by output row
    const float* H0;         // columns [0, split)
    const float* H1;         // columns [split, ...) (the halo rows), may be null when no entry references them
    int split;
    const int* rowids;       // compact row -> output row, null when the identity
    float* dvals;
    int f;
    unsigned int* counter;   // work-item counter of the persistent ring kernel (zeroed before the launch)
};

constexpr int kSddmmG = 8;          // edges per completion group = edges per transposing reduction
constexpr int kSddmmNG = 2;         // groups in the ring: 16 row slots per warp, one group in flight while one is consumed
constexpr int kSddmmWarps = 4;

__host__ __device__ constexpr size_t sddmm_warp_bytes(int nv)
{
    return ((size_t)kSddmmG * kSddmmNG * nv * 512 + (size_t)kSddmmNG * 8 + 127) / 128 * 128;
}
__host__ __device__ constexpr size_t sddmm_smem_bytes(int nv) { return sddmm_warp_bytes(nv) * kSddmmWarps + 128; }

// ---- multi-head SDDMM ----------------------------------------------------------------------------------------------
//
//     dalpha[e, h] = < gZ[row(e), h d:(h+1) d], [H_own ; H_halo][col(e), h d:(h+1) d] >        d = f / K
//
// sddmm_heads_ring_kernel<NV, K> is sddmm_ring_kernel with K heads (f = 128 NV, NV = 1, 2 or 4, K = 2, 4 or 8): the
// same row blocks, slots, bulk copies and gZ rows in registers. What changes is the partial sums and their reduction.
// Lane l holds the float4 of features 128 v + 4 l (v < NV). When d >= 128 a head spans whole 128-float slices, so a lane
// keeps K chains per edge (slices summed in order) and all 32 lanes reduce them; when d < 128 every slice holds
// 128 / d heads of 32 / (128 / d) consecutive lanes each, so a lane keeps NV chains per edge (one per slice) and only
// the lanes of one head reduce them. Either way the 8 U values of a lane (U chains x 8 edges) go through a transposing
// butterfly over the lanes of the head that stops as soon as every (edge, head) sum is complete, and a lane stores the
// values it holds. Every output is added in one fixed order.
template <int NV, int K>
struct SddmmHeadShape {
    static constexpr int HPV = K > NV ? K / NV : 1;    // heads in one 128-float slice
    static constexpr int U = K > NV ? NV : K;          // chains per edge and lane
    static constexpr int VPC = K > NV ? 1 : NV / K;    // slices per chain
    static constexpr int L = 32 / HPV;                 // lanes that share a head
    static constexpr int N = 8 * U;                    // values per lane before the reduction
};

__host__ __device__ constexpr int ilog2(int x) { return x <= 1 ? 0 : 1 + ilog2(x >> 1); }

// head of chain u of lane `lane`
template <int NV, int K>
__device__ __forceinline__ int sddmm_chain_head(int u, int lane)
{
    typedef SddmmHeadShape<NV, K> S;
    return K > NV ? u * S::HPV + lane / S::L : u;
}

// p[n], n = u * 8 + j (chain u, edge j): transposing butterfly over the L lanes of a head. After step t (lane mask
// L >> (t + 1)) a lane keeps the half of its values whose bit LN - 1 - t equals its lane bit; after S = min(LN, LB)
// steps it holds the R = N >> S values n = (its lane bits LB-1 .. LB-S) << (LN - S) | r, r < R, summed over 2^S lanes;
// plain xor steps over the remaining lane bits finish the sums. Returns the R sums in q[0 .. R).
template <int N, int L>
__device__ __forceinline__ void sddmm_reduce_heads(float (&p)[N], int lane)
{
    constexpr int LN = ilog2(N), LB = ilog2(L), S = LN < LB ? LN : LB;
#pragma unroll
    for (int t = 0; t < S; ++t) {
        const int half = N >> (t + 1);
        const bool up = lane & (L >> (t + 1));
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            if (i < half) {
                const float keep = up ? p[i + half] : p[i], send = up ? p[i] : p[i + half];
                p[i] = keep + __shfl_xor_sync(0xffffffffu, send, L >> (t + 1));
            }
        }
    }
#pragma unroll
    for (int t = S; t < LB; ++t) p[0] += __shfl_xor_sync(0xffffffffu, p[0], L >> (t + 1));
}

// The per-element term of the multi-head SDDMM: s += gZ_c * H_c (g: the row held in registers, r: the gathered row).
struct SddmmDot {
    __device__ __forceinline__ void operator()(float& s, const float4& g, const float4& r, int) const
    {
        s = fmaf(g.x, r.x, s); s = fmaf(g.y, r.y, s);
        s = fmaf(g.z, r.z, s); s = fmaf(g.w, r.w, s);
    }
};

// The ring walk of sddmm_heads_ring_kernel with the per-element term C (called with the chain sum, the register row's
// float4 v, the gathered row's float4 v and v): the SDDMM's dot product, or GATv2's score (gatv2.cuh).
template <int NV, int K, class C>
__device__ __forceinline__ void sddmm_heads_ring_walk(const SddmmArgs& a, const C& comb)
{
    typedef SddmmHeadShape<NV, K> S;
    constexpr int G = kSddmmG, NG = kSddmmNG, NS = G * NG;
    constexpr uint32_t RB = NV * 512;
    constexpr int RV = RB / 16;
    constexpr int LN = ilog2(S::N), LB = ilog2(S::L), SS = LN < LB ? LN : LB, R = S::N >> SS;
    extern __shared__ __align__(128) unsigned char sddmm_smem[];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* wbase = sddmm_smem + (size_t)warp * sddmm_warp_bytes(NV);
    const uint32_t s_data = smem_u32(wbase);
    const uint32_t s_bar = s_data + NS * RB;
    const float4* data_gen = reinterpret_cast<const float4*>(wbase) + lane;

    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < NG; ++i) mbar_init(s_bar + i * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncwarp();

    const unsigned long long pol_hot = l2_policy_evict_last();
    const unsigned long long pol_cold = l2_policy_evict_first();
    const size_t pitch = (size_t)a.f * 4;
    const unsigned usplit = a.H1 ? (unsigned)a.split : 0xffffffffu;
    const char* hb0 = reinterpret_cast<const char*>(a.H0);
    const char* hb1 = a.H1 ? reinterpret_cast<const char*>(a.H1) - (size_t)a.split * pitch : hb0;
    uint32_t gpar = 0;
    // the values this lane stores: n0 + r, r < R, when it is the first of the lanes that hold them
    const int n0 = ((lane % S::L) >> (LB - SS)) << (LN - SS);
    const bool storer = (lane & ((1 << (LB - SS)) - 1)) == 0;

    auto load_g = [&](float4 (&g)[NV], int row) {
        const int orow = a.rowids ? __ldg(a.rowids + row) : row;
        const float4* gp = reinterpret_cast<const float4*>(a.gZ + (size_t)(unsigned)orow * a.f) + lane;
#pragma unroll
        for (int v = 0; v < NV; ++v) g[v] = __ldg(gp + v * 32);
    };

    int w;
    if (lane == 0) w = (int)atomicAdd(a.counter, 1u);
    w = __shfl_sync(0xffffffffu, w, 0);
    while (w < a.nblocks) {
        const int4 b = __ldg(a.blocks + w);
        const bool seg = b.y < 0;
        const int e0 = b.z, e1 = b.w;
        int row = b.x;
        const int row_last = seg ? b.x : b.x + b.y - 1;
        const int gA = e0 / G, gB = (e1 - 1) / G;

        float4 gcur[NV], gnext[NV];
        load_g(gcur, row);
        if (row < row_last) load_g(gnext, row + 1);

        auto fetch = [&](int gi, int& col, uint32_t& bits) {
            col = 0; bits = 0;
            const int e = gi * G + lane;
            if (lane < G && gi <= gB && e >= e0 && e < e1) {
                const int* pc = a.pieces + (size_t)(e >> 5) * kPieceInts;
                col = __ldg(pc + (e & 31));
                const uint2 m = __ldg(reinterpret_cast<const uint2*>(pc + 64));
                bits = 1u | (((m.x >> (e & 31)) & 1u) << 1) | (((m.y >> (e & 31)) & 1u) << 2);
            }
        };
        uint32_t vmask[NG], emask[NG];
        auto issue = [&](int sg, int col, uint32_t bits) {
            const uint32_t vm = __ballot_sync(0xffffffffu, bits & 1u) & 0xffu;
            const uint32_t em = __ballot_sync(0xffffffffu, (bits >> 1) & 1u) & 0xffu;
            reg_set(vmask, sg, vm);
            reg_set(emask, sg, seg ? 0u : em);
            if (vm == 0) return;
            if (lane == 0) mbar_expect_tx(s_bar + sg * 8, (uint32_t)__popc(vm) * RB);
            if (bits & 1u) {
                const unsigned cj = (unsigned)col;
                bulk_g2s(s_data + (sg * G + lane) * RB, (cj >= usplit ? hb1 : hb0) + (size_t)cj * pitch, RB, s_bar + sg * 8,
                         (bits & 4u) ? pol_cold : pol_hot);
            }
        };

        int ncol;
        uint32_t nbits;
#pragma unroll
        for (int i = 0; i < NG; ++i) { fetch(gA + i, ncol, nbits); issue(i, ncol, nbits); }
        fetch(gA + NG, ncol, nbits);

#pragma unroll 1
        for (int gi = gA; gi <= gB; ++gi) {
            const int sg = (gi - gA) % NG;
            const uint32_t vm = reg_get(vmask, sg), em = reg_get(emask, sg);
            mbar_wait(s_bar + sg * 8, (gpar >> sg) & 1);
            gpar ^= 1u << sg;
            const float4* slot = data_gen + (size_t)(sg * G) * RV;
            float p[S::N];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float s[S::U];
#pragma unroll
                for (int u = 0; u < S::U; ++u) s[u] = 0.f;
#pragma unroll
                for (int v = 0; v < NV; ++v) {
                    const int u = v / S::VPC;
                    const float4 r = slot[j * RV + v * 32];
                    comb(s[u], gcur[v], r, v);
                }
#pragma unroll
                for (int u = 0; u < S::U; ++u) p[u * 8 + j] = (vm >> j & 1u) ? s[u] : 0.f;
                if (em >> j & 1u) {
                    ++row;
#pragma unroll
                    for (int v = 0; v < NV; ++v) gcur[v] = gnext[v];
                    if (row < row_last) load_g(gnext, row + 1);
                }
            }
            sddmm_reduce_heads<S::N, S::L>(p, lane);
            if (storer) {
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int n = n0 + r, j = n & 7, u = n >> 3;
                    if (vm >> j & 1u) a.dvals[((size_t)gi * G + j) * K + sddmm_chain_head<NV, K>(u, lane)] = p[r];
                }
            }
            __syncwarp();
            issue(sg, ncol, nbits);
            fetch(gi + NG + 1, ncol, nbits);
        }

        if (lane == 0) w = (int)atomicAdd(a.counter, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
    }
}

template <int NV, int K>
__global__ void __maxnreg__(232)         // launched with kSddmmWarps * 32 threads; without a limit ptxas caps some at 128 and spills
sddmm_heads_ring_kernel(const SddmmArgs a)
{
    sddmm_heads_ring_walk<NV, K>(a, SddmmDot());
}

// NV = f / 128: what one lane holds of a row (NV float4, 512 bytes apart).
// A warp walks one row block of the forward schedule at a time (persistent CTAs take blocks from a counter) in
// globally aligned groups of 8 entries. Per group: lanes 0..7 read their entry's column and row-end / cold bits (one
// group ahead) and fire one bulk copy of the whole H row each into the group's 8 slots; lane 0 arms the group's
// mbarrier. Consumption: per edge, NV x LDS.128 and 4 NV FFMA against the warp's current gZ row, held in registers
// (the next row's gZ is loaded one row ahead); the 8 partials go through the transposing butterfly (sddmm_heads_ring_walk
// at K = 1: 4 + 2 + 1 transposing shuffles over all 32 lanes, then two plain ones) and lanes 0, 4, .., 28 store the 8
// results (32 contiguous bytes). Entries are independent: split rows need no fixup.
template <int NV>
__global__ void __launch_bounds__(kSddmmWarps * 32)
sddmm_ring_kernel(const SddmmArgs a)
{
    sddmm_heads_ring_walk<NV, 1>(a, SddmmDot());
}

// Any f, K and alignment: one warp per row block of the register kernel's schedule, one lane per edge (32 edges at a
// time, rows from a ballot of the row-end bits), each lane a sequential fp32 dot product per head over its d = f / K
// features.
__device__ __forceinline__ void sddmm_plain_walk(const SddmmArgs& a, int K)
{
    const int lane = threadIdx.x & 31;
    const int w = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    if (w >= a.nblocks) return;
    const int4 b = __ldg(a.blocks + w);
    const bool seg = b.y < 0;
    const int d = a.f / K;
    int row = b.x;
    for (int e = b.z; e < b.w; e += 32) {
        const int ei = e + lane;
        const bool ok = ei < b.w;
        int col = 0;
        bool end = false;
        if (ok) {
            const int* pc = a.pieces + (size_t)(ei >> 5) * kPieceInts;
            col = __ldg(pc + (ei & 31));
            end = !seg && ((__ldg(reinterpret_cast<const unsigned*>(pc + 64)) >> (ei & 31)) & 1u);
        }
        const unsigned ends = __ballot_sync(0xffffffffu, end);
        if (ok) {
            const int r = row + __popc(ends & ((1u << lane) - 1u));
            const int orow = a.rowids ? __ldg(a.rowids + r) : r;
            const float* g = a.gZ + (size_t)(unsigned)orow * a.f;
            const float* hrow = (a.H1 && col >= a.split) ? a.H1 + (size_t)(col - a.split) * a.f : a.H0 + (size_t)col * a.f;
            for (int h = 0; h < K; ++h) {
                float s = 0.f;
                for (int c = h * d; c < (h + 1) * d; ++c) s = fmaf(__ldg(g + c), __ldg(hrow + c), s);
                a.dvals[(size_t)ei * K + h] = s;
            }
        }
        row += __popc(ends);
    }
}

__global__ void __launch_bounds__(256)
sddmm_plain_kernel(const SddmmArgs a)
{
    sddmm_plain_walk(a, 1);
}

__global__ void __launch_bounds__(256)
sddmm_plain_heads_kernel(const SddmmArgs a, int K)
{
    sddmm_plain_walk(a, K);
}

}  // namespace pgcn
