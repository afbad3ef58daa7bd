// spmm_kernels.cuh — sm_90a kernels of the PGCN aggregation path.
//
// Replaces, on an H100:
//   torch.sparse.mm(A, H)        GPU/PGCN.py:127      -> spmm_rowblock_kernel (forward CSR)
//   torch.sparse.mm(A.t(), g)    GPU/PGCN.py:132      -> spmm_rowblock_kernel (pre-transposed CSR)
//   H[send_map[p]] per peer      GPU/PGCN.py:104      -> pack_rows_kernel (all peers, one launch)
//   X[recv_map[p]] = buf         GPU/PGCN.py:115      -> fwd: nothing (SpMM reads the halo slab in place)
//                                                        bwd: unpack_add_kernel (fixed-order sum)
//   GrB_mxm PLUS_TIMES_FP32      Parallel-GCN/main.c:271,295
//
// The SpMM is an HBM/L2-bound sparse gather-reduce (<= 0.5 flop/byte): no tensor cores.
// Design:
//   * the host cuts the row range into "row blocks" of ~equal nnz; one LANE GROUP of LPE lanes
//     (LPE = 4..32, a sub-warp for narrow feature tiles) walks one block's edge range and keeps
//     a segmented running sum: the last entry of every row is marked in bit 31 of its column
//     index and the accumulator is flushed when the mark is met, so column indices and values
//     are read fully coalesced (LPE at a time) no matter how short the rows are and the kernel
//     never touches row pointers;
//   * each gathered H row segment is read with 16-byte loads by consecutive lanes
//     (LPE*16 B contiguous = whole 128-B lines for LPE >= 8), two rows in flight per lane group
//     (register double buffer) times ~48 resident warps per SM;
//   * rows longer than `long_row` are split into segments that write partial sums to a side
//     buffer; a second tiny kernel adds the segments in a fixed order (deterministic, no atomics);
//   * blockIdx.y walks feature tiles, so a wide H can be processed one L2-resident column slice
//     at a time (tile_floats option) and any f is supported (scalar path when f % 4 != 0 or an operand is not
//     16-byte aligned: .v4 accesses need natural alignment).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pgcn {

// Bit 31 of a stored column index marks the LAST entry of its row: the kernel needs no row
// pointers at all — it walks a block's edge range and flushes when it meets the mark.
// Bit 30 marks a COLD column (few references): its H row is loaded with an L2 evict_first policy
// while the hot rows (hubs, the part of H that fits in L2) are loaded evict_last, so streaming
// traffic does not push the re-used rows out of the 50 MB L2.
// Device layout of a CSR's entries: consecutive PIECES of 32 entries, one 272-byte record each (one TMA bulk copy):
//   int   col[32]    plain column indices (no flag bits: they go straight into TMA row coordinates)
//   float val[32]
//   uint  emask      bit i: entry i is the LAST of its row        uint cmask   bit i: entry i's column is COLD
//   uint  smask      bit i: entry i's column is COLD for 64-float slices (the ring kernel's larger slice hot set)
//   uint  pad
// Entry e lives in piece e >> 5 at index e & 31. The register kernel rebuilds {col | flags, val} pairs as it loads.
constexpr int kPieceInts = 68;
constexpr int kPieceBytes = kPieceInts * 4;
constexpr int kLastFlag = (int)0x80000000;
constexpr int kColdFlag = 0x40000000;
constexpr int kColMask = 0x3fffffff;

#ifndef PGCN_LDMODE
#define PGCN_LDMODE 2      // 0: ld.global.nc   1: + L1::no_allocate   2: L2 hot/cold hints   3: 2 + L1::no_allocate
#endif

struct SpmmArgs {
    const int4* blocks;      // {first row (compact id), nrows | -(slot+1), e_begin, e_end}
    int nblocks;
    const int* pieces;       // the matrix entries in PIECES of 32 (kPieceInts ints = 272 bytes each, see below)
    const float* H0;         // columns [0, split)
    const float* H1;         // columns [split, ...)   (halo slab), may be null when unused
    int split;
    float* Z0;               // output rows [0, zsplit)
    float* Z1;               // output rows [zsplit, ...)
    int zsplit;
    const int* rowids;       // optional: compact row id -> output row (empty rows squeezed out,
                             // or the halo-part matrix that only holds boundary rows)
    float* partial;          // side buffer for split rows, row stride f
    int f;                   // feature width == leading dimension of H0/H1/Z0/Z1/partial
    int beta;                // 0: Z = A*H ; 1: Z += A*H
    // fused layer epilogue (GPU/PGCN.py:144-148 applies relu after the aggregation + dense step): when `relu` is set
    // a row is clamped at zero by the launch that writes it LAST — every row of a single-pass launch
    // (final == nullptr), else the rows whose byte in `final` (indexed by the walked row id) is non-zero
    int relu;
    const unsigned char* final;
    // double-buffered halo slab of the peer-memory exchange: while the plan's exchange epoch (*epoch, device memory) is
    // odd, H_odd replaces the operand that holds the slab (H1 with HALO, else H0). epoch == nullptr: no such operand.
    const float* H_odd;
    const unsigned long long* epoch;
};

// The exchange epoch lives on the device so that a captured CUDA graph sees the value of the replay, not the value of
// the capture: a fused multi-rank call advances it on its stream, every kernel of the call reads it.
__global__ void epoch_advance_kernel(unsigned long long* epoch) { ++*epoch; }

__device__ __forceinline__ bool epoch_odd(const unsigned long long* epoch) { return epoch != nullptr && (*epoch & 1ull); }

// relu that keeps NaN, as torch.relu does (fmaxf(NaN, 0) would return 0 and hide a diverging run). max.NaN (sm_80+) is
// the same single min/max instruction as fmaxf, so the kernels keep their registers; finite results are fmaxf's.
__device__ __forceinline__ float relu1(float x)
{
    float r;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float4 vrelu(const float4& a) { return make_float4(relu1(a.x), relu1(a.y), relu1(a.z), relu1(a.w)); }
__device__ __forceinline__ float vrelu(const float& a) { return relu1(a); }

template <int VW> struct Vec;
template <> struct Vec<4> { typedef float4 type; };
template <> struct Vec<1> { typedef float type; };

__device__ __forceinline__ float4 vzero(float4*) { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float vzero(float*) { return 0.f; }
__device__ __forceinline__ void vfma(float4& a, float w, const float4& r) {
    a.x = fmaf(w, r.x, a.x); a.y = fmaf(w, r.y, a.y); a.z = fmaf(w, r.z, a.z); a.w = fmaf(w, r.w, a.w);
}
__device__ __forceinline__ void vfma(float& a, float w, const float& r) { a = fmaf(w, r, a); }
__device__ __forceinline__ void vfma(float2& a, float w, const float2& r) { a.x = fmaf(w, r.x, a.x); a.y = fmaf(w, r.y, a.y); }
__device__ __forceinline__ void vadd(float2& a, const float2& r) { a.x += r.x; a.y += r.y; }
__device__ __forceinline__ float2 vrelu(const float2& a) { return make_float2(relu1(a.x), relu1(a.y)); }
__device__ __forceinline__ float2 vzero(float2*) { return make_float2(0.f, 0.f); }
__device__ __forceinline__ void vadd(float4& a, const float4& r) { a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w; }
__device__ __forceinline__ void vadd(float& a, const float& r) { a += r; }

// H rows: read-only path, default L1/L2 allocation (hub rows are re-used).
__device__ __forceinline__ float4 ld_feat(const float4* p) { return __ldg(p); }
__device__ __forceinline__ float ld_feat(const float* p) { return __ldg(p); }

__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// gather of one H-row vector with an explicit L2 eviction policy
__device__ __forceinline__ float4 ld_feat_hint(const float4* p, unsigned long long pol) {
    float4 r;
#if PGCN_LDMODE == 3
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol));
#elif PGCN_LDMODE == 2
    asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol));
#elif PGCN_LDMODE == 1
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
#else
    r = __ldg(p);
#endif
    return r;
}
__device__ __forceinline__ float ld_feat_hint(const float* p, unsigned long long pol) {
    float r;
#if PGCN_LDMODE >= 2
    asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
#else
    r = __ldg(p);
#endif
    return r;
}
// column indices / values: touched once -> streaming, do not displace H rows.
// entry e of the piece array as the {column | kLastFlag | kColdFlag, value bits} pair the register kernel walks
__device__ __forceinline__ int2 ld_entry(const int* pieces, int e)
{
    const int* pc = pieces + (size_t)(e >> 5) * kPieceInts;
    const int i = e & 31;
    const int col = __ldcs(pc + i);
    const int val = __ldcs(pc + 32 + i);
    const int2 m = __ldcs(reinterpret_cast<const int2*>(pc + 64));
    return make_int2(col | (((unsigned)m.x >> i) & 1u ? kLastFlag : 0) | (((unsigned)m.y >> i) & 1u ? kColdFlag : 0), val);
}
// outputs: written once -> streaming stores.
__device__ __forceinline__ void st_out(float4* p, const float4& v) { __stcs(p, v); }
__device__ __forceinline__ void st_out(float* p, const float& v) { __stcs(p, v); }
__device__ __forceinline__ void st_out(float2* p, const float2& v) { __stcs(p, v); }

constexpr int kSpmmThreads = 256;

// LPE lanes per edge group, VPL vectors per lane, VW floats per vector; gathers are issued in
// groups of U rows and double-buffered, so up to 2U rows are in flight per lane group.
// Occupancy target: the gathers are latency-bound and 2 rows in flight per lane group with ~48
// resident warps per SM measured best (deeper per-warp pipelines only cost registers), so the
// register budget is capped to keep 6 CTAs of 256 threads per SM for the one-vector-per-lane case.
#ifndef PGCN_OCC
#define PGCN_OCC 2
#endif
constexpr int spmm_min_ctas(int vpl)
{
#if PGCN_OCC == 0
    return 1;                                   // let ptxas pick the register count
#elif PGCN_OCC == 1
    return vpl <= 1 ? 8 : (vpl <= 2 ? 6 : 4);
#else
    return vpl <= 1 ? 6 : (vpl <= 2 ? 5 : 3);
#endif
}

// LPE lanes per edge group, VPL vectors per lane, VW floats per vector, HALO: columns >= split
// live in a second base pointer (the halo slab).
//
// Per chunk of LPE edges a lane group stages its (column|flags, value) pairs in shared memory, so
// the inner loop costs one broadcast LDS.64 per edge instead of two divergence-guarded shuffles;
// the H row address is one IMAD.WIDE.U32 (32-bit column x row pitch in bytes + 64-bit base); the
// own/halo base is a select, not a branch; full chunks run a predicate-free loop. Two gathers are in
// flight per lane group (register double buffer A/B); the next chunk's index pairs are already in
// flight in registers while the current chunk is processed.
template <int LPE, int VPL, int VW, bool HALO>
__global__ void __launch_bounds__(kSpmmThreads, spmm_min_ctas(VPL))
spmm_rowblock_kernel(const SpmmArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    __shared__ int2 s_cw[2][kSpmmThreads];

    const int lane_w = threadIdx.x & 31;
    const int gl = threadIdx.x & (LPE - 1);
    const int gbase = threadIdx.x & ~(LPE - 1);
    const unsigned gmask = (LPE == 32) ? 0xffffffffu
                                       : (((1u << (LPE & 31)) - 1u) << (lane_w & ~(LPE - 1)));
    const int group = (int)((blockIdx.x * (unsigned)kSpmmThreads + threadIdx.x) / LPE);
    if (group >= a.nblocks) return;           // whole lane groups leave together

    const int4 b = a.blocks[group];
    const bool seg = b.y < 0;                 // a segment of one split row: row marks are ignored
    const int lastmask = seg ? 0 : kLastFlag;
    const int e_end = b.w;
    int e = b.z;
    int row = b.x;

    // this lane's slice of a feature row: byte offset of its first vector inside the row
    const unsigned pitch = (unsigned)a.f * 4u;                       // row pitch in bytes
    const int f0 = blockIdx.y * (LPE * VPL * VW) + gl * VW;          // first float of vector 0
    bool fok[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) fok[v] = f0 + v * LPE * VW < a.f;  // f % VW == 0 (launcher)
    const bool odd = epoch_odd(a.epoch);
    const float* H0 = (!HALO && odd) ? a.H_odd : a.H0;
    const float* H1 = (HALO && odd) ? a.H_odd : a.H1;
    const char* hb0 = reinterpret_cast<const char*>(H0) + (size_t)f0 * 4;
    const char* hb1 = HALO ? reinterpret_cast<const char*>(H1) + (size_t)f0 * 4 - (size_t)a.split * pitch
                           : hb0;

#if PGCN_LDMODE >= 2
    const unsigned long long pol_hot = l2_policy_evict_last();
    const unsigned long long pol_cold = l2_policy_evict_first();
#endif

    vec_t acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = vzero((vec_t*)nullptr);

    auto flush_row = [&]() {
        // write the finished row, clear the accumulator, advance to the next row of the block
        const int orow = (a.rowids != nullptr) ? __ldg(a.rowids + row) : row;
        const bool relu_row = a.relu && (a.final == nullptr || __ldg(a.final + row) != 0);
        char* zb = (orow < a.zsplit)
                       ? reinterpret_cast<char*>(a.Z0) + (size_t)(unsigned)orow * pitch
                       : reinterpret_cast<char*>(a.Z1) + (size_t)(unsigned)(orow - a.zsplit) * pitch;
        zb += (size_t)f0 * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            if (fok[v]) {
                vec_t* zp = reinterpret_cast<vec_t*>(zb + v * LPE * VW * 4);
                if (a.beta) vadd(acc[v], *zp);
                if (relu_row) acc[v] = vrelu(acc[v]);
                st_out(zp, acc[v]);
            }
            acc[v] = vzero((vec_t*)nullptr);
        }
        ++row;
    };

    auto gather = [&](vec_t (&r)[VPL], int craw) {
        const unsigned cj = (unsigned)(craw & kColMask);
        const char* hb = (HALO && cj >= (unsigned)a.split) ? hb1 : hb0;
        const char* hp = hb + (size_t)cj * pitch;
#if PGCN_LDMODE >= 2
        const unsigned long long pol = (craw & kColdFlag) ? pol_cold : pol_hot;
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) r[v] = ld_feat_hint(reinterpret_cast<const vec_t*>(hp + v * LPE * VW * 4), pol);
#else
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) r[v] = ld_feat(reinterpret_cast<const vec_t*>(hp + v * LPE * VW * 4));
#endif
    };
    auto consume = [&](const vec_t (&r)[VPL], int2 cw) {
        const float w = __int_as_float(cw.y);
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) vfma(acc[v], w, r[v]);
        if (cw.x & lastmask) flush_row();
    };

    // chunk 0 -> shared; chunk 1 -> registers (in flight)
    int buf = 0;
    {
        int2 cw = make_int2(0, 0);
        if (e + gl < e_end) cw = ld_entry(a.pieces, e + gl);
        s_cw[0][threadIdx.x] = cw;
    }
    int2 cw_next = make_int2(0, 0);
    if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
    __syncwarp(gmask);

    while (e < e_end) {
        const int n = min(LPE, e_end - e);
        const int2* cwp = &s_cw[buf][gbase];
        // two register buffers: edge j+1 is gathered before edge j is consumed. (A ring of 4 buffers
        // was measured 27 % SLOWER on C2: 1.31 vs 1.03 ms — deeper per-warp pipelines lose to occupancy.)
        vec_t rA[VPL], rB[VPL];
        int2 cwA = cwp[0], cwB;
        gather(rA, cwA.x);
        if (n == LPE) {
            // full chunk: no bounds predicates inside
#pragma unroll 1
            for (int j = 0; j < LPE - 2; j += 2) {
                cwB = cwp[j + 1];
                gather(rB, cwB.x);
                consume(rA, cwA);
                cwA = cwp[j + 2];
                gather(rA, cwA.x);
                consume(rB, cwB);
            }
            cwB = cwp[LPE - 1];
            gather(rB, cwB.x);
            consume(rA, cwA);
            consume(rB, cwB);
        } else {
#pragma unroll 1
            for (int j = 0; j < n; j += 2) {
                const bool hasB = j + 1 < n;
                if (hasB) { cwB = cwp[j + 1]; gather(rB, cwB.x); }
                consume(rA, cwA);
                if (j + 2 < n) { cwA = cwp[j + 2]; gather(rA, cwA.x); }
                if (hasB) consume(rB, cwB);
            }
        }
        e += n;
        // publish the next chunk (it has been in flight since the previous iteration), fetch the one after
        buf ^= 1;
        s_cw[buf][threadIdx.x] = cw_next;
        cw_next = make_int2(0, 0);
        if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
        __syncwarp(gmask);
    }

    if (seg) {
        char* pb = reinterpret_cast<char*>(a.partial) + (size_t)(unsigned)(-b.y - 1) * pitch + (size_t)f0 * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) *reinterpret_cast<vec_t*>(pb + v * LPE * VW * 4) = acc[v];
    }
}

// Weights of the multi-head aggregation (spmm_heads_kernel): alpha is nnz x NH in forward CSR order; amap takes an
// entry of the launched records to its forward entry (null: the identity, the forward records themselves); hd = f / NH.
struct SpmmHeadArgs {
    const float* alpha;
    const int* amap;
    int hd;
};

// The staged head weights of the NH-head instances: two chunks of NH floats per thread, next to s_cw.
template <int NH>
__device__ __forceinline__ float* spmm_head_smem()
{
    __shared__ float s_al[2 * kSpmmThreads * NH];
    return s_al;
}

// Multi-head aggregation: spmm_rowblock_kernel with one vector per lane (VPL = 1: the rest of a wide row is walked in
// blockIdx.y tiles) and another weight. Vector v of a lane is weighted by alpha[map(e) * NH + head], head = (its first
// float) / hd, instead of the entry's value: the same rows, segments, flushes and summation order. The NH weights of a
// chunk's entries are staged in shared memory next to s_cw, and the next chunk's are in flight in registers.
// Registers: 4 CTAs of 256 threads per SM instead of 6 (the NH staged weights in flight). The chunk staging and the
// register double buffer are spmm_rowblock_kernel's (see its comment).
template <int LPE, int VW, bool HALO, int NH>
__global__ void __launch_bounds__(kSpmmThreads, 4)
spmm_heads_kernel(const SpmmArgs a, const SpmmHeadArgs ha)
{
    constexpr int VPL = 1;
    typedef typename Vec<VW>::type vec_t;
    __shared__ int2 s_cw[2][kSpmmThreads];

    const int lane_w = threadIdx.x & 31;
    const int gl = threadIdx.x & (LPE - 1);
    const int gbase = threadIdx.x & ~(LPE - 1);
    const unsigned gmask = (LPE == 32) ? 0xffffffffu
                                       : (((1u << (LPE & 31)) - 1u) << (lane_w & ~(LPE - 1)));
    const int group = (int)((blockIdx.x * (unsigned)kSpmmThreads + threadIdx.x) / LPE);
    if (group >= a.nblocks) return;           // whole lane groups leave together

    const int4 b = a.blocks[group];
    const bool seg = b.y < 0;                 // a segment of one split row: row marks are ignored
    const int lastmask = seg ? 0 : kLastFlag;
    const int e_end = b.w;
    int e = b.z;
    int row = b.x;

    // this lane's slice of a feature row: byte offset of its first vector inside the row
    const unsigned pitch = (unsigned)a.f * 4u;                       // row pitch in bytes
    const int f0 = blockIdx.y * (LPE * VPL * VW) + gl * VW;          // first float of vector 0
    bool fok[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) fok[v] = f0 + v * LPE * VW < a.f;  // f % VW == 0 (launcher)
    const bool odd = epoch_odd(a.epoch);
    const float* H0 = (!HALO && odd) ? a.H_odd : a.H0;
    const float* H1 = (HALO && odd) ? a.H_odd : a.H1;
    const char* hb0 = reinterpret_cast<const char*>(H0) + (size_t)f0 * 4;
    const char* hb1 = HALO ? reinterpret_cast<const char*>(H1) + (size_t)f0 * 4 - (size_t)a.split * pitch
                           : hb0;
    // the head of each vector (a vector never straddles two heads: hd % VW == 0, launcher)
    float* s_al = spmm_head_smem<NH>();
    int hv[VPL];
    float al_next[NH];
#pragma unroll
    for (int v = 0; v < VPL; ++v) hv[v] = fok[v] ? (f0 + v * LPE * VW) / ha.hd : 0;
    // the NH weights of entry ee (zero past the block's end)
    auto ld_alpha = [&](float (&al)[NH], int ee) {
        const bool ok = ee < e_end;
        const int me = !ok ? 0 : (ha.amap ? __ldg(ha.amap + ee) : ee);
#pragma unroll
        for (int h = 0; h < NH; ++h) al[h] = ok ? __ldg(ha.alpha + (size_t)me * NH + h) : 0.f;
    };
    auto st_alpha = [&](int bf, const float (&al)[NH]) {
#pragma unroll
        for (int h = 0; h < NH; ++h) s_al[((size_t)bf * kSpmmThreads + threadIdx.x) * NH + h] = al[h];
    };

#if PGCN_LDMODE >= 2
    const unsigned long long pol_hot = l2_policy_evict_last();
    const unsigned long long pol_cold = l2_policy_evict_first();
#endif

    vec_t acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = vzero((vec_t*)nullptr);

    auto flush_row = [&]() {
        // write the finished row, clear the accumulator, advance to the next row of the block
        const int orow = (a.rowids != nullptr) ? __ldg(a.rowids + row) : row;
        const bool relu_row = a.relu && (a.final == nullptr || __ldg(a.final + row) != 0);
        char* zb = (orow < a.zsplit)
                       ? reinterpret_cast<char*>(a.Z0) + (size_t)(unsigned)orow * pitch
                       : reinterpret_cast<char*>(a.Z1) + (size_t)(unsigned)(orow - a.zsplit) * pitch;
        zb += (size_t)f0 * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            if (fok[v]) {
                vec_t* zp = reinterpret_cast<vec_t*>(zb + v * LPE * VW * 4);
                if (a.beta) vadd(acc[v], *zp);
                if (relu_row) acc[v] = vrelu(acc[v]);
                st_out(zp, acc[v]);
            }
            acc[v] = vzero((vec_t*)nullptr);
        }
        ++row;
    };

    auto gather = [&](vec_t (&r)[VPL], int craw) {
        const unsigned cj = (unsigned)(craw & kColMask);
        const char* hb = (HALO && cj >= (unsigned)a.split) ? hb1 : hb0;
        const char* hp = hb + (size_t)cj * pitch;
#if PGCN_LDMODE >= 2
        const unsigned long long pol = (craw & kColdFlag) ? pol_cold : pol_hot;
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) r[v] = ld_feat_hint(reinterpret_cast<const vec_t*>(hp + v * LPE * VW * 4), pol);
#else
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) r[v] = ld_feat(reinterpret_cast<const vec_t*>(hp + v * LPE * VW * 4));
#endif
    };
    auto consume = [&](const vec_t (&r)[VPL], int2 cw, int j, int bf) {
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) vfma(acc[v], s_al[((size_t)bf * kSpmmThreads + gbase + j) * NH + hv[v]], r[v]);
        if (cw.x & lastmask) flush_row();
    };

    // chunk 0 -> shared; chunk 1 -> registers (in flight)
    int buf = 0;
    {
        int2 cw = make_int2(0, 0);
        if (e + gl < e_end) cw = ld_entry(a.pieces, e + gl);
        s_cw[0][threadIdx.x] = cw;
        float al[NH];
        ld_alpha(al, e + gl);
        st_alpha(0, al);
    }
    int2 cw_next = make_int2(0, 0);
    if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
    ld_alpha(al_next, e + LPE + gl);
    __syncwarp(gmask);

    while (e < e_end) {
        const int n = min(LPE, e_end - e);
        const int2* cwp = &s_cw[buf][gbase];
        // two register buffers: edge j+1 is gathered before edge j is consumed. (A ring of 4 buffers
        // was measured 27 % SLOWER on C2: 1.31 vs 1.03 ms — deeper per-warp pipelines lose to occupancy.)
        vec_t rA[VPL], rB[VPL];
        int2 cwA = cwp[0], cwB;
        gather(rA, cwA.x);
        if (n == LPE) {
            // full chunk: no bounds predicates inside
#pragma unroll 1
            for (int j = 0; j < LPE - 2; j += 2) {
                cwB = cwp[j + 1];
                gather(rB, cwB.x);
                consume(rA, cwA, j, buf);
                cwA = cwp[j + 2];
                gather(rA, cwA.x);
                consume(rB, cwB, j + 1, buf);
            }
            cwB = cwp[LPE - 1];
            gather(rB, cwB.x);
            consume(rA, cwA, LPE - 2, buf);
            consume(rB, cwB, LPE - 1, buf);
        } else {
#pragma unroll 1
            for (int j = 0; j < n; j += 2) {
                const bool hasB = j + 1 < n;
                if (hasB) { cwB = cwp[j + 1]; gather(rB, cwB.x); }
                consume(rA, cwA, j, buf);
                if (j + 2 < n) { cwA = cwp[j + 2]; gather(rA, cwA.x); }
                if (hasB) consume(rB, cwB, j + 1, buf);
            }
        }
        e += n;
        // publish the next chunk (it has been in flight since the previous iteration), fetch the one after
        buf ^= 1;
        s_cw[buf][threadIdx.x] = cw_next;
        cw_next = make_int2(0, 0);
        if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
        st_alpha(buf, al_next);
        ld_alpha(al_next, e + LPE + gl);
        __syncwarp(gmask);
    }

    if (seg) {
        char* pb = reinterpret_cast<char*>(a.partial) + (size_t)(unsigned)(-b.y - 1) * pitch + (size_t)f0 * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v)
            if (fok[v]) *reinterpret_cast<vec_t*>(pb + v * LPE * VW * 4) = acc[v];
    }
}

// Rows without any stored entry are squeezed out of the schedule; they are zero-filled here.
struct ZeroArgs {
    const int* rows; int nrows_empty;
    float* Z0; float* Z1; int zsplit; int f;
};

template <int VW>
__global__ void __launch_bounds__(256)
zero_rows_kernel(const ZeroArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    const int nvec = a.f / VW;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.nrows_empty * nvec) return;
    const int i = (int)(t / nvec);
    const int v = (int)(t - (long long)i * nvec);
    const int orow = __ldg(a.rows + i);
    float* zrow = (orow < a.zsplit) ? a.Z0 + (size_t)orow * a.f : a.Z1 + (size_t)(orow - a.zsplit) * a.f;
    reinterpret_cast<vec_t*>(zrow)[v] = vzero((vec_t*)nullptr);
}

// Z[row] (+)= sum of the row's segments (fixed combination order, run-to-run identical).
struct FixupArgs {
    const int4* long_rows;   // {row, first_slot, nseg, 0}
    int nlong;
    const float* partial;
    float* Z0; float* Z1; int zsplit;
    const int* rowids;
    int f; int beta;
    int relu; const unsigned char* final;
};

// One CTA per (split row, chunk of 32 vectors): 8 warps each sum every 8th segment (independent
// loads in flight), then warp 0 adds the 8 partial sums in a fixed order — deterministic, and ~8x
// shorter dependent chains than one thread per vector (a hub row has hundreds of segments; the
// serial version cost 11 % of the whole aggregation on C2).
constexpr int kFixupGroups = 8;

template <int VW>
__global__ void __launch_bounds__(32 * kFixupGroups)
spmm_fixup_kernel(const FixupArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    __shared__ vec_t s_part[kFixupGroups][32];
    const int nvec = a.f / VW;
    const int chunks = (nvec + 31) / 32;
    const int lr = blockIdx.x / chunks;
    const int v = (blockIdx.x - lr * chunks) * 32 + (threadIdx.x & 31);
    const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int4 d = a.long_rows[lr];                       // {compact row, first slot, nseg, 0}
    vec_t acc = vzero((vec_t*)nullptr);
    if (v < nvec) {
        const vec_t* base = reinterpret_cast<const vec_t*>(a.partial + (size_t)d.y * a.f) + v;
        const size_t stride = (size_t)a.f / VW;           // vectors per partial row
        int i = grp;
        for (; i + 3 * kFixupGroups < d.z; i += 4 * kFixupGroups) {
            const vec_t x0 = __ldcs(base + (size_t)i * stride);
            const vec_t x1 = __ldcs(base + (size_t)(i + kFixupGroups) * stride);
            const vec_t x2 = __ldcs(base + (size_t)(i + 2 * kFixupGroups) * stride);
            const vec_t x3 = __ldcs(base + (size_t)(i + 3 * kFixupGroups) * stride);
            vadd(acc, x0); vadd(acc, x1); vadd(acc, x2); vadd(acc, x3);
        }
        for (; i < d.z; i += kFixupGroups) vadd(acc, __ldcs(base + (size_t)i * stride));
    }
    s_part[grp][lane] = acc;
    __syncthreads();
    if (grp == 0 && v < nvec) {
        vec_t t = s_part[0][lane];
#pragma unroll
        for (int g = 1; g < kFixupGroups; ++g) vadd(t, s_part[g][lane]);
        const int orow = a.rowids ? __ldg(a.rowids + d.x) : d.x;
        float* zrow = (orow < a.zsplit) ? a.Z0 + (size_t)orow * a.f : a.Z1 + (size_t)(orow - a.zsplit) * a.f;
        vec_t* zp = reinterpret_cast<vec_t*>(zrow) + v;
        if (a.beta) vadd(t, *zp);
        if (a.relu && (a.final == nullptr || __ldg(a.final + d.x) != 0)) t = vrelu(t);
        *zp = t;
    }
}

// send_slab[j, :] = H[send_idx[j], :] for all peers in one launch (the staging copy of the NCCL transport and the
// step-by-step entry point pgcn_pack; the peer-memory transport uses put_rows_kernel instead).
struct PackArgs {
    const int* send_idx;       // S
    long long S;
    const float* H;
    float* slab;
    int f;
};

template <int VW>
__global__ void __launch_bounds__(256)
pack_rows_kernel(const PackArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    const int nvec = a.f / VW;
    const long long total = a.S * nvec;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const long long j = t / nvec;
        const int v = (int)(t - j * nvec);
        const int src = __ldg(a.send_idx + j);
        reinterpret_cast<vec_t*>(a.slab + (size_t)j * a.f)[v] =
            ld_feat(reinterpret_cast<const vec_t*>(a.H + (size_t)src * a.f) + v);
    }
}

// One destination of the peer-memory exchange, fused: gather (or copy) the rows that go to ONE peer, store them
// straight into that peer's slab through its NVLink-mapped address, and publish the epoch flag once the last
// CTA's stores are visible system-wide. No staging slab, no separate signal launch, and the receiver can start
// on this peer's rows while the rows of the other peers are still in flight (Parallel-GCN/main.c:275-299:
// MPI_Waitany -> accumulate per received block).
//   forward : rows = H[send_idx[j0 .. j0+nrows)]      (GPU/PGCN.py:104 per peer)
//   backward: rows = src[j0 .. j0+nrows) (halo partials of A^T g, already in wire order; send_idx == nullptr)
struct PutArgs {
    const int* send_idx;             // null: identity (row j0 + i of src)
    long long j0, nrows;
    const float* src;
    float* dst[2];                   // "rows from me" inside the peer's slab, per epoch parity
    int f;
    unsigned int* done;              // CTA completion counter of this destination (self-resetting)
    unsigned long long* flag;        // peer's flag slot for me
    const unsigned long long* epoch; // this plan's exchange epoch (already advanced for this call)
};

template <int VW>
__global__ void __launch_bounds__(256)
put_rows_kernel(const PutArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    const unsigned long long epoch = *a.epoch;
    float* dst = (epoch & 1ull) ? a.dst[1] : a.dst[0];
    const int nvec = a.f / VW;
    const long long total = a.nrows * nvec;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const long long i = t / nvec;
        const int v = (int)(t - i * nvec);
        const long long srow = a.send_idx ? (long long)__ldg(a.send_idx + a.j0 + i) : a.j0 + i;
        const vec_t val = ld_feat(reinterpret_cast<const vec_t*>(a.src + (size_t)srow * a.f) + v);
        reinterpret_cast<vec_t*>(dst + (size_t)i * a.f)[v] = val;
    }
    // last CTA out publishes the epoch: every CTA fences its own stores system-wide before it counts itself
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const unsigned int t = atomicAdd(a.done, 1u);
        if (t == gridDim.x - 1) {
            atomicExch(a.done, 0u);
            __threadfence_system();
            asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(a.flag), "l"(epoch) : "memory");
        }
    }
}

// Spin until ONE peer's slot in my flag array has reached my epoch (one tiny CTA: it never competes for SMs with
// the kernels whose stores it waits for).
__global__ void p2p_wait_kernel(const unsigned long long* flag, const unsigned long long* my_epoch)
{
    if (threadIdx.x == 0) {
        const unsigned long long epoch = *my_epoch;
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
        } while (v < epoch);
        __threadfence_system();
    }
}

// G[brow[i], :] += sum_{q in bpos[bptr[i] .. bptr[i+1])} recv[q, :], in list order.
struct UnpackArgs {
    const int* brow;     // nb boundary rows (local ids)
    const int* bptr;     // nb + 1
    const int* bpos;     // positions in the recv slab
    int nb;
    const float* recv;
    float* G;
    int f;
    const float* recv_odd;               // the peer transport's reverse slab of odd epochs (with `epoch`, else null)
    const unsigned long long* epoch;
};

template <int VW>
__global__ void __launch_bounds__(256)
unpack_add_kernel(const UnpackArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    const float* recv = epoch_odd(a.epoch) ? a.recv_odd : a.recv;
    const int nvec = a.f / VW;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.nb * nvec) return;
    const int i = (int)(t / nvec);
    const int v = (int)(t - (long long)i * nvec);
    const int r = __ldg(a.brow + i);
    vec_t* gp = reinterpret_cast<vec_t*>(a.G + (size_t)r * a.f) + v;
    vec_t s = *gp;
    const int q0 = __ldg(a.bptr + i), q1 = __ldg(a.bptr + i + 1);
    for (int q = q0; q < q1; ++q)
        vadd(s, __ldcs(reinterpret_cast<const vec_t*>(recv + (size_t)__ldg(a.bpos + q) * a.f) + v));
    *gp = s;
}

}  // namespace pgcn
