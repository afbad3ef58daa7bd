// spmm_max.cuh — sm_90a kernels of the max aggregation (GraphSAGE "pool", PyG aggr="max").
//
//   Z[i, c]   = X[col(e*), c],  X = [H_own ; H_halo]
//   arg[i, c] = e*, the FIRST stored entry of row i (forward CSR order) whose X value is >= every other entry's,
//               NaN counting as larger than any number: numpy.argmax over the row. Values of A are not read.
//   rows without an entry: Z = 0, arg = -1
//   backward: G[j, c] = sum of gZ[i, c] over the rows i whose arg[i, c] is an entry of column j
//
// Both kernels are siblings of the register SpMM (spmm_kernels.cuh): the same row blocks, split-row segments, chunks of
// LPE index pairs staged in shared memory, two gathers in flight, one vector per lane with wide rows in blockIdx.y tiles
// and the halo slab picked by the epoch parity. The forward carries a (value, entry) pair per float in place of the FMA;
// a max is exact, so Z equals a serial scan bit for bit whatever the block size, width or alignment. The backward walks
// the transposed records and adds gZ where the forward's arg names the forward entry of the walked record.
#pragma once
#include "spmm_kernels.cuh"

namespace pgcn {

template <int VW> struct IVec;
template <> struct IVec<4> { typedef int4 type; };
template <> struct IVec<1> { typedef int type; };

__device__ __forceinline__ int4 ifill(int4*, int v) { return make_int4(v, v, v, v); }
__device__ __forceinline__ int ifill(int*, int v) { return v; }

// One step of the scan in entry order: x of entry e replaces the best so far when there is none yet, when it is larger,
// or when it is NaN and the best is not. Equal values (and -0.0 / +0.0) keep the earlier entry.
__device__ __forceinline__ void max_step(float& b, int& j, float x, int e)
{
    if (j < 0 || x > b || (isnan(x) && !isnan(b))) { b = x; j = e; }
}
__device__ __forceinline__ void max_step(float4& b, int4& j, const float4& x, int e)
{
    max_step(b.x, j.x, x.x, e); max_step(b.y, j.y, x.y, e); max_step(b.z, j.z, x.z, e); max_step(b.w, j.w, x.w, e);
}

// (x, i) beats (b, j) in the order the scan defines, whatever order candidates are met in: NaN above every number, then
// the larger value, then on equal values the earlier entry. j < 0: no candidate yet.
__device__ __forceinline__ bool max_beats(float x, int i, float b, int j)
{
    if (i < 0) return false;
    if (j < 0) return true;
    const bool xn = isnan(x), bn = isnan(b);
    if (xn != bn) return xn;
    if (!xn && x != b) return x > b;
    return i < j;
}
__device__ __forceinline__ void max_merge(float& b, int& j, float x, int i)
{
    if (max_beats(x, i, b, j)) { b = x; j = i; }
}
__device__ __forceinline__ void max_merge(float4& b, int4& j, const float4& x, const int4& i)
{
    max_merge(b.x, j.x, x.x, i.x); max_merge(b.y, j.y, x.y, i.y); max_merge(b.z, j.z, x.z, i.z); max_merge(b.w, j.w, x.w, i.w);
}

// a += g where the forward's arg names entry fe
__device__ __forceinline__ void add_routed(float& a, const float& g, int ia, int fe) { if (ia == fe) a += g; }
__device__ __forceinline__ void add_routed(float4& a, const float4& g, const int4& ia, int fe)
{
    add_routed(a.x, g.x, ia.x, fe); add_routed(a.y, g.y, ia.y, fe); add_routed(a.z, g.z, ia.z, fe); add_routed(a.w, g.w, ia.w, fe);
}

__device__ __forceinline__ int4 ld_arg_hint(const int4* p, unsigned long long pol)
{
    int4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ int ld_arg_hint(const int* p, unsigned long long pol)
{
    int r;
    asm volatile("ld.global.nc.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
    return r;
}

// Forward: the launch walks the forward records of the register schedule; arg has Z0's layout (row stride f); apart is
// the int partial of the split rows next to a.partial (a split row's segments write their (value, entry) pairs there).
// Only Z0 is written (the forward's rows are all below zsplit); beta, relu and H1 / Z1 of the sum kernel do not apply.
template <int LPE, int VW, bool HALO>
__global__ void __launch_bounds__(kSpmmThreads, 4)
spmm_max_kernel(const SpmmArgs a, int* __restrict__ arg, int* __restrict__ apart)
{
    typedef typename Vec<VW>::type vec_t;
    typedef typename IVec<VW>::type ivec_t;
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

    const unsigned pitch = (unsigned)a.f * 4u;                       // row pitch in bytes (floats and ints alike)
    const int f0 = blockIdx.y * (LPE * VW) + gl * VW;                // first float of this lane's vector
    const bool fok = f0 < a.f;                                       // f % VW == 0 (launcher)
    const bool odd = epoch_odd(a.epoch);
    const float* H0 = (!HALO && odd) ? a.H_odd : a.H0;
    const float* H1 = (HALO && odd) ? a.H_odd : a.H1;
    const char* hb0 = reinterpret_cast<const char*>(H0) + (size_t)f0 * 4;
    const char* hb1 = HALO ? reinterpret_cast<const char*>(H1) + (size_t)f0 * 4 - (size_t)a.split * pitch
                           : hb0;
    const unsigned long long pol_hot = l2_policy_evict_last();
    const unsigned long long pol_cold = l2_policy_evict_first();

    vec_t best = vzero((vec_t*)nullptr);
    ivec_t ent = ifill((ivec_t*)nullptr, -1);

    auto flush_row = [&]() {
        const int orow = (a.rowids != nullptr) ? __ldg(a.rowids + row) : row;
        const size_t off = (size_t)(unsigned)orow * pitch + (size_t)f0 * 4;
        if (fok) {
            st_out(reinterpret_cast<vec_t*>(reinterpret_cast<char*>(a.Z0) + off), best);
            __stcs(reinterpret_cast<ivec_t*>(reinterpret_cast<char*>(arg) + off), ent);
        }
        best = vzero((vec_t*)nullptr);
        ent = ifill((ivec_t*)nullptr, -1);
        ++row;
    };
    auto gather = [&](vec_t& r, int craw) {
        const unsigned cj = (unsigned)(craw & kColMask);
        const char* hb = (HALO && cj >= (unsigned)a.split) ? hb1 : hb0;
        const unsigned long long pol = (craw & kColdFlag) ? pol_cold : pol_hot;
        if (fok) r = ld_feat_hint(reinterpret_cast<const vec_t*>(hb + (size_t)cj * pitch), pol);
    };
    auto consume = [&](const vec_t& r, int2 cw, int ee) {
        if (fok) max_step(best, ent, r, ee);
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
        vec_t rA, rB;
        int2 cwA = cwp[0], cwB;
        gather(rA, cwA.x);
        if (n == LPE) {
#pragma unroll 1
            for (int j = 0; j < LPE - 2; j += 2) {
                cwB = cwp[j + 1];
                gather(rB, cwB.x);
                consume(rA, cwA, e + j);
                cwA = cwp[j + 2];
                gather(rA, cwA.x);
                consume(rB, cwB, e + j + 1);
            }
            cwB = cwp[LPE - 1];
            gather(rB, cwB.x);
            consume(rA, cwA, e + LPE - 2);
            consume(rB, cwB, e + LPE - 1);
        } else {
#pragma unroll 1
            for (int j = 0; j < n; j += 2) {
                const bool hasB = j + 1 < n;
                if (hasB) { cwB = cwp[j + 1]; gather(rB, cwB.x); }
                consume(rA, cwA, e + j);
                if (j + 2 < n) { cwA = cwp[j + 2]; gather(rA, cwA.x); }
                if (hasB) consume(rB, cwB, e + j + 1);
            }
        }
        e += n;
        buf ^= 1;
        s_cw[buf][threadIdx.x] = cw_next;
        cw_next = make_int2(0, 0);
        if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
        __syncwarp(gmask);
    }

    if (seg && fok) {
        const size_t off = (size_t)(unsigned)(-b.y - 1) * pitch + (size_t)f0 * 4;
        *reinterpret_cast<vec_t*>(reinterpret_cast<char*>(a.partial) + off) = best;
        *reinterpret_cast<ivec_t*>(reinterpret_cast<char*>(apart) + off) = ent;
    }
}

// The segments of a split row, combined: one CTA per (split row, chunk of 32 vectors), 8 warps each take every 8th
// segment, then warp 0 merges the 8 results. max_merge orders candidates by (value, entry), so the result is the serial
// scan's in any combination order.
struct MaxFixupArgs {
    const int4* long_rows;   // {compact row, first slot, nseg, 0}
    const float* partial;
    const int* apart;
    float* Z;
    int* arg;
    const int* rowids;
    int f;
};

template <int VW>
__global__ void __launch_bounds__(32 * kFixupGroups)
spmm_max_fixup_kernel(const MaxFixupArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    typedef typename IVec<VW>::type ivec_t;
    __shared__ vec_t s_best[kFixupGroups][32];
    __shared__ ivec_t s_ent[kFixupGroups][32];
    const int nvec = a.f / VW;
    const int chunks = (nvec + 31) / 32;
    const int lr = blockIdx.x / chunks;
    const int v = (blockIdx.x - lr * chunks) * 32 + (threadIdx.x & 31);
    const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int4 d = a.long_rows[lr];
    vec_t best = vzero((vec_t*)nullptr);
    ivec_t ent = ifill((ivec_t*)nullptr, -1);
    if (v < nvec) {
        const size_t stride = (size_t)a.f / VW;           // vectors per partial row
        const vec_t* pb = reinterpret_cast<const vec_t*>(a.partial + (size_t)d.y * a.f) + v;
        const ivec_t* pe = reinterpret_cast<const ivec_t*>(a.apart + (size_t)d.y * a.f) + v;
        for (int i = grp; i < d.z; i += kFixupGroups)
            max_merge(best, ent, __ldcs(pb + (size_t)i * stride), __ldcs(pe + (size_t)i * stride));
    }
    s_best[grp][lane] = best;
    s_ent[grp][lane] = ent;
    __syncthreads();
    if (grp == 0 && v < nvec) {
#pragma unroll
        for (int g = 1; g < kFixupGroups; ++g) max_merge(best, ent, s_best[g][lane], s_ent[g][lane]);
        const int orow = a.rowids ? __ldg(a.rowids + d.x) : d.x;
        reinterpret_cast<vec_t*>(a.Z + (size_t)orow * a.f)[v] = best;
        reinterpret_cast<ivec_t*>(a.arg + (size_t)orow * a.f)[v] = ent;
    }
}

// Rows without a stored entry: Z = 0, arg = -1.
struct MaxEmptyArgs {
    const int* rows; int nrows_empty;
    float* Z; int* arg; int f;
};

template <int VW>
__global__ void __launch_bounds__(256)
max_empty_rows_kernel(const MaxEmptyArgs a)
{
    typedef typename Vec<VW>::type vec_t;
    typedef typename IVec<VW>::type ivec_t;
    const int nvec = a.f / VW;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.nrows_empty * nvec) return;
    const int i = (int)(t / nvec);
    const int v = (int)(t - (long long)i * nvec);
    const size_t r = (size_t)__ldg(a.rows + i);
    reinterpret_cast<vec_t*>(a.Z + r * a.f)[v] = vzero((vec_t*)nullptr);
    reinterpret_cast<ivec_t*>(a.arg + r * a.f)[v] = ifill((ivec_t*)nullptr, -1);
}

// Backward: the launch walks the TRANSPOSED records of the register schedule (rows = forward columns, columns = forward
// rows). H0 = gZ; arg (m x f, the forward's) is gathered beside it at the same offsets; amap takes a transposed entry to
// its forward entry (the value map of pgcn_plan_bind_values), staged per chunk in shared memory like the multi-head
// weights. Rows [0, zsplit) go to Z0, the rest to Z1; split rows write float partials that spmm_fixup_kernel sums.
template <int LPE, int VW>
__global__ void __launch_bounds__(kSpmmThreads, 4)
spmm_max_backward_kernel(const SpmmArgs a, const int* __restrict__ arg, const int* __restrict__ amap)
{
    typedef typename Vec<VW>::type vec_t;
    typedef typename IVec<VW>::type ivec_t;
    __shared__ int2 s_cw[2][kSpmmThreads];
    __shared__ int s_fe[2][kSpmmThreads];

    const int lane_w = threadIdx.x & 31;
    const int gl = threadIdx.x & (LPE - 1);
    const int gbase = threadIdx.x & ~(LPE - 1);
    const unsigned gmask = (LPE == 32) ? 0xffffffffu
                                       : (((1u << (LPE & 31)) - 1u) << (lane_w & ~(LPE - 1)));
    const int group = (int)((blockIdx.x * (unsigned)kSpmmThreads + threadIdx.x) / LPE);
    if (group >= a.nblocks) return;           // whole lane groups leave together

    const int4 b = a.blocks[group];
    const bool seg = b.y < 0;
    const int lastmask = seg ? 0 : kLastFlag;
    const int e_end = b.w;
    int e = b.z;
    int row = b.x;

    const unsigned pitch = (unsigned)a.f * 4u;
    const int f0 = blockIdx.y * (LPE * VW) + gl * VW;
    const bool fok = f0 < a.f;
    const char* gb = reinterpret_cast<const char*>(a.H0) + (size_t)f0 * 4;
    const char* ab = reinterpret_cast<const char*>(arg) + (size_t)f0 * 4;
    const unsigned long long pol_hot = l2_policy_evict_last();
    const unsigned long long pol_cold = l2_policy_evict_first();

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
    auto gather = [&](vec_t& g, ivec_t& ia, int craw) {
        const size_t off = (size_t)(unsigned)(craw & kColMask) * pitch;
        const unsigned long long pol = (craw & kColdFlag) ? pol_cold : pol_hot;
        if (fok) {
            g = ld_feat_hint(reinterpret_cast<const vec_t*>(gb + off), pol);
            ia = ld_arg_hint(reinterpret_cast<const ivec_t*>(ab + off), pol);
        }
    };
    auto consume = [&](const vec_t& g, const ivec_t& ia, int2 cw, int j, int bf) {
        if (fok) add_routed(acc, g, ia, s_fe[bf][gbase + j]);
        if (cw.x & lastmask) flush_row();
    };
    auto ld_fe = [&](int ee) { return ee < e_end ? __ldg(amap + ee) : -1; };

    int buf = 0;
    {
        int2 cw = make_int2(0, 0);
        if (e + gl < e_end) cw = ld_entry(a.pieces, e + gl);
        s_cw[0][threadIdx.x] = cw;
        s_fe[0][threadIdx.x] = ld_fe(e + gl);
    }
    int2 cw_next = make_int2(0, 0);
    if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
    int fe_next = ld_fe(e + LPE + gl);
    __syncwarp(gmask);

    while (e < e_end) {
        const int n = min(LPE, e_end - e);
        const int2* cwp = &s_cw[buf][gbase];
        vec_t gA, gB;
        ivec_t iA, iB;
        int2 cwA = cwp[0], cwB;
        gather(gA, iA, cwA.x);
        if (n == LPE) {
#pragma unroll 1
            for (int j = 0; j < LPE - 2; j += 2) {
                cwB = cwp[j + 1];
                gather(gB, iB, cwB.x);
                consume(gA, iA, cwA, j, buf);
                cwA = cwp[j + 2];
                gather(gA, iA, cwA.x);
                consume(gB, iB, cwB, j + 1, buf);
            }
            cwB = cwp[LPE - 1];
            gather(gB, iB, cwB.x);
            consume(gA, iA, cwA, LPE - 2, buf);
            consume(gB, iB, cwB, LPE - 1, buf);
        } else {
#pragma unroll 1
            for (int j = 0; j < n; j += 2) {
                const bool hasB = j + 1 < n;
                if (hasB) { cwB = cwp[j + 1]; gather(gB, iB, cwB.x); }
                consume(gA, iA, cwA, j, buf);
                if (j + 2 < n) { cwA = cwp[j + 2]; gather(gA, iA, cwA.x); }
                if (hasB) consume(gB, iB, cwB, j + 1, buf);
            }
        }
        e += n;
        buf ^= 1;
        s_cw[buf][threadIdx.x] = cw_next;
        s_fe[buf][threadIdx.x] = fe_next;
        cw_next = make_int2(0, 0);
        if (e + LPE + gl < e_end) cw_next = ld_entry(a.pieces, e + LPE + gl);
        fe_next = ld_fe(e + LPE + gl);
        __syncwarp(gmask);
    }

    if (seg && fok) {
        char* pb = reinterpret_cast<char*>(a.partial) + (size_t)(unsigned)(-b.y - 1) * pitch + (size_t)f0 * 4;
        *reinterpret_cast<vec_t*>(pb) = acc;
    }
}

}  // namespace pgcn
