// spmm_ring.cuh — the Hopper (sm_90a) SpMM of the PGCN aggregation path: gathered H rows are staged
// ASYNCHRONOUSLY in shared memory (TMA: 1-D cp.async.bulk or 2-D tensor-map copies, mbarrier complete_tx),
// the segmented FMA runs out of shared memory.
//
// Replaces torch.sparse.mm(A, H) / torch.sparse.mm(A.t(), g) of GPU/PGCN.py:127,132 for feature widths
// that are multiples of 128 floats (the benchmark widths 128 and 256); other widths take the register
// pipeline of spmm_kernels.cuh.
//
// Why: the register-buffered gather of spmm_rowblock_kernel keeps bytes-in-flight in REGISTERS (2 rows per
// warp x 48 warps), spends ~35 issue slots per edge and is capped by occupancy. Here
//   * every WARP owns a private ring of NS row slots (NS x f x 4 bytes of shared memory) and a small ring
//     of index pieces; nothing is shared between warps, so there is no CTA-level synchronisation at all;
//   * lanes 0..G-1 each issue ONE bulk copy (UBLKCP) of a whole H row (512 B at f = 128) per group of G
//     edges; the group's mbarrier completes when all G rows have landed (expect_tx = G x row bytes);
//   * the (column|flags, value) stream is fetched the same way in 256-byte pieces of 32 entries, so the
//     kernel issues no ordinary global loads at all on its hot path;
//   * consumption is one broadcast LDS.64 (index pair) + one conflict-free LDS.128 per edge and lane,
//     4 FFMA, a row-end test; bytes in flight per SM = warps x NS x row bytes (e.g. 12 x 32 x 512 B =
//     192 KB) instead of 48 KB, at ~10 issue slots per edge.
//   * MODE 1 is the same ring filled with per-lane 16-byte cp.async (LDGSTS) copies — kept for comparison.
//   * a slot holds a row TILE of TF floats: the full width (128 or 256) or a 64-float slice (256 B; one LDS.64 and
//     2 FFMA per edge and lane). Slices are walked one after the other, so only TF / f of H is live in L2 at a
//     time: more of the gathered rows hit, for twice the issue work per edge.
// Row blocks come from the same host schedule as the register kernel (rows cut into blocks of about
// edges_per_block entries, long rows split into single-row segments that the fixup kernel sums in a fixed
// order), one block per warp; with `counter` set, the CTAs are persistent and warps fetch blocks dynamically.
#pragma once
#include <cuda.h>
#include "spmm_kernels.cuh"

namespace pgcn {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
// 1-D TMA bulk copy global -> shared, completion counted in bytes on an mbarrier; L2 eviction policy per copy.
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar,
                                         unsigned long long pol)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
// 2-D tensor-map TMA in tile mode: one row tile of H (row r, column offset x; the map's box is {tile, 1 row}) lands
// in one row slot (UTMALDG.2D). The map carries the row pitch, so no address is computed.
// The copy is issued ONCE for the whole warp, by the lane elect.sync picks. Every lane calls it, converged, with
// warp-uniform operands; ptxas then emits a bare UTMALDG fed from uniform registers. A per-lane form (each lane its
// own row) costs a waterfall loop per copy instead: ELECT, six R2UR, two PLOP3 and a branch around each UTMALDG.
__device__ __forceinline__ void tma_row_warp(uint32_t dst, const CUtensorMap* tm, int x, int r, uint32_t bar,
                                            unsigned long long pol)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t"
        "@p cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%2, %3}], [%4], %5;\n\t}"
        ::"r"(dst), "l"(tm), "r"(x), "r"(r), "r"(bar), "l"(pol) : "memory");
}
// A value every lane of the warp holds, moved into a uniform register (REDUX writes one), so that ptxas can treat
// what is computed from it as warp-uniform.
__device__ __forceinline__ uint32_t warp_uniform(uint32_t v) { return __reduce_or_sync(0xffffffffu, v); }
__device__ __forceinline__ unsigned long long warp_uniform64(unsigned long long v)
{
    return ((unsigned long long)warp_uniform((uint32_t)(v >> 32)) << 32) | warp_uniform((uint32_t)v);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, unsigned long long pol)
{
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// One call site per row end would replicate the store sequence 32+ times in the unrolled consumer; keeping it
// out of line keeps the hot loop inside the instruction cache (the rows-end path runs once per ~17 edges).
template <class V, int NV>
__device__ __noinline__ void ring_store_row(V a0, V a1, const int* rowids, int row, float* Z0, float* Z1,
                                            int zsplit, size_t pitch, size_t off, int beta, int relu, const unsigned char* final)
{
    const bool relu_row = relu && (final == nullptr || __ldg(final + row) != 0);
    const int orow = (rowids != nullptr) ? __ldg(rowids + row) : row;
    char* zb = (orow < zsplit) ? reinterpret_cast<char*>(Z0) + (size_t)(unsigned)orow * pitch
                               : reinterpret_cast<char*>(Z1) + (size_t)(unsigned)(orow - zsplit) * pitch;
    zb += off;
    V* zp = reinterpret_cast<V*>(zb);
    if (beta) vadd(a0, *zp);
    if (relu_row) a0 = vrelu(a0);
    st_out(zp, a0);
    if (NV == 2) {
        V* zq = reinterpret_cast<V*>(zb + 512);
        if (beta) vadd(a1, *zq);
        if (relu_row) a1 = vrelu(a1);
        st_out(zq, a1);
    }
}

// Cost probe, for variant builds only (PGCN_B200_VARIANT + PGCN_B200_DEFS=-DPGCN_RING_DIAG=n, timed by
// tools/tune_spmm.py --gather-sweep --all-hit): bit 0 drops the consumer's slot reads and FFMA, bit 1 makes the
// tensor-map ring issue no row copy and wait on none. Such a build computes wrong results; the library is built with 0.
#ifndef PGCN_RING_DIAG
#define PGCN_RING_DIAG 0
#endif
constexpr bool kDiagNoFma = (PGCN_RING_DIAG & 1) != 0, kDiagNoCopy = (PGCN_RING_DIAG & 2) != 0;

constexpr int kRingPieces = 4;       // index pieces (32 entries, kPieceBytes each) resident per warp

struct RingArgs {
    unsigned int* counter;   // null: block blockIdx.x * warps per CTA + warp of tile blockIdx.y; else the next
                             // (tile, block) work item, tile-major (persistent CTAs)
    const float* hub;        // reserved (hub rows resident in shared memory)
    int nhub;
};

// per warp: NS row slots of tf floats | NP index pieces | NG + NP mbarriers
__host__ __device__ constexpr size_t ring_warp_bytes(int tf, int ns, int ng)
{
    return ((size_t)ns * tf * 4 + (size_t)kRingPieces * kPieceBytes + (size_t)(ng + kRingPieces) * 8 + 127) / 128 * 128;
}
// Warps per CTA. The warps are fully independent, so the CTA size only sets the shared-memory granule, and every CTA
// also costs the SM 1 KB of reserved shared memory (sm_90: 228 KB per SM, at most 227 KB per CTA). Where the ring is
// bounded by shared memory, 4-warp CTAs fit more warps per SM than 2-warp CTAs: 24 instead of 22 for the 64-float,
// 32-slot ring (9.1 KB per warp). Otherwise (a tie, or a CTA over 227 KB) CTAs keep 2 warps.
constexpr size_t kSmemPerSm = 228 * 1024, kSmemPerCtaMax = 227 * 1024, kSmemReservedPerCta = 1024;
__host__ __device__ constexpr int ring_resident_warps(size_t warp_bytes, int warps)
{
    return (int)(kSmemPerSm / (warp_bytes * warps + 128 + kSmemReservedPerCta)) * warps;
}
__host__ __device__ constexpr int ring_cta_warps(int tf, int ns, int ng)
{
    return (ring_warp_bytes(tf, ns, ng) * 4 + 128 <= kSmemPerCtaMax &&
            ring_resident_warps(ring_warp_bytes(tf, ns, ng), 4) > ring_resident_warps(ring_warp_bytes(tf, ns, ng), 2)) ? 4 : 2;
}
__host__ __device__ constexpr size_t ring_smem_bytes(int tf, int ns, int ng)
{
    return ring_warp_bytes(tf, ns, ng) * ring_cta_warps(tf, ns, ng) + 128;
}

// What one lane holds of a row tile of TF floats: one float2 (64-float slices, 256 B), one float4 (128 floats) or
// two float4 (256 floats; the second 512 B further on).
template <int TF> struct RingLane { typedef float4 V; static constexpr int NV = TF / 128; };
template <> struct RingLane<64> { typedef float2 V; static constexpr int NV = 1; };

// runtime-indexed access to a tiny register array (compare chain instead of local memory)
template <int N>
__device__ __forceinline__ uint32_t reg_get(const uint32_t (&a)[N], int i)
{
    uint32_t v = a[0];
#pragma unroll
    for (int k = 1; k < N; ++k) v = (i == k) ? a[k] : v;
    return v;
}
template <int N>
__device__ __forceinline__ void reg_set(uint32_t (&a)[N], int i, uint32_t v)
{
#pragma unroll
    for (int k = 0; k < N; ++k) a[k] = (i == k) ? v : a[k];
}

// TF  : floats per row tile (64, 128 or 256; f is walked in f / TF tiles, each one row slot wide).
// G   : edges per completion group (8, 16 or 32); NG: groups in the ring (2 or 4); the warp owns NS = G * NG row slots.
// MODE: 0 = 1-D TMA bulk copies (UBLKCP, one per row), 1 = per-lane 16-byte cp.async (LDGSTS + wait_group),
//       2 = 2-D tensor-map TMA in tile mode (UTMALDG.2D, one row per instruction; own and halo rows through
//           their own tensor map).
// HALO: columns >= split live in a second matrix (the halo slab).
//
// The entries are walked in GLOBALLY ALIGNED units: a piece = entries [32 P, 32 P + 32) (one 272-byte record =
// one bulk copy: 32 plain column indices, 32 values, a row-end bit mask and a cold-column bit mask), a group =
// entries [G g, G g + G) (one completion unit of the row ring, slot group g % NG). A row block [e0, e1) starts and
// ends anywhere; entries of its first / last group outside the block are masked. The steady state per group is:
//   issue   : one broadcast LDS.64 (masks); lane 0 arms the group's mbarrier with G x row bytes. MODE 2: the warp reads
//             the G column indices 4 at a time (broadcast LDS.128), moves each into a uniform register and one
//             elected lane fires the copy (tma_row_warp). MODES 0 / 1: lanes 0..G-1 each copy the row of their column;
//   consume : mbarrier wait, 8 x LDS.128 rows + 2 x LDS.128 values (straight from the resident piece), 32 FFMA per
//             8 edges; a row-end test per edge only in groups whose row-end mask is non-zero.
// Pieces stay resident until their last group has been CONSUMED (the values are read at consumption time), so
// nothing is copied between issue and consumption except the row-end mask, which travels in a register.
//
// Work item w = (tile w / nblocks, row block w % nblocks). Persistent CTAs take items from ONE counter, so the tiles
// run one after the other: while tile t is gathered only that tile of H (TF / f of it) competes for L2, which
// is what makes 64-float slices pay (a 256-byte slice of a row is twice as likely to still be in L2 as a 512-byte
// row). Each output element sums the same products in the same order whatever TF is: results are bit-identical.
// Double-buffered halo slab (a.epoch set): while the exchange epoch is odd, a.H_odd replaces the operand that holds the
// slab (H1 with HALO, else H0). The tensor-map variant passes the maps of the call's buffers in tm0 / tm1; modes 0 and 1
// read the parity with every work item (an L1 hit), because holding it for the whole CTA costs one of their instances a
// register.
template <int TF, int G, int NG, int MODE, bool HALO>
__device__ __forceinline__ void ring_body(const SpmmArgs& a, const RingArgs& ra, const CUtensorMap* tm0, const CUtensorMap* tm1)
{
    typedef typename RingLane<TF>::V V;
    constexpr int NV = RingLane<TF>::NV;
    constexpr int NS = G * NG, NP = kRingPieces;
    constexpr int PG = 32 / G;                                           // groups per index piece
    constexpr int U = (NG > PG) ? NG / PG : 1;                           // pieces per loop body (body groups % NG == 0)
    constexpr uint32_t RB = TF * 4;                                      // bytes of one row tile
    constexpr int RV = RB / sizeof(V);                                   // lane vectors per row slot
    constexpr uint32_t FULL = (G == 32) ? 0xffffffffu : ((1u << G) - 1u);
    static_assert((G == 8 || G == 16 || G == 32) && (NG == 2 || NG == 4), "unsupported ring shape");
    static_assert((U * PG) % NG == 0, "slot groups must repeat with the loop body");
    static_assert(NP * 32 >= NS + 64, "pieces must stay resident from prefetch to consumption");
    static_assert(MODE != 1 || TF >= 128, "the cp.async fill copies 16 bytes per lane");
    extern __shared__ __align__(128) unsigned char ring_smem[];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* wbase = ring_smem + (size_t)warp * ring_warp_bytes(TF, NS, NG);
    // MODE 2 issues each row copy once per warp from uniform registers (tma_row_warp)
    const uint32_t s_data = MODE == 2 ? warp_uniform(smem_u32(wbase)) : smem_u32(wbase);   // NS slots of RB bytes
    const uint32_t s_idx = s_data + NS * RB;                             // NP pieces
    const uint32_t s_gbar = s_idx + NP * kPieceBytes;                    // NG group barriers
    const uint32_t s_pbar = s_gbar + NG * 8;                             // NP piece barriers
    const int* idx_gen = reinterpret_cast<const int*>(wbase + (size_t)NS * RB);
    const V* data_gen = reinterpret_cast<const V*>(wbase) + lane;

    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < NG + NP; ++i) mbar_init(s_gbar + i * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncwarp();

    const unsigned long long pol_hot = MODE == 2 ? warp_uniform64(l2_policy_evict_last()) : l2_policy_evict_last();
    const unsigned long long pol_cold = MODE == 2 ? warp_uniform64(l2_policy_evict_first()) : l2_policy_evict_first();
    // row pitch f * 4; tile t covers floats [t TF, t TF + TF)
    const size_t pitch = (size_t)a.f * 4;
    const unsigned usplit = HALO ? (unsigned)a.split : 0xffffffffu;
    unsigned int* counter = ra.counter;
    const int nitems = a.nblocks * (a.f / TF);

    uint32_t gpar = 0;                   // phase parity of each group barrier (bit sg)
    // pieces move through the NP slots as a FIFO: fetched -> landed (issue side) -> consumed
    uint32_t pfetch = 0, pwait = 0, pcons = 0;

    V acc[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = vzero((V*)nullptr);

    // without a counter: one item per warp, tile blockIdx.y
    int w = (int)(blockIdx.x * ring_cta_warps(TF, NS, NG) + warp);
    w = w < a.nblocks ? (int)blockIdx.y * a.nblocks + w : nitems;
    if (counter) {
        if (lane == 0) w = (int)atomicAdd(counter, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
    }
    if (MODE == 2) w = (int)warp_uniform((uint32_t)w);

    while (w < nitems) {
        const int tile = w / a.nblocks, blk = w - tile * a.nblocks;
        const size_t toff = (size_t)tile * RB;
        const int tx = MODE == 2 ? (int)warp_uniform((uint32_t)(tile * TF)) : 0;   // the tile's first column in H
        const bool odd = MODE != 2 && epoch_odd(a.epoch);
        const char* hb0 = reinterpret_cast<const char*>((!HALO && odd) ? a.H_odd : a.H0) + toff;
        const char* hb1 = HALO ? reinterpret_cast<const char*>(odd ? a.H_odd : a.H1) + toff - (size_t)a.split * pitch : hb0;
        int4 b = __ldg(a.blocks + blk);
        if (MODE == 2) {
            // uniform block bounds make every loop and branch around the warp-level copies warp-uniform, so ptxas keeps
            // their operands in uniform registers (else it moves them back, and wraps each copy in an ELECT loop)
            b = make_int4((int)warp_uniform((uint32_t)b.x), (int)warp_uniform((uint32_t)b.y),
                          (int)warp_uniform((uint32_t)b.z), (int)warp_uniform((uint32_t)b.w));
        }
        const bool seg = b.y < 0;
        const int e0 = b.z, e1 = b.w;
        int row = b.x;
        const int gA = e0 / G, gB = (e1 - 1) / G;                        // first / last (aligned) group
        const int P0 = e0 >> 5, P1 = (e1 - 1) >> 5;                      // first / last piece
        uint32_t vmask[NG], emask[NG];                                   // per slot group: valid edges, row ends
#pragma unroll
        for (int i = 0; i < NG; ++i) vmask[i] = emask[i] = 0;
        int pnext = P0;                                                  // next piece to fetch
        const int* pi = idx_gen;                                         // piece being issued from
        const int* pc = idx_gen + (pcons % NP) * kPieceInts;             // piece being consumed from

        auto fetch_piece = [&]() {
            if (pnext <= P1) {
                if (lane == 0) {
                    const uint32_t q = pfetch % NP;
                    mbar_expect_tx(s_pbar + q * 8, kPieceBytes);
                    bulk_g2s(s_idx + q * kPieceBytes, a.pieces + (size_t)pnext * kPieceInts, kPieceBytes, s_pbar + q * 8, pol_cold);
                }
                ++pfetch;
                ++pnext;
            }
        };
        auto wait_piece = [&]() {                                        // the next piece in FIFO order has landed
            const uint32_t q = pwait % NP;
            mbar_wait(s_pbar + q * 8, (pwait / NP) & 1);
            pi = idx_gen + q * kPieceInts;
            ++pwait;
        };
        auto piece_consumed = [&]() {                                    // the consumer leaves its piece: slot is free
            ++pcons;
            pc = idx_gen + (pcons % NP) * kPieceInts;
            fetch_piece();
        };
        auto flush_row = [&]() {
            ring_store_row<V, NV>(acc[0], acc[NV - 1], a.rowids, row, a.Z0, a.Z1, a.zsplit, pitch, toff + lane * sizeof(V), a.beta,
                                  a.relu, a.final);
#pragma unroll
            for (int v = 0; v < NV; ++v) acc[v] = vzero((V*)nullptr);
            ++row;
        };
        // issue the group at sub-position qs of piece `pi` into slot group sg; vm = valid entries (FULL inside the block:
        // `whole`, a compile-time constant at every call)
        auto issue = [&](int qs, int sg, uint32_t vm, bool whole) {
            // {row-end mask, cold mask} of the piece; 64-float slices use the cold mask of their own (larger) hot set
            uint2 m;
            if (TF == 64) { const uint4 q = *reinterpret_cast<const uint4*>(pi + 64); m = make_uint2(q.x, q.z); }
            else m = *reinterpret_cast<const uint2*>(pi + 64);
            const uint32_t em = seg ? 0u : ((m.x >> (qs * G)) & vm);
            const uint32_t cm = (m.y >> (qs * G)) & FULL;
            reg_set(emask, sg, em);
            reg_set(vmask, sg, vm);
            const int* cols = pi + qs * G;
            if (MODE == 1) {
#pragma unroll
                for (int j = 0; j < G; ++j) {
                    if (vm >> j & 1) {
                        const unsigned cj = (unsigned)cols[j];
                        const char* src = (cj >= usplit ? hb1 : hb0) + (size_t)cj * pitch + lane * 16;
#pragma unroll
                        for (int v = 0; v < NV; ++v)
                            cp_async16(s_data + (sg * G + j) * RB + v * 512 + lane * 16, src + v * 512,
                                       (cm >> j & 1) ? pol_cold : pol_hot);
                    }
                }
                cp_async_commit();
                return;
            }
            if (kDiagNoCopy && MODE == 2) return;
            if (lane == 0) mbar_expect_tx(s_gbar + sg * 8, (uint32_t)__popc(vm) * RB);
            if (MODE == 2) {
                // the whole warp walks the group's columns 4 at a time (broadcast LDS.128); one elected lane copies
                const uint32_t vu = whole ? FULL : warp_uniform(vm), cu = warp_uniform(cm);
                const uint32_t dst = s_data + sg * G * RB, bar = s_gbar + sg * 8;
#pragma unroll 1
                for (int j = 0; j < G; j += 4) {
                    const int4 c4 = *reinterpret_cast<const int4*>(cols + j);
                    const int cc[4] = {c4.x, c4.y, c4.z, c4.w};
                    const uint32_t vj = vu >> j, cmj = cu >> j;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (whole || (vj >> k & 1)) {
                            const unsigned cj = warp_uniform((unsigned)cc[k]);
                            const bool halo = HALO && cj >= usplit;
                            tma_row_warp(dst + (j + k) * RB, halo ? tm1 : tm0, tx, (int)(halo ? cj - usplit : cj), bar,
                                         (cmj >> k & 1) ? pol_cold : pol_hot);
                        }
                    }
                }
                return;
            }
            if (lane < G && (vm >> lane & 1)) {
                const unsigned cj = (unsigned)cols[lane];
                const bool halo = cj >= usplit;
                const unsigned long long pol = (cm >> lane & 1) ? pol_cold : pol_hot;
                bulk_g2s(s_data + (sg * G + lane) * RB, (halo ? hb1 : hb0) + (size_t)cj * pitch, RB, s_gbar + sg * 8, pol);
            }
        };
        // consume slot group sg = the group at sub-position qs of piece `pc`
        auto consume = [&](int qs, int sg, bool interior) {
            const uint32_t vm = interior ? FULL : reg_get(vmask, sg);
            if (vm == 0) {                                               // group outside the block: nothing was issued
                if (MODE == 1) cp_async_wait<NG - 1>();
                return;
            }
            if (MODE == 1) cp_async_wait<NG - 1>();
            else if (!(kDiagNoCopy && MODE == 2)) { mbar_wait(s_gbar + sg * 8, (gpar >> sg) & 1); gpar ^= 1u << sg; }
            const uint32_t em = reg_get(emask, sg);
            const V* slot = data_gen + (size_t)(sg * G) * RV;
            const float* wv = reinterpret_cast<const float*>(pc) + 32 + qs * G;
            if (vm == FULL) {
#pragma unroll
                for (int c = 0; c < G; c += 8) {                         // 8 rows at a time: 8 x LDS.64 / LDS.128 in flight
                    const float4 wa = *reinterpret_cast<const float4*>(wv + c);
                    const float4 wb = *reinterpret_cast<const float4*>(wv + c + 4);
                    const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
                    V r[8][NV];
#pragma unroll
                    for (int j = 0; j < 8; ++j)
#pragma unroll
                        for (int v = 0; v < NV; ++v) r[j][v] = slot[(c + j) * RV + v * 32];
                    if (((em >> c) & 0xffu) == 0) {                      // no row end inside: 8 x (LDS, TF / 32 FFMA)
#pragma unroll
                        for (int j = 0; j < 8; ++j)
#pragma unroll
                            for (int v = 0; v < NV; ++v) if (!kDiagNoFma) vfma(acc[v], w[j], r[j][v]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
#pragma unroll
                            for (int v = 0; v < NV; ++v) if (!kDiagNoFma) vfma(acc[v], w[j], r[j][v]);
                            if (em >> (c + j) & 1) flush_row();
                        }
                    }
                }
            } else {                                                     // first / last group of a block
#pragma unroll 1
                for (int j = 0; j < G; ++j) {
                    if (vm >> j & 1) {
                        const float wj = wv[j];
#pragma unroll
                        for (int v = 0; v < NV; ++v) if (!kDiagNoFma) vfma(acc[v], wj, slot[j * RV + v * 32]);
                        if (em >> j & 1) flush_row();
                    }
                }
            }
            __syncwarp();                                                // every lane is done with these slots
        };
        // valid-entry mask of aligned group gi with respect to the block [e0, e1)
        auto group_mask = [&](int gi) -> uint32_t {
            if (gi < gA || gi > gB) return 0u;
            uint32_t vm = FULL;
            if (gi == gA) vm &= FULL << (e0 - gA * G);
            if (gi == gB) vm &= FULL >> (G - 1 - ((e1 - 1) - gB * G));
            return vm;
        };
        auto issue_checked = [&](int gi, int qs, int sg) {
            const uint32_t vm = group_mask(gi);
            if (vm == 0) { reg_set(vmask, sg, 0u); if (MODE == 1) cp_async_commit(); return; }
            issue(qs, sg, vm, false);
        };

        // prologue: index pieces in flight, first piece landed, the first NG groups issued
#pragma unroll
        for (int i = 0; i < NP; ++i) fetch_piece();
        wait_piece();
#pragma unroll 1
        for (int i = 0; i < NG; ++i) {
            if (i > 0 && i % PG == 0 && P0 + i / PG <= P1) wait_piece();     // the ring spans more than one piece
            if (P0 + i / PG <= P1) issue_checked(PG * P0 + i, i % PG, i);
            else { reg_set(vmask, i, 0u); if (MODE == 1) cp_async_commit(); }
        }

        // The loops below are deliberately NOT unrolled over the groups of a piece: slot group and sub-group are
        // runtime values (a handful of integer instructions per group), which keeps the whole kernel inside the
        // instruction cache; the 8-row consume chunks inside a group are unrolled.
        for (int P = P0; P <= P1; P += U) {
            // interior: every group consumed AND every group issued by this body lies strictly inside the block
            const bool interior = PG * P > gA && PG * (P + U) - 1 + NG < gB;
#pragma unroll 1
            for (int idx = 0; idx < U * PG; ++idx) {
                const int sg = idx % NG;
                const int qc = idx % PG;                                 // sub-position of the consumed group
                consume(qc, sg, interior);
                if (qc == PG - 1) piece_consumed();
                const int qi = (idx + NG) % PG;                          // sub-position of the group NG ahead
                const int Pi = P + (idx + NG) / PG;                      // its piece
                if (interior) {
                    if (qi == 0) wait_piece();
                    issue(qi, sg, FULL, true);
                } else {
                    if (qi == 0 && Pi <= P1) wait_piece();               // first group of a new piece
                    if (Pi <= P1) issue_checked(PG * Pi + qi, qi, sg);
                    else { reg_set(vmask, sg, 0u); if (MODE == 1) cp_async_commit(); }
                }
            }
        }
        // pieces P1+1 .. (rounded up to the body) were never fetched, but the body counted them as consumed
        pcons = pwait;

        if (seg) {
            char* pb = reinterpret_cast<char*>(a.partial) + (size_t)(unsigned)(-b.y - 1) * pitch + toff;
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                reinterpret_cast<V*>(pb + v * 512)[lane] = acc[v];
                acc[v] = vzero((V*)nullptr);
            }
        }

        if (!counter) break;
        if (lane == 0) w = (int)atomicAdd(counter, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
        if (MODE == 2) w = (int)warp_uniform((uint32_t)w);
    }
    if (MODE == 1) cp_async_wait<0>();
}

template <int TF, int G, int NG, int MODE, bool HALO>
__global__ void __launch_bounds__(ring_cta_warps(TF, G * NG, NG) * 32)
spmm_ring_kernel(const SpmmArgs a, const RingArgs ra)
{
    ring_body<TF, G, NG, MODE, HALO>(a, ra, nullptr, nullptr);
}

// tensor-map variant: the tensor maps of H_own (tm0) and of the halo slab (tm1) travel as __grid_constant__ parameters;
// tm_odd maps the halo slab of odd exchange epochs (it replaces tm1 with HALO, else tm0; unused when a.epoch is null)
template <int TF, int G, int NG, bool HALO>
__global__ void __launch_bounds__(ring_cta_warps(TF, G * NG, NG) * 32)
spmm_ring_tm_kernel(const SpmmArgs a, const RingArgs ra, const __grid_constant__ CUtensorMap tm0,
                    const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm_odd)
{
    // the map pointers feed the warp-level copies: uniform values, computed once
    const bool odd = epoch_odd(a.epoch);
    const CUtensorMap* m0 = reinterpret_cast<const CUtensorMap*>(warp_uniform64((unsigned long long)((!HALO && odd) ? &tm_odd : &tm0)));
    const CUtensorMap* m1 = reinterpret_cast<const CUtensorMap*>(warp_uniform64((unsigned long long)((HALO && odd) ? &tm_odd : &tm1)));
    ring_body<TF, G, NG, 2, HALO>(a, ra, m0, m1);
}

}  // namespace pgcn
