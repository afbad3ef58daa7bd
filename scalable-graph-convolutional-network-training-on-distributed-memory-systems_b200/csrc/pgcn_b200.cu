// pgcn_b200.cu — C-ABI implementation (see include/pgcn_b200.h for the contract and the
// reference file:line each entry point replaces).
//
// Host side of the hot path: plan construction (device CSR copies, row-block schedule, boundary
// CSR for the gradient scatter-add), kernel dispatch, and the two transports of the halo
// exchange (NCCL grouped send/recv resolved at run time from the process's libnccl, and the
// peer-memory path that stores rows directly into the neighbour GPU's slab over NVLink).
#include "../../include/pgcn_b200.h"
#include "../../include/pgcn_b200_halo.h"
#include "spmm_kernels.cuh"
#include "spmm_ring.cuh"
#include "sddmm.cuh"
#include "attention.cuh"
#include "spmm_max.cuh"
#include "gatv2.cuh"

#include <dlfcn.h>
#include <unistd.h>
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

using namespace pgcn;

// ------------------------------------------------------------------------------------------
// NCCL, resolved lazily from whatever libnccl the process already has (torch's bundled copy),
// so this library has no link-time NCCL dependency and loads on a box without it.
// ------------------------------------------------------------------------------------------
namespace {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess_ = 0, ncclFloat_ = 7 };

struct NcclApi {
    bool tried = false, ok = false;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;

bool load_nccl()
{
    if (g_nccl.tried) return g_nccl.ok;
    g_nccl.tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);  // torch's copy, if loaded
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return false;
#define PGCN_SYM(field, name)                                              \
    *(void**)(&g_nccl.field) = dlsym(h, name);                             \
    if (!g_nccl.field) return false;
    PGCN_SYM(GetUniqueId, "ncclGetUniqueId")
    PGCN_SYM(CommInitRank, "ncclCommInitRank")
    PGCN_SYM(CommDestroy, "ncclCommDestroy")
    PGCN_SYM(Send, "ncclSend")
    PGCN_SYM(Recv, "ncclRecv")
    PGCN_SYM(GroupStart, "ncclGroupStart")
    PGCN_SYM(GroupEnd, "ncclGroupEnd")
    PGCN_SYM(GetErrorString, "ncclGetErrorString")
#undef PGCN_SYM
    g_nccl.ok = true;
    return true;
}

std::string g_lib_error = "";

constexpr int kMaxPeers = 16;

struct DevCsr {
    int nrows = 0;                  // rows of the matrix (output rows)
    int nrows_c = 0;                // non-empty rows = rows the schedule walks
    int64_t nnz = 0;
    std::vector<int> h_rowptr;      // COMPACT row pointers (empty rows squeezed out), for scheduling
    int* d_cw = nullptr;            // entries in 272-byte pieces of 32: col[32] | val[32] | row-end mask | cold mask |
                                    // cold mask of 64-float slices | pad
    int* d_rowids = nullptr;        // compact row -> output row, null when the identity
    int* d_empty = nullptr;         // output rows without entries (zero-filled when beta == 0)
    int nempty = 0;
    bool view = false;              // a row range of another matrix: d_cw / d_rowids / d_empty are borrowed
    int row_base = 0;               // compact id of the first walked row (views: offset into the parent's numbering)
    std::vector<int> h_rowids, h_empty;   // host copies (parents of views only)
    unsigned char* d_final = nullptr;     // per walked row: this matrix is the LAST launch of the forward that writes it
    int* d_vmap = nullptr;          // pgcn_plan_bind_values: entry -> forward entry (null for the forward matrix itself)
    int64_t tuned_epb[2] = {0, 0};  // per-matrix autotune results (0: use the plan option): [0] register, [1] ring
    int tuned_slots = 0;
    int tuned_tile = 0;             // ring row tile in floats (0: the full width 128 or 256)
    // schedules: [0] register-pipeline kernel (small row blocks, one per lane group),
    //            [1] shared-memory ring kernel (large row blocks, one per warp)
    struct Sched {
        int4* d_blocks = nullptr;
        int nblocks = 0;
        int4* d_long = nullptr;
        int nlong = 0;
        int nslots = 0;
        float* d_partial = nullptr;
        int* d_apart = nullptr;     // entries of the max aggregation's split-row partials (forward register schedule,
                                    // bound plans only: allocated by the first max call or pgcn_plan_prepare)
        float* d_datt = nullptr;    // GATv2 datt partials, f_max floats per chunk of kGatv2Chunk row blocks (forward
                                    // register schedule, bound plans only: first GATv2 backward or pgcn_plan_prepare)
        int64_t epb = -1, long_row = -1;
    } sched[2];
};

struct P2PBlob {                     // what pgcn_p2p_export writes (PGCN_P2P_HANDLE_BYTES)
    cudaIpcMemHandle_t ipc;          // 64 bytes
    int64_t arena_bytes;
    int64_t off_flags, off_fwd[2], off_bwd[2];
    int32_t k, rank, f_max, pad;
    int64_t pid;                     // exporting process: a peer in the same process is reached through local_ptr
    void* local_ptr;
    int64_t send_off[kMaxPeers + 1];
    int64_t recv_off[kMaxPeers + 1];
};
static_assert(sizeof(P2PBlob) <= PGCN_P2P_HANDLE_BYTES, "blob too large");

}  // namespace

struct pgcn_plan {
    int device = 0;
    int m = 0, h = 0, k = 1, rank = 0, f_max = 0;
    int64_t S = 0;
    DevCsr fwd, tr;                  // A_local over [own | halo] columns, and its transpose
    // split A_local = [A_own | A_halo(peer 0) | ... ] (Parallel-GCN/main.c:271 then :295 per received block):
    DevCsr own;                      // columns < m
    std::vector<DevCsr> halo_q;      // per source peer: boundary rows x that peer's columns (slab-relative)
    DevCsr tr_own;                   // view: rows [0, m) of tr
    std::vector<DevCsr> tr_halo_q;   // views: rows of tr that belong to each peer
    bool have_split = false;
    int64_t cols_ref = 0, rows_ref_t = 0;

    std::vector<int64_t> send_off, recv_off;
    int* d_send_idx = nullptr;
    // boundary CSR for unpack_add
    int* d_brow = nullptr; int* d_bptr = nullptr; int* d_bpos = nullptr; int nb = 0;

    // slabs (local transport)
    float* d_send_slab = nullptr;    // S x f_max
    float* d_halo_slab = nullptr;    // h x f_max   (forward receive)
    float* d_rrecv_slab = nullptr;   // S x f_max   (reverse receive)
    float* d_hsend_slab = nullptr;   // h x f_max   (reverse send: halo partials of A^T g)

    // options
    int64_t opt_epb = 128, opt_long = 0, opt_tile = 0, opt_overlap = 1, opt_hot_mb = 24;
    int64_t opt_relu = 0;            // fused layer epilogue of pgcn_forward: Z = max(0, A_local * H)
    // kernel: 0 auto (ring with TMA bulk copies where it applies), 4 register pipeline, 5 ring/1-D TMA,
    //         6 ring/cp.async, 7 ring/2-D tensor-map TMA (= auto)
    int64_t opt_ring_groups = 2;
    int64_t opt_persistent_multi = 0;
    int64_t opt_kernel = 0, opt_ring_slots = 16, opt_ring_epb = 512, opt_ring_long = 0, opt_persistent = 1;
    int64_t opt_ring_tile = 0;       // ring row tile in floats: 0 = tuned (else full width), 64 | 128 | 256
    std::unordered_map<const void*, int> ctas_per_sm;   // kernels opted in to their dynamic shared memory: CTAs per SM
    unsigned int* d_counter = nullptr;     // work-item counter of the persistent ring kernel
    int num_sms = 132;

    // NCCL
    ncclComm_t comm = nullptr;
    bool comm_borrowed = false;            // pgcn_comm_share: the communicator belongs to another plan
    cudaStream_t comm_stream = nullptr;
    cudaStream_t host_stream = nullptr;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    std::vector<cudaEvent_t> ev_step;      // one per peer step of the pipelined exchange
    unsigned int* d_done = nullptr;        // per-destination CTA counters of put_rows_kernel

    // peer-memory transport
    bool p2p = false;
    int64_t opt_p2p = 1;                   // 0: never use the peer transport (all ranks must agree)
    void* arena = nullptr; int64_t arena_bytes = 0;
    int64_t off_flags = 0, off_fwd[2] = {0, 0}, off_bwd[2] = {0, 0};
    void* peer_arena[kMaxPeers] = {nullptr};
    bool peer_local[kMaxPeers] = {false};   // peer lives in THIS process (same-process plans: no IPC mapping)
    P2PBlob peer_blob[kMaxPeers];
    // exchange epoch of the peer transport, in device memory: advanced on the caller's stream by every fused multi-rank
    // call over peer memory, read there by the kernels (flag value, parity of the double-buffered slabs), so a CUDA
    // graph replay uses the epoch of the replay
    unsigned long long* d_epoch = nullptr;

    // pgcn_plan_prepare has run: schedules replaced from then on are retired instead of freed (a captured graph may
    // still read them) and released by pgcn_plan_destroy
    bool prepared = false;
    std::vector<void*> retired;
    int64_t nretired = 0;

    // pgcn_plan_bind_values: the record sets whose value words pgcn_plan_set_values rewrites, and the creation values
    bool bound = false;
    float* d_vals0 = nullptr;              // nnz, forward CSR order
    ValueSet* d_vsets = nullptr;
    int nvsets = 0;
    long long vtotal = 0;                  // entries over all sets
    int* d_rowptr = nullptr;               // m + 1, the forward rowptr (edge softmax)
    int* d_long_rows = nullptr;            // rows of more than kAttnLongRow entries (one CTA each in the edge softmax)
    int nlong_rows = 0;

    // host-buffer variant: two device slots, copy-in / compute / copy-out streams chained by events
    float* d_hostH[2] = {nullptr, nullptr}; float* d_hostZ[2] = {nullptr, nullptr}; int64_t host_cap = 0;
    cudaStream_t s_in = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
    int64_t host_steps = 0;

    int64_t launches = 0;
    std::string err;
};

namespace {

int fail(pgcn_plan* p, int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (p) p->err = buf; else g_lib_error = buf;
    return code;
}

#define CU(p, expr)                                                                         \
    do {                                                                                    \
        cudaError_t e__ = (expr);                                                           \
        if (e__ != cudaSuccess)                                                             \
            return fail(p, PGCN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                   \
                        cudaGetErrorString(e__), __FILE__, __LINE__);                       \
    } while (0)

#define NC(p, expr)                                                                         \
    do {                                                                                    \
        int e__ = (expr);                                                                   \
        if (e__ != ncclSuccess_)                                                            \
            return fail(p, PGCN_ERR_NCCL, "%s failed: %s", #expr, g_nccl.GetErrorString(e__)); \
    } while (0)

template <class T>
int upload(pgcn_plan* p, T** dst, const T* src, size_t n)
{
    *dst = nullptr;
    CU(p, cudaMalloc((void**)dst, std::max<size_t>(n, 1) * sizeof(T)));
    if (n) CU(p, cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

// Upload one CSR. Rows without entries are squeezed out of the walked row space (their outputs are
// zero-filled by a separate launch); `ext_rowmap` maps the rows of an already-compact matrix (the
// halo-column part, which only holds boundary rows) to output rows.
// `col_refs[j]` = number of stored entries in column j and `cold[0]` the reference count at or
// below which a column is COLD for full-width rows, `cold[1]` the same for 64-float slices (-1: no marking):
// cold columns are gathered with an L2 evict_first policy, the most-referenced rows of H (as many as fit the hot
// budget) evict_last.
int csr_upload(pgcn_plan* p, DevCsr& c, int nrows, const int* rowptr, const int* colidx, const float* vals,
               const std::vector<int>* ext_rowmap = nullptr, const int* col_refs = nullptr, const int* cold = nullptr,
               bool keep_host = false)
{
    c.nrows = nrows;
    c.nnz = rowptr[nrows];
    const size_t npieces = (size_t)((c.nnz + 31) / 32 + 1);
    std::vector<int> cw(npieces * kPieceInts, 0);
    for (int64_t e = 0; e < c.nnz; ++e) {
        int* pc = cw.data() + (size_t)(e >> 5) * kPieceInts;
        const int i = (int)(e & 31);
        pc[i] = colidx[e];
        memcpy(&pc[32 + i], &vals[e], 4);
        for (int w = 0; w < 2; ++w)
            if (col_refs && cold && cold[w] >= 0 && col_refs[colidx[e]] <= cold[w]) pc[65 + w] |= (int)(1u << i);
    }
    std::vector<int> rowids, empty;
    c.h_rowptr.clear();
    c.h_rowptr.push_back(0);
    for (int r = 0; r < nrows; ++r) {
        if (rowptr[r + 1] > rowptr[r]) {
            { const int64_t e = (int64_t)rowptr[r + 1] - 1; cw[(size_t)(e >> 5) * kPieceInts + 64] |= (int)(1u << (e & 31)); }
            c.h_rowptr.push_back(rowptr[r + 1]);
            rowids.push_back(ext_rowmap ? (*ext_rowmap)[r] : r);
        } else if (!ext_rowmap) {
            empty.push_back(r);
        }
    }
    c.nrows_c = (int)rowids.size();
    c.nempty = (int)empty.size();
    int rc;
    if ((rc = upload(p, &c.d_cw, cw.data(), cw.size()))) return rc;
    if (ext_rowmap || c.nempty > 0) {
        if ((rc = upload(p, &c.d_rowids, rowids.data(), rowids.size()))) return rc;
    }
    if (c.nempty > 0) {
        if ((rc = upload(p, &c.d_empty, empty.data(), empty.size()))) return rc;
    }
    if (keep_host) { c.h_rowids.swap(rowids); c.h_empty.swap(empty); }
    return 0;
}

// Rows [r0, r1) of an uploaded matrix as a matrix of its own (no copy): the transposed CSR's own rows and the
// rows that belong to one peer are contiguous row ranges, so the pipelined backward needs no second copy of A^T.
void csr_view(const DevCsr& base, DevCsr& v, int r0, int r1)
{
    v = DevCsr();
    v.view = true;
    int c0 = r0, c1 = r1, e0 = 0, e1 = 0;
    if (base.d_rowids) {                     // rows were squeezed: compact ids of the range
        c0 = (int)(std::lower_bound(base.h_rowids.begin(), base.h_rowids.end(), r0) - base.h_rowids.begin());
        c1 = (int)(std::lower_bound(base.h_rowids.begin(), base.h_rowids.end(), r1) - base.h_rowids.begin());
        e0 = (int)(std::lower_bound(base.h_empty.begin(), base.h_empty.end(), r0) - base.h_empty.begin());
        e1 = (int)(std::lower_bound(base.h_empty.begin(), base.h_empty.end(), r1) - base.h_empty.begin());
    }
    v.nrows = r1 - r0;
    v.nrows_c = c1 - c0;
    v.row_base = c0;
    v.h_rowptr.assign(base.h_rowptr.begin() + c0, base.h_rowptr.begin() + c1 + 1);   // absolute entry offsets
    v.nnz = (int64_t)v.h_rowptr.back() - v.h_rowptr.front();
    v.d_cw = base.d_cw;
    v.d_rowids = base.d_rowids;
    v.d_empty = base.d_empty ? base.d_empty + e0 : nullptr;
    v.nempty = e1 - e0;
}

void csr_free(DevCsr& c)
{
    if (!c.view) { cudaFree(c.d_cw); cudaFree(c.d_rowids); cudaFree(c.d_empty); cudaFree(c.d_vmap); }
    cudaFree(c.d_final);
    for (auto& sc : c.sched) { cudaFree(sc.d_blocks); cudaFree(sc.d_long); cudaFree(sc.d_partial); cudaFree(sc.d_apart); cudaFree(sc.d_datt); }
    c = DevCsr();
}

// The matrices the plan launches: forward and transposed records and, when split, the own-column part, each peer's
// halo block and the transposed row ranges of the pipelined backward
std::vector<DevCsr*> plan_matrices(pgcn_plan* p)
{
    std::vector<DevCsr*> mats = {&p->fwd, &p->tr};
    if (p->have_split) {
        mats.push_back(&p->own);
        mats.push_back(&p->tr_own);
        for (auto& c : p->halo_q) mats.push_back(&c);
        for (auto& c : p->tr_halo_q) mats.push_back(&c);
    }
    return mats;
}

// Cut the (compact) row range into row blocks of about `epb` nnz (at most kMaxRowsPerBlock rows); rows longer
// than `long_row` become ceil(deg/epb) single-row segments with a slot each in the side buffer.
constexpr int kMaxRowsPerBlock = 128;

// Pure host function (also reachable through pgcn_debug_schedule for CPU-side tests).
void make_schedule(const int* rp, int nrows_c, int64_t epb, int64_t long_row,
                   std::vector<int4>& blocks, std::vector<int4>& longs, int& nslots,
                   int max_rows = kMaxRowsPerBlock, int row_base = 0)
{
    blocks.clear(); longs.clear(); nslots = 0;
    const int64_t nnz = nrows_c > 0 ? rp[nrows_c] : 0;
    blocks.reserve((size_t)(nnz / epb + nrows_c / kMaxRowsPerBlock + 16));
    int cur_begin = 0;         // first row of the open block
    int64_t cur_edges = 0;
    auto close = [&](int row_end) {
        if (row_end > cur_begin)
            blocks.push_back(make_int4(row_base + cur_begin, row_end - cur_begin, rp[cur_begin], rp[row_end]));
        cur_begin = row_end;
        cur_edges = 0;
    };
    for (int r = 0; r < nrows_c; ++r) {
        const int64_t d = (int64_t)rp[r + 1] - rp[r];
        if (d > long_row) {
            close(r);
            const int nseg = (int)((d + epb - 1) / epb);
            longs.push_back(make_int4(row_base + r, nslots, nseg, 0));
            for (int s = 0; s < nseg; ++s) {
                const int e0 = rp[r] + (int)(s * epb);
                const int e1 = (int)std::min<int64_t>((int64_t)rp[r + 1], (int64_t)e0 + epb);
                blocks.push_back(make_int4(row_base + r, -(nslots + 1), e0, e1));
                ++nslots;
            }
            cur_begin = r + 1;
            continue;
        }
        if (cur_edges > 0 && cur_edges + d > epb) close(r);
        cur_edges += d;
        if (r + 1 - cur_begin >= max_rows) close(r + 1);
    }
    close(nrows_c);
}

// A stream under CUDA graph capture takes only stream-ordered work. Set-up that would allocate, copy synchronously or
// set a function attribute is refused before any such call, so the caller's capture stays valid.
int refuse_under_capture(pgcn_plan* p, cudaStream_t st)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(st, &cs);
    if (e == cudaSuccess && cs == cudaStreamCaptureStatusNone) return 0;
    if (e != cudaSuccess) cudaGetLastError();
    return fail(p, PGCN_ERR_STATE, "this call needs set-up work (schedule upload or kernel attributes) that cannot run "
                "while the stream is being captured into a CUDA graph: call pgcn_plan_prepare(plan, f) before capturing");
}

// Matrix c's schedule for the ring (or register) kernel, with the block size and long-row threshold of the current
// options or the autotune. It is built on first use, which is refused while `st` is being captured.
int schedule(pgcn_plan* p, DevCsr& c, bool ring, cudaStream_t st, DevCsr::Sched** out)
{
    DevCsr::Sched& sc = c.sched[ring ? 1 : 0];
    *out = &sc;
    int64_t epb, long_row;
    if (ring) {
        epb = std::max<int64_t>(c.tuned_epb[1] > 0 ? c.tuned_epb[1] : p->opt_ring_epb, 64);
        long_row = p->opt_ring_long > 0 ? p->opt_ring_long : 2 * epb;
    } else {
        epb = std::max<int64_t>(c.tuned_epb[0] > 0 ? c.tuned_epb[0] : p->opt_epb, 8);
        long_row = p->opt_long > 0 ? p->opt_long : 4 * epb;
    }
    if (sc.epb == epb && sc.long_row == long_row) return 0;
    int rc = refuse_under_capture(p, st);
    if (rc) return rc;

    std::vector<int4> blocks, longs;
    int nslots = 0;
    make_schedule(c.h_rowptr.data(), c.nrows_c, epb, long_row, blocks, longs, nslots,
                  ring ? (1 << 30) : kMaxRowsPerBlock, c.row_base);

    if (p->prepared && sc.epb >= 0) {
        // a graph captured after pgcn_plan_prepare may still launch the old schedule: keep it until pgcn_plan_destroy
        p->retired.insert(p->retired.end(), {(void*)sc.d_blocks, (void*)sc.d_long, (void*)sc.d_partial, (void*)sc.d_apart,
                                             (void*)sc.d_datt});
        ++p->nretired;
    } else {
        cudaFree(sc.d_blocks); cudaFree(sc.d_long); cudaFree(sc.d_partial); cudaFree(sc.d_apart); cudaFree(sc.d_datt);
    }
    sc.d_blocks = nullptr; sc.d_long = nullptr; sc.d_partial = nullptr; sc.d_apart = nullptr; sc.d_datt = nullptr;
    if ((rc = upload(p, &sc.d_blocks, blocks.data(), blocks.size()))) return rc;
    if ((rc = upload(p, &sc.d_long, longs.data(), longs.size()))) return rc;
    CU(p, cudaMalloc((void**)&sc.d_partial, std::max<size_t>((size_t)nslots * p->f_max, 1) * sizeof(float)));
    sc.nblocks = (int)blocks.size();
    sc.nlong = (int)longs.size();
    sc.nslots = nslots;
    sc.epb = epb;
    sc.long_row = long_row;
    return 0;
}

// ---- kernel dispatch ---------------------------------------------------------------------

struct TileCfg { int lpe, vpl, vw, tiles; };

int pow2ceil(int x) { int p = 1; while (p < x) p <<= 1; return p; }

// vw: floats per vector access, 4 or 1 (vec_width). Each output element sums the same products in the same order
// at either width, so the width changes the launch shape but not a bit of the result.
TileCfg choose_tile(const pgcn_plan* p, int f, int vw)
{
    TileCfg t;
    t.vw = vw;
    const int nvec = f / t.vw;
    int tile_vecs = nvec;
    if (p->opt_tile > 0) tile_vecs = std::max<int>(1, (int)std::min<int64_t>(nvec, p->opt_tile / t.vw));
    tile_vecs = std::min(tile_vecs, 128);
    t.lpe = std::max(4, std::min(32, pow2ceil(tile_vecs)));
    int vpl = (tile_vecs + t.lpe - 1) / t.lpe;
    t.vpl = vpl <= 1 ? 1 : (vpl <= 2 ? 2 : 4);
    t.tiles = (nvec + t.lpe * t.vpl - 1) / (t.lpe * t.vpl);
    return t;
}

typedef void (*spmm_fn)(const SpmmArgs);

// choose_tile takes lpe = pow2ceil(tile_vecs) below 32 lanes, which covers the tile: only LPE = 32 has VPL 2 and 4
template <int LPE, int VW>
spmm_fn pick_vpl(int vpl, bool halo)
{
    if constexpr (LPE < 32) return halo ? spmm_rowblock_kernel<LPE, 1, VW, true> : spmm_rowblock_kernel<LPE, 1, VW, false>;
    else switch (vpl) {
        case 1: return halo ? spmm_rowblock_kernel<LPE, 1, VW, true> : spmm_rowblock_kernel<LPE, 1, VW, false>;
        case 2: return halo ? spmm_rowblock_kernel<LPE, 2, VW, true> : spmm_rowblock_kernel<LPE, 2, VW, false>;
        default: return halo ? spmm_rowblock_kernel<LPE, 4, VW, true> : spmm_rowblock_kernel<LPE, 4, VW, false>;
    }
}

template <int VW>
spmm_fn pick_lpe(int lpe, int vpl, bool halo)
{
    switch (lpe) {
        case 4: return pick_vpl<4, VW>(vpl, halo);
        case 8: return pick_vpl<8, VW>(vpl, halo);
        case 16: return pick_vpl<16, VW>(vpl, halo);
        default: return pick_vpl<32, VW>(vpl, halo);
    }
}

// Multi-head instances of the register kernel (spmm_heads_kernel): one vector per lane (the feature row is walked in
// blockIdx.y tiles of LPE vectors), NH heads staged per chunk.
typedef void (*spmm_heads_fn)(const SpmmArgs, const SpmmHeadArgs);

// 8 heads need f >= 8 floats, i.e. 8 or more lanes of one vector (choose_tile_heads): LPE = 4 has no 8-head instance
// (null: the launch fails with an error instead of running a wrong shape)
template <int LPE, int VW, bool HALO>
spmm_heads_fn pick_heads_nh(int nh)
{
    switch (nh) {
        case 1: return spmm_heads_kernel<LPE, VW, HALO, 1>;
        case 2: return spmm_heads_kernel<LPE, VW, HALO, 2>;
        case 4: return spmm_heads_kernel<LPE, VW, HALO, 4>;
        default:
            if constexpr (LPE > 4) return spmm_heads_kernel<LPE, VW, HALO, 8>;
            else return nullptr;
    }
}

template <int VW, bool HALO>
spmm_heads_fn pick_heads_lpe(int lpe, int nh)
{
    switch (lpe) {
        case 4: return pick_heads_nh<4, VW, HALO>(nh);
        case 8: return pick_heads_nh<8, VW, HALO>(nh);
        case 16: return pick_heads_nh<16, VW, HALO>(nh);
        default: return pick_heads_nh<32, VW, HALO>(nh);
    }
}

spmm_heads_fn pick_heads(int lpe, int vw, bool halo, int nh)
{
    if (vw == 4) return halo ? pick_heads_lpe<4, true>(lpe, nh) : pick_heads_lpe<4, false>(lpe, nh);
    return halo ? pick_heads_lpe<1, true>(lpe, nh) : pick_heads_lpe<1, false>(lpe, nh);
}

// Launch shape of the multi-head instances: one vector per lane, as many lanes as the row needs (4 .. 32), the rest
// of the row in blockIdx.y tiles.
TileCfg choose_tile_heads(int f, int vw)
{
    TileCfg t;
    t.vw = vw;
    const int nvec = f / vw;
    t.lpe = std::max(4, std::min(32, pow2ceil(nvec)));
    t.vpl = 1;
    t.tiles = (nvec + t.lpe - 1) / t.lpe;
    return t;
}

// Max aggregation instances (spmm_max.cuh): one vector per lane, the launch shape of the multi-head instances.
typedef void (*spmm_max_fn)(const SpmmArgs, int*, int*);
typedef void (*spmm_max_bwd_fn)(const SpmmArgs, const int*, const int*);

template <int VW, bool HALO>
spmm_max_fn pick_max_lpe(int lpe)
{
    switch (lpe) {
        case 4: return spmm_max_kernel<4, VW, HALO>;
        case 8: return spmm_max_kernel<8, VW, HALO>;
        case 16: return spmm_max_kernel<16, VW, HALO>;
        default: return spmm_max_kernel<32, VW, HALO>;
    }
}

spmm_max_fn pick_max(int lpe, int vw, bool halo)
{
    if (vw == 4) return halo ? pick_max_lpe<4, true>(lpe) : pick_max_lpe<4, false>(lpe);
    return halo ? pick_max_lpe<1, true>(lpe) : pick_max_lpe<1, false>(lpe);
}

template <int VW>
spmm_max_bwd_fn pick_max_bwd_lpe(int lpe)
{
    switch (lpe) {
        case 4: return spmm_max_backward_kernel<4, VW>;
        case 8: return spmm_max_backward_kernel<8, VW>;
        case 16: return spmm_max_backward_kernel<16, VW>;
        default: return spmm_max_backward_kernel<32, VW>;
    }
}

spmm_max_bwd_fn pick_max_bwd(int lpe, int vw) { return vw == 4 ? pick_max_bwd_lpe<4>(lpe) : pick_max_bwd_lpe<1>(lpe); }

typedef void (*ring_fn)(const SpmmArgs, const RingArgs);
typedef void (*ring_tm_fn)(const SpmmArgs, const RingArgs, const CUtensorMap, const CUtensorMap, const CUtensorMap);

// cuTensorMapEncodeTiled, resolved through the runtime (no link-time dependency on libcuda)
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
encode_tiled_fn g_encode_tiled = nullptr;
bool g_encode_tried = false;

encode_tiled_fn encode_tiled()
{
    if (!g_encode_tried) {
        g_encode_tried = true;
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            g_encode_tiled = reinterpret_cast<encode_tiled_fn>(fn);
        else
            cudaGetLastError();
    }
    return g_encode_tiled;
}

// Tensor map of a row-major fp32 matrix [rows, f] for tile loads of `tile` floats of `box_rows` rows.
bool make_row_map(CUtensorMap* tm, const float* base, int64_t rows, int f, int tile, int box_rows)
{
    encode_tiled_fn enc = encode_tiled();
    if (!enc || !base) return false;
    const cuuint64_t gdim[2] = {(cuuint64_t)f, (cuuint64_t)std::max<int64_t>(rows, 1)};
    const cuuint64_t gstride[1] = {(cuuint64_t)f * 4};
    const cuuint32_t box[2] = {(cuuint32_t)tile, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Ring kernel instances: shape id = 0: G=8,NG=2 (16 slots)  1: G=16,NG=2 (32)  2: G=32,NG=2 (64)  3: G=16,NG=4 (64)
struct RingShape { int g, ng; };
const RingShape kRingShapes[4] = {{8, 2}, {16, 2}, {32, 2}, {16, 4}};

// Row tiles: tf = 64 (256-byte slices), 128 or 256 floats. The cp.async fill (mode 1) needs tf >= 128.
template <int TF, bool HALO>
ring_fn pick_ring_t(int shape, int mode)
{
    if constexpr (TF >= 128) {
        if (mode == 1) return spmm_ring_kernel<TF, 8, 2, 1, HALO>;
    }
    return shape == 1 ? spmm_ring_kernel<TF, 16, 2, 0, HALO> : spmm_ring_kernel<TF, 8, 2, 0, HALO>;
}
ring_fn pick_ring(int tf, int shape, int mode, bool halo)
{
    if (tf == 256) return halo ? pick_ring_t<256, true>(shape, mode) : pick_ring_t<256, false>(shape, mode);
    if (tf == 64) return halo ? pick_ring_t<64, true>(shape, mode) : pick_ring_t<64, false>(shape, mode);
    return halo ? pick_ring_t<128, true>(shape, mode) : pick_ring_t<128, false>(shape, mode);
}
template <int TF, bool HALO>
ring_tm_fn pick_ring_tm_t(int shape)
{
    switch (shape) {
        case 1: return spmm_ring_tm_kernel<TF, 16, 2, HALO>;
        case 2: return spmm_ring_tm_kernel<TF, 32, 2, HALO>;
        case 3: return spmm_ring_tm_kernel<TF, 16, 4, HALO>;
        default: return spmm_ring_tm_kernel<TF, 8, 2, HALO>;
    }
}
ring_tm_fn pick_ring_tm(int tf, int shape, bool halo)
{
    if (tf == 256) return halo ? pick_ring_tm_t<256, true>(shape) : pick_ring_tm_t<256, false>(shape);
    if (tf == 64) return halo ? pick_ring_tm_t<64, true>(shape) : pick_ring_tm_t<64, false>(shape);
    return halo ? pick_ring_tm_t<128, true>(shape) : pick_ring_tm_t<128, false>(shape);
}

// A ring instance of row tile tf, shape and fill mode (2: tensor map, 0: 1-D bulk copies, 1: cp.async): its kernel,
// dynamic shared memory and warps per CTA
struct RingInst { const void* fn; size_t smem; int warps; };

RingInst ring_inst(int tf, int shape, int mode, bool halo)
{
    const int g = kRingShapes[shape].g, ng = kRingShapes[shape].ng;
    return {mode == 2 ? (const void*)pick_ring_tm(tf, shape, halo) : (const void*)pick_ring(tf, shape, mode, halo),
            ring_smem_bytes(tf, g * ng, ng), ring_cta_warps(tf, g * ng, ng)};
}

// fn(ring instance) for every instance launch_spmm can pick: the tensor-map fill in every shape, the 1-D bulk fill in
// the two 16-row-slot-group shapes, the cp.async fill (full-width tiles) in shape 0; stops at the first nonzero return.
template <class F>
int for_each_ring(F fn)
{
    int rc;
    for (int tf = 64; tf <= 256; tf *= 2)
        for (int halo = 0; halo < 2; ++halo) {
            for (int shape = 0; shape < 4; ++shape)
                if ((rc = fn(ring_inst(tf, shape, 2, halo != 0)))) return rc;
            for (int shape = 0; shape < 2; ++shape)
                if ((rc = fn(ring_inst(tf, shape, 0, halo != 0)))) return rc;
            if (tf >= 128 && (rc = fn(ring_inst(tf, 0, 1, halo != 0)))) return rc;
        }
    return 0;
}

typedef void (*attn_fn)(const AttnArgs);

// the edge softmax instance of K heads (VEC: vector loads of the K values of an entry or row)
template <int K>
attn_fn pick_softmax_k(bool vec, bool backward)
{
    if (vec) return backward ? edge_softmax_backward_kernel<K, true> : edge_softmax_kernel<K, true>;
    return backward ? edge_softmax_backward_kernel<K, false> : edge_softmax_kernel<K, false>;
}
attn_fn pick_softmax(int k, bool vec, bool backward)
{
    switch (k) {
        case 1: return backward ? edge_softmax_backward_kernel<1, false> : edge_softmax_kernel<1, false>;
        case 2: return pick_softmax_k<2>(vec, backward);
        case 4: return pick_softmax_k<4>(vec, backward);
        default: return pick_softmax_k<8>(vec, backward);
    }
}

typedef void (*sddmm_fn)(const SddmmArgs);

template <int NV>
sddmm_fn pick_sddmm_heads_nv(int k)
{
    switch (k) {
        case 2: return sddmm_heads_ring_kernel<NV, 2>;
        case 4: return sddmm_heads_ring_kernel<NV, 4>;
        default: return sddmm_heads_ring_kernel<NV, 8>;
    }
}
// the multi-head SDDMM ring instance of f = 128 nv (nv = 1, 2, 4) and k = 2, 4, 8 heads
sddmm_fn pick_sddmm_heads(int nv, int k)
{
    if (nv == 1) return pick_sddmm_heads_nv<1>(k);
    if (nv == 2) return pick_sddmm_heads_nv<2>(k);
    return pick_sddmm_heads_nv<4>(k);
}

// GATv2 instances (gatv2.cuh): the score ring kernel of f = 128 nv (nv = 1, 2) and k heads, the raw-score softmax,
// and the two backward walks with the multi-head launch shape
typedef void (*gatv2_score_fn)(SddmmArgs, const Gatv2Halo, const float*, float);
template <int NV>
gatv2_score_fn pick_gatv2_ring_nv(int k)
{
    switch (k) {
        case 1: return gatv2_score_ring_kernel<NV, 1>;
        case 2: return gatv2_score_ring_kernel<NV, 2>;
        case 4: return gatv2_score_ring_kernel<NV, 4>;
        default: return gatv2_score_ring_kernel<NV, 8>;
    }
}
gatv2_score_fn pick_gatv2_ring(int nv, int k) { return nv == 1 ? pick_gatv2_ring_nv<1>(k) : pick_gatv2_ring_nv<2>(k); }

template <int K>
attn_fn pick_softmax_raw_k(bool vec, bool backward)
{
    if (vec) return backward ? edge_softmax_raw_backward_kernel<K, true> : edge_softmax_raw_kernel<K, true>;
    return backward ? edge_softmax_raw_backward_kernel<K, false> : edge_softmax_raw_kernel<K, false>;
}
attn_fn pick_softmax_raw(int k, bool vec, bool backward)
{
    switch (k) {
        case 1: return backward ? edge_softmax_raw_backward_kernel<1, false> : edge_softmax_raw_kernel<1, false>;
        case 2: return pick_softmax_raw_k<2>(vec, backward);
        case 4: return pick_softmax_raw_k<4>(vec, backward);
        default: return pick_softmax_raw_k<8>(vec, backward);
    }
}

typedef void (*gatv2_bwd_fn)(const SpmmArgs, const Gatv2BwdArgs);

template <int LPE, int VW>
gatv2_bwd_fn pick_gatv2_bwd_nh(int nh, bool col, bool halo)
{
    switch (nh) {
        case 1: return col ? gatv2_col_backward_kernel<LPE, VW, 1>
                           : (halo ? gatv2_row_backward_kernel<LPE, VW, true, 1> : gatv2_row_backward_kernel<LPE, VW, false, 1>);
        case 2: return col ? gatv2_col_backward_kernel<LPE, VW, 2>
                           : (halo ? gatv2_row_backward_kernel<LPE, VW, true, 2> : gatv2_row_backward_kernel<LPE, VW, false, 2>);
        case 4: return col ? gatv2_col_backward_kernel<LPE, VW, 4>
                           : (halo ? gatv2_row_backward_kernel<LPE, VW, true, 4> : gatv2_row_backward_kernel<LPE, VW, false, 4>);
        default:   // no 8-head instance at LPE = 4, as pick_heads_nh
            if constexpr (LPE > 4)
                return col ? gatv2_col_backward_kernel<LPE, VW, 8>
                           : (halo ? gatv2_row_backward_kernel<LPE, VW, true, 8> : gatv2_row_backward_kernel<LPE, VW, false, 8>);
            else return nullptr;
    }
}
template <int VW>
gatv2_bwd_fn pick_gatv2_bwd_lpe(int lpe, int nh, bool col, bool halo)
{
    switch (lpe) {
        case 4: return pick_gatv2_bwd_nh<4, VW>(nh, col, halo);
        case 8: return pick_gatv2_bwd_nh<8, VW>(nh, col, halo);
        case 16: return pick_gatv2_bwd_nh<16, VW>(nh, col, halo);
        default: return pick_gatv2_bwd_nh<32, VW>(nh, col, halo);
    }
}
// col: the transposed (dxl) walk, else the row (dxr, datt) walk with or without a halo operand
gatv2_bwd_fn pick_gatv2_bwd(int lpe, int vw, int nh, bool col, bool halo)
{
    return vw == 4 ? pick_gatv2_bwd_lpe<4>(lpe, nh, col, halo) : pick_gatv2_bwd_lpe<1>(lpe, nh, col, halo);
}

// CUDA loads kernels lazily, at their first launch, and that load synchronises with the device. A rank whose
// stream already holds a spinning p2p_wait_kernel must therefore never launch a not-yet-loaded kernel behind it
// when the ranks it waits for live in the SAME process (single-process multi-rank use: tests, smoke) — their put
// kernels would never be enqueued. Touching every kernel once, when the peer transport is set up, removes the hazard.
template <class F>
void touch_kernel(F fn)
{
    cudaFuncAttributes fa;
    if (fn && cudaFuncGetAttributes(&fa, (const void*)fn) != cudaSuccess) cudaGetLastError();   // null: no such instance
}

void preload_kernels()
{
    static bool done = false;
    if (done) return;
    done = true;
    for (int halo = 0; halo < 2; ++halo)
        for (int lpe = 4; lpe <= 32; lpe *= 2)
            for (int vpl = 1; vpl <= 4; vpl *= 2) { touch_kernel(pick_lpe<4>(lpe, vpl, halo != 0)); touch_kernel(pick_lpe<1>(lpe, vpl, halo != 0)); }
    for_each_ring([](const RingInst& ri) { touch_kernel(ri.fn); return 0; });
    touch_kernel(zero_rows_kernel<4>); touch_kernel(zero_rows_kernel<1>);
    touch_kernel(spmm_fixup_kernel<4>); touch_kernel(spmm_fixup_kernel<1>);
    touch_kernel(pack_rows_kernel<4>); touch_kernel(pack_rows_kernel<1>);
    touch_kernel(unpack_add_kernel<4>); touch_kernel(unpack_add_kernel<1>);
    touch_kernel(put_rows_kernel<4>); touch_kernel(put_rows_kernel<1>); touch_kernel(p2p_wait_kernel); touch_kernel(epoch_advance_kernel);
    touch_kernel(set_values_kernel); touch_kernel(copy_halo_kernel); touch_kernel(sddmm_plain_kernel);
    touch_kernel(sddmm_ring_kernel<1>); touch_kernel(sddmm_ring_kernel<2>);
    touch_kernel(sddmm_ring_kernel<3>); touch_kernel(sddmm_ring_kernel<4>);
    touch_kernel(edge_softmax_kernel<1, false>); touch_kernel(edge_softmax_backward_kernel<1, false>);
    for (int halo = 0; halo < 2; ++halo)
        for (int lpe = 4; lpe <= 32; lpe *= 2)
            for (int nh = 1; nh <= 8; nh *= 2) { touch_kernel(pick_heads(lpe, 4, halo != 0, nh)); touch_kernel(pick_heads(lpe, 1, halo != 0, nh)); }
    for (int nh = 2; nh <= 8; nh *= 2)
        for (int vec = 0; vec < 2; ++vec) { touch_kernel(pick_softmax(nh, vec != 0, false)); touch_kernel(pick_softmax(nh, vec != 0, true)); }
    for (int nv = 1; nv <= 4; nv *= 2)
        for (int nh = 2; nh <= 8; nh *= 2) touch_kernel(pick_sddmm_heads(nv, nh));
    touch_kernel(sddmm_plain_heads_kernel);
    for (int lpe = 4; lpe <= 32; lpe *= 2)
        for (int vw = 1; vw <= 4; vw += 3) {
            touch_kernel(pick_max(lpe, vw, false)); touch_kernel(pick_max(lpe, vw, true)); touch_kernel(pick_max_bwd(lpe, vw));
        }
    touch_kernel(spmm_max_fixup_kernel<4>); touch_kernel(spmm_max_fixup_kernel<1>);
    touch_kernel(max_empty_rows_kernel<4>); touch_kernel(max_empty_rows_kernel<1>);
    for (int nh = 1; nh <= 8; nh *= 2) {
        for (int nv = 1; nv <= 2; ++nv) touch_kernel(pick_gatv2_ring(nv, nh));
        for (int vec = 0; vec < 2; ++vec) { touch_kernel(pick_softmax_raw(nh, vec != 0, false)); touch_kernel(pick_softmax_raw(nh, vec != 0, true)); }
        for (int lpe = 4; lpe <= 32; lpe *= 2)
            for (int vw = 1; vw <= 4; vw += 3)
                for (int kind = 0; kind < 3; ++kind) touch_kernel(pick_gatv2_bwd(lpe, vw, nh, kind == 2, kind == 1));
    }
    touch_kernel(gatv2_score_plain_kernel); touch_kernel(gatv2_datt_kernel);
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

// Vector width of the element-wise kernels (register SpMM, zero-rows, fixup, pack, unpack, put): 16-byte accesses need
// whole 4-float vectors AND every operand the launch accesses by vector 16-byte aligned (null operands do not count).
// Any other operand takes the scalar instances, which are slower but compute the same bits.
int vec_width(int f, std::initializer_list<const void*> ops)
{
    if (f % 4 != 0) return 1;
    for (const void* q : ops)
        if (!aligned16(q)) return 1;
    return 4;
}

// Which SpMM kernel serves width f with these operands: the shared-memory ring (TMA bulk copies) needs whole
// 128-float vectors and 16-byte aligned rows; everything else takes the register pipeline.
bool use_ring(const pgcn_plan* p, const float* H0, const float* H1, int f)
{
    if (p->opt_kernel == 4) return false;
    return f % 128 == 0 && aligned16(H0) && aligned16(H1);
}

// Opt kernel fn in to its dynamic shared memory (> 48 KB) and record its occupancy at `threads` threads, once per plan;
// *ctas (when not null) = its CTAs per SM. Setting the attribute is refused while `st` is being captured.
int opt_in(pgcn_plan* p, const void* fn, size_t smem, int threads, cudaStream_t st, int* ctas)
{
    auto it = p->ctas_per_sm.find(fn);
    if (it == p->ctas_per_sm.end()) {
        int rc = refuse_under_capture(p, st);
        if (rc) return rc;
        CU(p, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int nb = 0;
        CU(p, cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(&nb, fn, threads, smem, 0));
        it = p->ctas_per_sm.emplace(fn, std::max(nb, 1)).first;
    }
    if (ctas) *ctas = it->second;
    return 0;
}

// Grid of a register-schedule launch: one group of t.lpe lanes per row block, kSpmmThreads / t.lpe groups per CTA, the
// row's tiles along y.
dim3 walk_grid(const DevCsr::Sched& sc, const TileCfg& t)
{
    const int groups_per_cta = kSpmmThreads / t.lpe;
    return dim3((unsigned)((sc.nblocks + groups_per_cta - 1) / groups_per_cta), (unsigned)t.tiles);
}

const auto no_setup = [](const DevCsr::Sched&) { return 0; };

// One launch over a schedule of matrix c and the launches around it: the schedule, the caller's setup(sc), the
// zero-fill of the empty rows (beta == 0), launch(args, sc) over the row blocks, then the fixup of the split rows. All
// set-up runs before the first launch, so a call refused under capture has enqueued nothing. `a` holds the operands,
// outputs and epilogue (the schedule's fields are filled in here); vw: the vector width of the zero-fill and fixup.
template <class Setup, class Launch>
int launch_walk(pgcn_plan* p, DevCsr& c, bool ring, SpmmArgs a, int vw, cudaStream_t st, Setup setup, Launch launch)
{
    if (c.nrows == 0) return 0;
    DevCsr::Sched* sc;
    int rc;
    if ((rc = schedule(p, c, ring, st, &sc)) || (rc = setup(*sc))) return rc;
    if (c.nempty > 0 && !a.beta) {
        ZeroArgs za;
        za.rows = c.d_empty; za.nrows_empty = c.nempty; za.Z0 = a.Z0; za.Z1 = a.Z1; za.zsplit = a.zsplit; za.f = a.f;
        const unsigned grid = (unsigned)(((long long)c.nempty * (a.f / vw) + 255) / 256);
        if (vw == 4) zero_rows_kernel<4><<<grid, 256, 0, st>>>(za);
        else zero_rows_kernel<1><<<grid, 256, 0, st>>>(za);
        ++p->launches;
    }
    a.blocks = sc->d_blocks; a.nblocks = sc->nblocks;
    a.pieces = c.d_cw;
    a.rowids = c.d_rowids;
    a.partial = sc->d_partial;
    if (sc->nblocks > 0) {
        if ((rc = launch(a, *sc))) return rc;
        ++p->launches;
    }
    if (sc->nlong > 0) {
        FixupArgs fa;
        fa.long_rows = sc->d_long; fa.nlong = sc->nlong; fa.partial = sc->d_partial;
        fa.Z0 = a.Z0; fa.Z1 = a.Z1; fa.zsplit = a.zsplit; fa.rowids = c.d_rowids; fa.f = a.f; fa.beta = a.beta;
        fa.relu = a.relu; fa.final = a.final;
        const unsigned grid = (unsigned)sc->nlong * (unsigned)((a.f / vw + 31) / 32);
        if (vw == 4) spmm_fixup_kernel<4><<<grid, 32 * kFixupGroups, 0, st>>>(fa);
        else spmm_fixup_kernel<1><<<grid, 32 * kFixupGroups, 0, st>>>(fa);
        ++p->launches;
    }
    CU(p, cudaGetLastError());
    return 0;
}

// Weights of a multi-head aggregation: nh heads of width f / nh; alpha is nnz x nh in forward CSR order, map (null for
// the forward records) takes an entry of the launched matrix to its forward entry.
struct HeadArgs {
    const float* alpha;
    const int* map;
    int nh;
};

// H_odd: the halo slab of odd exchange epochs when the operand that holds the halo slab (H1, or H0 without H1) is the
// peer transport's double-buffered slab; the kernels then pick the buffer from the plan's device epoch.
// heads: multi-head weights instead of the records' values; the launch then takes the register kernel (schedule 0) and
// its multi-head instance. Null: nothing changes.
int launch_spmm(pgcn_plan* p, DevCsr& c, const float* H0, const float* H1, int split,
                float* Z0, float* Z1, int zsplit, int f, int beta, cudaStream_t st, int relu = 0, bool use_final = false,
                const float* H_odd = nullptr, const HeadArgs* heads = nullptr)
{
    const bool ring = !heads && use_ring(p, H0, H1, f) && aligned16(Z0) && aligned16(Z1) && (!H_odd || aligned16(H_odd));
    // multi-head: 4-float vectors also need whole vectors per head
    const int vw = (heads && (f / heads->nh) % 4 != 0) ? 1 : vec_width(f, {H0, H1, H_odd, Z0, Z1});
    const bool halo = (H1 != nullptr);
    SpmmArgs a = {};
    a.H0 = H0; a.H1 = H1; a.split = split;
    a.Z0 = Z0; a.Z1 = Z1; a.zsplit = zsplit;
    a.f = f; a.beta = beta;
    a.relu = relu; a.final = (relu && use_final) ? c.d_final : nullptr;
    a.H_odd = H_odd; a.epoch = H_odd ? p->d_epoch : nullptr;
    if (!ring) {
        const TileCfg t = heads ? choose_tile_heads(f, vw) : choose_tile(p, f, vw);
        return launch_walk(p, c, false, a, vw, st, no_setup, [&](const SpmmArgs& args, const DevCsr::Sched& sc) {
            if (heads) {
                SpmmHeadArgs ha;
                ha.alpha = heads->alpha; ha.amap = heads->map; ha.hd = f / heads->nh;
                pick_heads(t.lpe, t.vw, halo, heads->nh)<<<walk_grid(sc, t), kSpmmThreads, 0, st>>>(args, ha);
            } else {
                spmm_fn fn = (t.vw == 4) ? pick_lpe<4>(t.lpe, t.vpl, halo) : pick_lpe<1>(t.lpe, t.vpl, halo);
                fn<<<walk_grid(sc, t), kSpmmThreads, 0, st>>>(args);
            }
            return 0;
        });
    }
    int mode = p->opt_kernel == 6 ? 1 : (p->opt_kernel == 5 ? 0 : 2);   // default: 2-D tensor-map TMA
    // row tile: the option, else the tuned width, else the full width (256 floats when f allows, else 128);
    // a width that does not divide f, and 64-float slices with the cp.async fill, take the full width
    const int full = (f % 256 == 0) ? 256 : 128;
    int tf = (int)(p->opt_ring_tile > 0 ? p->opt_ring_tile : (c.tuned_tile > 0 ? c.tuned_tile : full));
    if (f % tf != 0 || (mode == 1 && tf < 128)) tf = full;
    const int tiles = f / tf;
    // ring shape from the options: ring_slots = 16 | 32 | 64, ring_groups = 2 | 4 (only with 64 slots)
    const int64_t want_slots = c.tuned_slots > 0 ? c.tuned_slots : p->opt_ring_slots;
    int shape = want_slots <= 16 ? 0 : (want_slots <= 32 ? 1 : (p->opt_ring_groups == 4 ? 3 : 2));
    CUtensorMap tm0, tm1, tm_odd;
    if (mode == 2) {
        // H0 holds the columns below `split` (all of them when there is no halo slab), H1 the rest
        bool ok = make_row_map(&tm0, H0, 1 << 30, f, tf, 1);
        if (ok && H1) ok = make_row_map(&tm1, H1, 1 << 30, f, tf, 1);
        else if (ok) tm1 = tm0;
        if (ok && H_odd) ok = make_row_map(&tm_odd, H_odd, 1 << 30, f, tf, 1);
        else if (ok) tm_odd = tm1;
        if (!ok) mode = 0;                                   // no driver entry point: 1-D bulk copies
    }
    if (mode == 1) shape = 0;
    if (mode == 0 && shape > 1) shape = 1;
    const RingInst ri = ring_inst(tf, shape, mode, halo);
    int ctas = 0;
    auto setup = [&](const DevCsr::Sched& sc) {
        return sc.nblocks > 0 ? opt_in(p, ri.fn, ri.smem, ri.warps * 32, st, &ctas) : 0;
    };
    return launch_walk(p, c, true, a, vw, st, setup, [&](const SpmmArgs& args, const DevCsr::Sched& sc) -> int {
        RingArgs ra;
        ra.counter = nullptr; ra.hub = nullptr; ra.nhub = 0;
        dim3 grid((unsigned)((sc.nblocks + ri.warps - 1) / ri.warps), (unsigned)tiles);
        // Persistent CTAs own their SM (shared memory + registers) until the whole launch is done; a put / NCCL kernel
        // of the exchange stream would then wait behind the SpMM it is supposed to overlap (measured at 8 GPUs: step =
        // sum of puts + sum of SpMMs). Multi-rank plans with overlap therefore run one block per warp (CTAs retire
        // every few dozen microseconds and the higher-priority exchange kernels take the freed slots) unless
        // `persistent_multi` asks otherwise.
        const bool persistent = p->opt_persistent && (p->k == 1 || !p->opt_overlap || p->opt_persistent_multi);
        if (persistent) {
            // one counter over all (tile, row block) items, tile-major: the tiles run one after the other
            CU(p, cudaMemsetAsync(p->d_counter, 0, sizeof(unsigned int), st));
            ra.counter = p->d_counter;
            const unsigned items = (unsigned)(((int64_t)sc.nblocks * tiles + ri.warps - 1) / ri.warps);
            grid.x = std::min<unsigned>(items, (unsigned)(p->num_sms * ctas));
            grid.y = 1;
        }
        if (mode == 2) pick_ring_tm(tf, shape, halo)<<<grid, ri.warps * 32, ri.smem, st>>>(args, ra, tm0, tm1, tm_odd);
        else pick_ring(tf, shape, mode, halo)<<<grid, ri.warps * 32, ri.smem, st>>>(args, ra);
        return 0;
    });
}

int check_f(pgcn_plan* p, int f)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (f <= 0 || f > p->f_max) return fail(p, PGCN_ERR_INVALID, "f=%d outside (0, f_max=%d]", f, p->f_max);
    return 0;
}

unsigned grid_for(long long total, int num_sms)
{
    long long g = (total + 255) / 256;
    return (unsigned)std::max<long long>(1, std::min<long long>(g, 32LL * num_sms));
}

int launch_pack(pgcn_plan* p, const float* H, float* slab, int f, cudaStream_t st)
{
    if (p->S == 0) return 0;
    PackArgs a;
    a.send_idx = p->d_send_idx; a.S = p->S; a.H = H; a.slab = slab; a.f = f;
    const int vw = vec_width(f, {H, slab});
    const unsigned grid = grid_for(p->S * (f / vw), p->num_sms);
    if (vw == 4) pack_rows_kernel<4><<<grid, 256, 0, st>>>(a);
    else pack_rows_kernel<1><<<grid, 256, 0, st>>>(a);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// recv_odd: the reverse slab of odd exchange epochs when `recv` is the peer transport's double-buffered slab
int launch_unpack(pgcn_plan* p, const float* recv, float* G, int f, cudaStream_t st, const float* recv_odd = nullptr)
{
    if (p->nb == 0) return 0;
    UnpackArgs a;
    a.brow = p->d_brow; a.bptr = p->d_bptr; a.bpos = p->d_bpos; a.nb = p->nb;
    a.recv = recv; a.G = G; a.f = f;
    a.recv_odd = recv_odd; a.epoch = recv_odd ? p->d_epoch : nullptr;
    const int vw = vec_width(f, {recv, recv_odd, G});
    const long long total = (long long)p->nb * (f / vw);
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (vw == 4) unpack_add_kernel<4><<<grid, 256, 0, st>>>(a);
    else unpack_add_kernel<1><<<grid, 256, 0, st>>>(a);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// ---- max aggregation -------------------------------------------------------------------------

// The entries of the (value, entry) partials of a schedule's split rows: allocated once per schedule, the first time a
// max call or pgcn_plan_prepare of a bound plan needs them (never under capture), and retired with the schedule.
int max_partial(pgcn_plan* p, DevCsr::Sched& sc, cudaStream_t st)
{
    if (sc.nslots == 0 || sc.d_apart) return 0;
    int rc = refuse_under_capture(p, st);
    if (rc) return rc;
    CU(p, cudaMalloc((void**)&sc.d_apart, (size_t)sc.nslots * p->f_max * sizeof(int)));
    return 0;
}

// Z, arg = the max over each forward row's entries of [H0 | H1] (H1: the halo slab, H_odd its odd-epoch twin or null),
// on the register schedule of the forward records.
int launch_max(pgcn_plan* p, const float* H0, const float* H1, const float* H_odd, float* Z, int* arg, int f,
               cudaStream_t st)
{
    DevCsr& c = p->fwd;
    if (c.nrows == 0) return 0;
    DevCsr::Sched* sc;
    int rc;
    if ((rc = schedule(p, c, false, st, &sc)) || (rc = max_partial(p, *sc, st))) return rc;
    const int vw = vec_width(f, {H0, H1, H_odd, Z, arg});
    const TileCfg t = choose_tile_heads(f, vw);
    if (c.nempty > 0) {
        MaxEmptyArgs za;
        za.rows = c.d_empty; za.nrows_empty = c.nempty; za.Z = Z; za.arg = arg; za.f = f;
        const unsigned grid = (unsigned)(((long long)c.nempty * (f / vw) + 255) / 256);
        if (vw == 4) max_empty_rows_kernel<4><<<grid, 256, 0, st>>>(za);
        else max_empty_rows_kernel<1><<<grid, 256, 0, st>>>(za);
        ++p->launches;
    }
    if (sc->nblocks > 0) {
        SpmmArgs a;
        a.blocks = sc->d_blocks; a.nblocks = sc->nblocks;
        a.pieces = c.d_cw;
        a.H0 = H0; a.H1 = H1; a.split = p->m;
        a.Z0 = Z; a.Z1 = nullptr; a.zsplit = p->m;
        a.rowids = c.d_rowids;
        a.partial = sc->d_partial; a.f = f; a.beta = 0;
        a.relu = 0; a.final = nullptr;
        a.H_odd = H_odd; a.epoch = H_odd ? p->d_epoch : nullptr;
        pick_max(t.lpe, vw, H1 != nullptr)<<<walk_grid(*sc, t), kSpmmThreads, 0, st>>>(a, arg, sc->d_apart);
        ++p->launches;
    }
    if (sc->nlong > 0) {
        MaxFixupArgs fa;
        fa.long_rows = sc->d_long; fa.partial = sc->d_partial; fa.apart = sc->d_apart;
        fa.Z = Z; fa.arg = arg; fa.rowids = c.d_rowids; fa.f = f;
        const unsigned grid = (unsigned)sc->nlong * (unsigned)((f / vw + 31) / 32);
        if (vw == 4) spmm_max_fixup_kernel<4><<<grid, 32 * kFixupGroups, 0, st>>>(fa);
        else spmm_max_fixup_kernel<1><<<grid, 32 * kFixupGroups, 0, st>>>(fa);
        ++p->launches;
    }
    CU(p, cudaGetLastError());
    return 0;
}

// G_own (rows [0, m)) and G_halo (rows [m, m + h)) = gZ routed by arg, on the register schedule of the transposed records.
int launch_max_backward(pgcn_plan* p, const int* arg, const float* gZ, float* G_own, float* G_halo, int f, cudaStream_t st)
{
    const int vw = vec_width(f, {gZ, arg, G_own, G_halo});
    const TileCfg t = choose_tile_heads(f, vw);
    SpmmArgs a = {};
    a.H0 = gZ; a.split = p->m;
    a.Z0 = G_own; a.Z1 = G_halo; a.zsplit = p->m;
    a.f = f;
    return launch_walk(p, p->tr, false, a, vw, st, no_setup, [&](const SpmmArgs& args, const DevCsr::Sched& sc) {
        pick_max_bwd(t.lpe, vw)<<<walk_grid(sc, t), kSpmmThreads, 0, st>>>(args, arg, p->tr.d_vmap);
        return 0;
    });
}

// ---- edge values -----------------------------------------------------------------------------

sddmm_fn pick_sddmm(int nv)
{
    switch (nv) {
        case 1: return sddmm_ring_kernel<1>;
        case 2: return sddmm_ring_kernel<2>;
        case 3: return sddmm_ring_kernel<3>;
        default: return sddmm_ring_kernel<4>;
    }
}

// The SDDMM ring kernel serves f = 128 .. 512 in steps of 128 with 16-byte aligned operands, like the SpMM ring
bool sddmm_use_ring(const pgcn_plan* p, const float* gZ, const float* H0, const float* H1, int f)
{
    return use_ring(p, gZ, H0, f) && f <= 512 && (!H1 || aligned16(H1));
}

// The edge launch over the forward records shared by the SDDMM, the multi-head SDDMM and the GATv2 scores: gZ is the
// row operand, H0 / H1 the column operands (H1: the halo rows, columns >= m), out takes the values of the entries.
// On the ring schedule, persistent CTAs of ring_fn (its shared memory of width f opted in) take row blocks from the
// plan's counter; on the register schedule, the plain kernel takes 8 row blocks per CTA. launch(args, grid, threads,
// smem) launches ring_fn or the plain kernel with the call's further arguments.
template <class Launch>
int launch_edges(pgcn_plan* p, bool ring, const void* ring_fn, const float* gZ, const float* H0, const float* H1,
                 float* out, int f, cudaStream_t st, Launch launch)
{
    DevCsr& c = p->fwd;
    if (c.nnz == 0 || c.nrows == 0) return 0;
    DevCsr::Sched* sc;
    int rc = schedule(p, c, ring, st, &sc);
    if (rc || sc->nblocks == 0) return rc;
    SddmmArgs a;
    a.blocks = sc->d_blocks; a.nblocks = sc->nblocks;
    a.pieces = c.d_cw;
    a.gZ = gZ; a.H0 = H0; a.H1 = H1; a.split = p->m;
    a.rowids = c.d_rowids;
    a.dvals = out; a.f = f;
    a.counter = nullptr;
    if (ring) {
        const size_t smem = sddmm_smem_bytes(f / 128);
        int ctas = 0;
        if ((rc = opt_in(p, ring_fn, smem, kSddmmWarps * 32, st, &ctas))) return rc;
        CU(p, cudaMemsetAsync(p->d_counter, 0, sizeof(unsigned int), st));
        a.counter = p->d_counter;
        const unsigned nctas = (unsigned)((sc->nblocks + kSddmmWarps - 1) / kSddmmWarps);
        launch(a, std::min<unsigned>(nctas, (unsigned)(p->num_sms * ctas)), kSddmmWarps * 32, smem);
    } else {
        launch(a, (unsigned)((sc->nblocks + 7) / 8), 256, (size_t)0);
    }
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// dvals = SDDMM over the forward matrix (H1: the halo rows, columns >= m)
int launch_sddmm(pgcn_plan* p, const float* gZ, const float* H0, const float* H1, float* dvals, int f, cudaStream_t st)
{
    const bool ring = sddmm_use_ring(p, gZ, H0, H1, f);
    const sddmm_fn fn = pick_sddmm(f / 128);
    return launch_edges(p, ring, (const void*)fn, gZ, H0, H1, dvals, f, st,
                        [&](const SddmmArgs& a, unsigned grid, int threads, size_t smem) {
        if (ring) fn<<<grid, threads, smem, st>>>(a);
        else sddmm_plain_kernel<<<grid, threads, smem, st>>>(a);
    });
}

// The multi-head SDDMM ring instance serves f = 128, 256 or 512 with 2, 4 or 8 heads of at least 4 floats and 16-byte
// aligned operands (the single-head ring's rule); k == 1 is pgcn_sddmm itself.
bool sddmm_heads_use_ring(const pgcn_plan* p, const float* gZ, const float* H0, const float* H1, int f, int k)
{
    return k > 1 && (f == 128 || f == 256 || f == 512) && (f / k) % 4 == 0 && sddmm_use_ring(p, gZ, H0, H1, f);
}

// dalpha (nnz x k) = the SDDMM per head over the forward matrix; k == 1 is launch_sddmm
int launch_sddmm_heads(pgcn_plan* p, int k, const float* gZ, const float* H0, const float* H1, float* dalpha, int f,
                       cudaStream_t st)
{
    if (k == 1) return launch_sddmm(p, gZ, H0, H1, dalpha, f, st);
    const bool ring = sddmm_heads_use_ring(p, gZ, H0, H1, f, k);
    const sddmm_fn fn = pick_sddmm_heads(f / 128, k);
    return launch_edges(p, ring, (const void*)fn, gZ, H0, H1, dalpha, f, st,
                        [&](const SddmmArgs& a, unsigned grid, int threads, size_t smem) {
        if (ring) fn<<<grid, threads, smem, st>>>(a);
        else sddmm_plain_heads_kernel<<<grid, threads, smem, st>>>(a, k);
    });
}

// ---- GATv2 ----------------------------------------------------------------------------------

// The datt partials of the forward register schedule (f_max floats per chunk of kGatv2Chunk row blocks): allocated once
// per schedule, the first time a GATv2 backward or pgcn_plan_prepare of a bound plan needs them (never under capture),
// and retired with the schedule.
int gatv2_partial(pgcn_plan* p, DevCsr::Sched& sc, cudaStream_t st)
{
    if (sc.nblocks == 0 || sc.d_datt) return 0;
    int rc = refuse_under_capture(p, st);
    if (rc) return rc;
    const size_t nchunks = (size_t)(sc.nblocks + kGatv2Chunk - 1) / kGatv2Chunk;
    CU(p, cudaMalloc((void**)&sc.d_datt, nchunks * p->f_max * sizeof(float)));
    return 0;
}

// The GATv2 score ring instance serves f = 128 and 256 with 16-byte aligned operands (the multi-head SDDMM's rule)
bool gatv2_use_ring(const pgcn_plan* p, const float* xr, const float* xl, const float* H1, const float* H1_odd,
                    const float* att, int f)
{
    return (f == 128 || f == 256) && sddmm_use_ring(p, xr, xl, H1, f) && aligned16(H1_odd) && aligned16(att);
}

// scores (nnz x k, forward CSR order) of the forward records, written into `out`; H1 / H1_odd: the halo slab of the
// call and its odd-epoch twin on the peer transport (or null)
int launch_gatv2_score(pgcn_plan* p, int k, const float* xr, const float* xl, const float* H1, const float* H1_odd,
                       const float* att, float slope, float* out, int f, cudaStream_t st)
{
    const bool ring = gatv2_use_ring(p, xr, xl, H1, H1_odd, att, f);
    const gatv2_score_fn fn = pick_gatv2_ring(f / 128, k);
    const Gatv2Halo hl = {H1_odd, H1_odd ? p->d_epoch : nullptr};
    return launch_edges(p, ring, (const void*)fn, xr, xl, H1, out, f, st,
                        [&](const SddmmArgs& a, unsigned grid, int threads, size_t smem) {
        if (ring) fn<<<grid, threads, smem, st>>>(a, hl, att, slope);
        else gatv2_score_plain_kernel<<<grid, threads, smem, st>>>(a, hl, att, slope, k);
    });
}

// One of the two backward walks on the register schedule of c (the forward records: dxr and the datt partials; the
// transposed ones: dxl and the halo partials), its empty rows and its split rows. vw: as the multi-head aggregation.
int launch_gatv2_walk(pgcn_plan* p, DevCsr& c, bool col, int k, const SpmmArgs& a, Gatv2BwdArgs g,
                      std::initializer_list<const void*> ops, cudaStream_t st)
{
    const int vw = (a.f / k) % 4 != 0 ? 1 : vec_width(a.f, ops);
    const TileCfg t = choose_tile_heads(a.f, vw);
    auto setup = [&](DevCsr::Sched& sc) { return col ? 0 : gatv2_partial(p, sc, st); };
    return launch_walk(p, c, false, a, vw, st, setup, [&](const SpmmArgs& args, const DevCsr::Sched& sc) {
        g.datt_part = sc.d_datt;
        pick_gatv2_bwd(t.lpe, vw, k, col, args.H1 != nullptr)<<<walk_grid(sc, t), kSpmmThreads, 0, st>>>(args, g);
        return 0;
    });
}

// dxr (m x f) and datt (f) from dscore (nnz x k) on the forward records
int launch_gatv2_rows(pgcn_plan* p, int k, const float* dscore, const float* xl, const float* xl_halo, const float* xr,
                      const float* att, float slope, float* dxr, float* datt, int f, cudaStream_t st)
{
    DevCsr& c = p->fwd;
    if (c.nrows > 0) {
        SpmmArgs a = {};
        a.H0 = xl; a.H1 = xl_halo; a.split = p->m;
        a.Z0 = dxr; a.Z1 = nullptr; a.zsplit = p->m;
        a.f = f;
        Gatv2BwdArgs g = {};
        g.dscore = dscore; g.att = att; g.slope = slope; g.hd = f / k; g.xv = xr;
        int rc = launch_gatv2_walk(p, c, false, k, a, g, {xl, xl_halo, xr, att, dxr}, st);
        if (rc) return rc;
    }
    const int nblocks = c.nrows > 0 ? c.sched[0].nblocks : 0;
    if (nblocks == 0) {
        CU(p, cudaMemsetAsync(datt, 0, (size_t)f * sizeof(float), st));
        return 0;
    }
    const int nchunks = (nblocks + kGatv2Chunk - 1) / kGatv2Chunk;
    gatv2_datt_kernel<<<(unsigned)((f + 31) / 32), 32 * kGatv2RedWarps, 0, st>>>(c.sched[0].d_datt, nchunks, f, datt);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// dxl (rows < m) and the halo partials (rows m .., into G_halo) on the transposed records
int launch_gatv2_cols(pgcn_plan* p, int k, const float* alpha, const float* dscore, const float* gZ, const float* xl,
                      const float* xl_halo, const float* xr, const float* att, float slope, float* dxl, float* G_halo,
                      int f, cudaStream_t st)
{
    DevCsr& c = p->tr;
    if (c.nrows == 0) return 0;
    SpmmArgs a = {};
    a.H0 = gZ; a.H1 = xr; a.split = p->m;
    a.Z0 = dxl; a.Z1 = G_halo; a.zsplit = p->m;
    a.f = f;
    Gatv2BwdArgs g = {};
    g.alpha = alpha; g.dscore = dscore; g.att = att; g.slope = slope; g.hd = f / k; g.amap = c.d_vmap;
    g.xv = xl; g.xv_halo = xl_halo;
    return launch_gatv2_walk(p, c, true, k, a, g, {gZ, xr, xl, xl_halo, att, dxl, G_halo}, st);
}

// Set-up copies of pgcn_plan_bind_values. They run on the plan's own non-blocking stream and wait for that stream only:
// a device-wide (or legacy-stream) synchronisation could wait for another rank's spinning p2p_wait_kernel when several
// ranks' plans share this process, and that rank's puts would then never be enqueued. No compute call writes the
// records (only pgcn_plan_set_values does, and it needs the binding), so nothing has to be waited for.
int copy_setup(pgcn_plan* p, void* dst, const void* src, size_t bytes, cudaMemcpyKind kind)
{
    if (bytes == 0) return 0;
    CU(p, cudaMemcpyAsync(dst, src, bytes, kind, p->host_stream));
    CU(p, cudaStreamSynchronize(p->host_stream));
    return 0;
}

template <class T>
int upload_setup(pgcn_plan* p, T** dst, const T* src, size_t n)
{
    *dst = nullptr;
    CU(p, cudaMalloc((void**)dst, std::max<size_t>(n, 1) * sizeof(T)));
    return copy_setup(p, *dst, src, n * sizeof(T), cudaMemcpyHostToDevice);
}

// Download the records of a matrix and decode, per entry: its column, its value bits and its output row.
int decode_records(pgcn_plan* p, const DevCsr& c, std::vector<int>& col, std::vector<int>& val, std::vector<int>& row)
{
    const int64_t nnz = c.nnz;
    col.resize((size_t)nnz); val.resize((size_t)nnz); row.resize((size_t)nnz);
    if (nnz == 0) return 0;
    const size_t npieces = (size_t)((nnz + 31) / 32);
    std::vector<int> cw(npieces * kPieceInts);
    int rc;
    if ((rc = copy_setup(p, cw.data(), c.d_cw, cw.size() * sizeof(int), cudaMemcpyDeviceToHost))) return rc;
    std::vector<int> rowids;
    if (c.d_rowids) {
        rowids.resize((size_t)c.nrows_c);
        if ((rc = copy_setup(p, rowids.data(), c.d_rowids, rowids.size() * sizeof(int), cudaMemcpyDeviceToHost))) return rc;
    }
    int r = 0;
    for (int64_t e = 0; e < nnz; ++e) {
        const int* pc = cw.data() + (size_t)(e >> 5) * kPieceInts;
        const int i = (int)(e & 31);
        col[(size_t)e] = pc[i];
        val[(size_t)e] = pc[32 + i];
        row[(size_t)e] = rowids.empty() ? r : rowids[(size_t)r];
        if (((unsigned)pc[64] >> i) & 1u) ++r;
    }
    return 0;
}

// ---- transports ----------------------------------------------------------------------------

int nccl_exchange(pgcn_plan* p, const float* send, float* recv, int f, int reverse, cudaStream_t st)
{
    if (p->k == 1) return 0;
    if (!p->comm) return fail(p, PGCN_ERR_STATE, "exchange needs pgcn_comm_init (k=%d)", p->k);
    const std::vector<int64_t>& so = reverse ? p->recv_off : p->send_off;
    const std::vector<int64_t>& ro = reverse ? p->send_off : p->recv_off;
    NC(p, g_nccl.GroupStart());
    for (int q = 0; q < p->k; ++q) {
        if (q == p->rank) continue;
        const int64_t ns = so[q + 1] - so[q], nr = ro[q + 1] - ro[q];
        if (ns > 0) NC(p, g_nccl.Send(send + (size_t)so[q] * f, (size_t)ns * f, ncclFloat_, q, p->comm, st));
        if (nr > 0) NC(p, g_nccl.Recv(recv + (size_t)ro[q] * f, (size_t)nr * f, ncclFloat_, q, p->comm, st));
    }
    NC(p, g_nccl.GroupEnd());
    return 0;
}

float* arena_ptr(void* base, int64_t off) { return reinterpret_cast<float*>(static_cast<char*>(base) + off); }

unsigned long long* flag_slot(void* arena, int64_t off_flags, int slot)
{
    return reinterpret_cast<unsigned long long*>(static_cast<char*>(arena) + off_flags) + slot;
}

// Fused put of the rows bound for peer `dst` + epoch signal (peer-memory transport). `reverse`: halo partials of
// A^T g back to their owner (rows already in wire order), else boundary rows of H gathered through send_idx.
int p2p_put(pgcn_plan* p, int dst, const float* src, int f, bool reverse, cudaStream_t st)
{
    PutArgs a;
    const P2PBlob& pb = p->peer_blob[dst];
    for (int par = 0; par < 2; ++par) {                 // the kernel picks the slab of this call's epoch parity
        if (!reverse) a.dst[par] = arena_ptr(p->peer_arena[dst], pb.off_fwd[par]) + (size_t)pb.recv_off[p->rank] * f;
        else a.dst[par] = arena_ptr(p->peer_arena[dst], pb.off_bwd[par]) + (size_t)pb.send_off[p->rank] * f;
    }
    if (!reverse) {
        a.send_idx = p->d_send_idx; a.j0 = p->send_off[dst]; a.nrows = p->send_off[dst + 1] - p->send_off[dst];
    } else {
        a.send_idx = nullptr; a.j0 = p->recv_off[dst]; a.nrows = p->recv_off[dst + 1] - p->recv_off[dst];
    }
    a.src = src; a.f = f;
    a.done = p->d_done + (reverse ? 32 : 0) + dst;     // kMaxPeers <= 16 destinations per direction
    a.flag = flag_slot(p->peer_arena[dst], pb.off_flags, p->rank);
    a.epoch = p->d_epoch;
    // the peer slabs are 16-byte aligned (f % 4 == 0 on this transport); the caller's rows may not be
    const int vw = vec_width(f, {src});
    // enough CTAs to keep the NVLink store queues full, few enough not to crowd out the SpMM running beside it
    const long long items = a.nrows * (f / vw);
    const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>((items + 255) / 256, 4LL * p->num_sms));
    if (vw == 4) put_rows_kernel<4><<<grid, 256, 0, st>>>(a);
    else put_rows_kernel<1><<<grid, 256, 0, st>>>(a);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

int p2p_wait(pgcn_plan* p, int src, cudaStream_t st)
{
    p2p_wait_kernel<<<1, 32, 0, st>>>(flag_slot(p->arena, p->off_flags, src), p->d_epoch);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// Start of a fused call over the peer transport: advance the device epoch on the caller's stream, ahead of every kernel
// of the call (the exchange stream joins after it).
int advance_epoch(pgcn_plan* p, cudaStream_t st)
{
    epoch_advance_kernel<<<1, 1, 0, st>>>(p->d_epoch);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// The transport of a multi-rank call at width f, and the slabs its exchanges land in: the peer transport when it is set
// up and the rows are whole 16-byte vectors (its slabs are double-buffered: the _odd twin serves odd exchange epochs),
// else NCCL, which needs pgcn_comm_init, into the plan's own slabs.
struct Transport {
    bool p2p;
    float* halo; const float* halo_odd;       // forward: the halo rows
    float* rrecv; const float* rrecv_odd;     // backward: the partials the peers send back
};

int transport(pgcn_plan* p, int f, Transport* x)
{
    x->p2p = p->p2p && f % 4 == 0;
    if (!x->p2p && !p->comm) return fail(p, PGCN_ERR_STATE, "k=%d: call pgcn_comm_init or pgcn_p2p_import first", p->k);
    x->halo = x->p2p ? arena_ptr(p->arena, p->off_fwd[0]) : p->d_halo_slab;
    x->halo_odd = x->p2p ? arena_ptr(p->arena, p->off_fwd[1]) : nullptr;
    x->rrecv = x->p2p ? arena_ptr(p->arena, p->off_bwd[0]) : p->d_rrecv_slab;
    x->rrecv_odd = x->p2p ? arena_ptr(p->arena, p->off_bwd[1]) : nullptr;
    return 0;
}

// Exchange schedule shared by both transports and both directions: at step i = 1 .. k-1 a rank sends to
// (rank + i) % k and receives from (rank - i) % k — every pair is active exactly once per step, and a receiver
// sees its sources arrive one after the other, so each block can be consumed while the next is in flight.
inline int step_dst(const pgcn_plan* p, int i) { return (p->rank + i) % p->k; }
inline int step_src(const pgcn_plan* p, int i) { return (p->rank - i + p->k) % p->k; }

int nccl_step(pgcn_plan* p, const float* send, float* recv, int f, int reverse, int i, cudaStream_t st)
{
    const std::vector<int64_t>& so = reverse ? p->recv_off : p->send_off;
    const std::vector<int64_t>& ro = reverse ? p->send_off : p->recv_off;
    const int d = step_dst(p, i), s = step_src(p, i);
    const int64_t ns = so[d + 1] - so[d], nr = ro[s + 1] - ro[s];
    if (ns == 0 && nr == 0) return 0;
    NC(p, g_nccl.GroupStart());
    if (ns > 0) NC(p, g_nccl.Send(send + (size_t)so[d] * f, (size_t)ns * f, ncclFloat_, d, p->comm, st));
    if (nr > 0) NC(p, g_nccl.Recv(recv + (size_t)ro[s] * f, (size_t)nr * f, ncclFloat_, s, p->comm, st));
    NC(p, g_nccl.GroupEnd());
    return 0;
}

// Send half of the forward exchange, shared by pgcn_forward and the unsplit forward: the owned rows leave for every peer
// in step order. Peer transport: the device epoch advances on `st` (every call of the plan that exchanges does this
// once, which is what picks the slab parity) and the rows are stored into each peer's slab of the new parity. NCCL: they
// are packed and sent, and each source's block is received into the halo slab. With `split` the sends run on the
// exchange stream, after `st`'s earlier work; ev_step[i] (NCCL) and ev_b (peer transport) mark their progress.
int forward_send(pgcn_plan* p, const float* H_own, int f, bool use_p2p, bool split, cudaStream_t st)
{
    int rc;
    if (use_p2p && (rc = advance_epoch(p, st))) return rc;
    cudaStream_t cs = split ? p->comm_stream : st;
    if (split) {
        CU(p, cudaEventRecord(p->ev_a, st));
        CU(p, cudaStreamWaitEvent(cs, p->ev_a, 0));
    }
    if (use_p2p) {
        for (int i = 1; i < p->k; ++i)
            if ((rc = p2p_put(p, step_dst(p, i), H_own, f, false, cs))) return rc;
        if (split) CU(p, cudaEventRecord(p->ev_b, cs));                   // H_own is free for the caller after this
    } else {
        if ((rc = launch_pack(p, H_own, p->d_send_slab, f, cs))) return rc;
        for (int i = 1; i < p->k; ++i) {
            if ((rc = nccl_step(p, p->d_send_slab, p->d_halo_slab, f, 0, i, cs))) return rc;
            if (split) CU(p, cudaEventRecord(p->ev_step[(size_t)i], cs));
        }
    }
    return 0;
}

// Peer transport: `st` waits for every source's rows (NCCL receives on the stream that needs them).
int p2p_wait_all(pgcn_plan* p, cudaStream_t st)
{
    int rc;
    for (int i = 1; i < p->k; ++i)
        if ((rc = p2p_wait(p, step_src(p, i), st))) return rc;
    return 0;
}

// Copy the halo rows (h x f) the last forward exchange delivered into dst; halo_odd: the peer transport's odd-epoch twin
// of the slab, picked from the device epoch. Nothing to copy on one rank, without halo rows or without dst.
int copy_halo(pgcn_plan* p, const float* halo, const float* halo_odd, float* dst, int f, cudaStream_t st)
{
    if (p->k == 1 || p->h == 0 || !dst) return 0;
    const long long n = (long long)p->h * f;
    copy_halo_kernel<<<grid_for(n, p->num_sms), 256, 0, st>>>(halo, halo_odd, halo_odd ? p->d_epoch : nullptr, dst, n);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// The unsplit forward exchange (pgcn_forward without its per-source overlap, both transports): every source's rows have
// landed before launch(halo, halo_odd) runs on `st`. halo is the slab the rows land in, halo_odd its odd-epoch twin on
// the peer transport (else null); on one rank there is no exchange.
template <class Launch>
int unsplit_forward(pgcn_plan* p, const float* H_own, int f, cudaStream_t st, Launch launch)
{
    if (p->k == 1) return launch(p->d_halo_slab, (const float*)nullptr);
    Transport x;
    int rc;
    if ((rc = transport(p, f, &x)) || (rc = forward_send(p, H_own, f, x.p2p, false, st))) return rc;
    if (x.p2p && (rc = p2p_wait_all(p, st))) return rc;
    return launch(x.halo, x.halo_odd);
}

// The unsplit backward exchange (pgcn_backward without its per-peer pipelining): launch() writes the rows of A^T gZ,
// [0, m) into G_own and the halo partials into the reverse send slab; they go back to their owners and every rank adds
// what it receives into G_own in a fixed order.
template <class Launch>
int unsplit_backward(pgcn_plan* p, float* G_own, int f, cudaStream_t st, Launch launch)
{
    if (p->k == 1) return launch();
    Transport x;
    int rc;
    if ((rc = transport(p, f, &x))) return rc;
    if (x.p2p && (rc = advance_epoch(p, st))) return rc;
    if ((rc = launch())) return rc;
    for (int i = 1; i < p->k; ++i) {
        if (x.p2p) { if ((rc = p2p_put(p, step_dst(p, i), p->d_hsend_slab, f, true, st))) return rc; }
        else if ((rc = nccl_step(p, p->d_hsend_slab, x.rrecv, f, 1, i, st))) return rc;
    }
    if (x.p2p && (rc = p2p_wait_all(p, st))) return rc;
    return launch_unpack(p, x.rrecv, G_own, f, st, x.rrecv_odd);
}

}  // namespace

// ==========================================================================================
// C ABI
// ==========================================================================================
extern "C" {

const char* pgcn_version(void) { return "pgcn_b200 0.1 (sm_90a, CSR row-block SpMM + halo exchange)"; }

int pgcn_device_count(void)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(nullptr, PGCN_ERR_NOGPU, "cudaGetDeviceCount: %s", cudaGetErrorString(e)); }
    return n;
}

const char* pgcn_last_error(const pgcn_plan* plan) { return plan ? plan->err.c_str() : g_lib_error.c_str(); }

int pgcn_plan_create(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                     int32_t m, int32_t h,
                     const int32_t* t_rowptr, const int32_t* t_colidx, const float* t_vals,
                     const int32_t* send_idx, const int64_t* send_off, const int64_t* recv_off,
                     int32_t k, int32_t rank, int32_t f_max, pgcn_plan** out)
{
    if (!out) return fail(nullptr, PGCN_ERR_INVALID, "out is null");
    *out = nullptr;
    if (!rowptr || !t_rowptr || !send_off || !recv_off) return fail(nullptr, PGCN_ERR_INVALID, "null index array");
    if ((int64_t)m + h >= (int64_t)kColMask) return fail(nullptr, PGCN_ERR_INVALID, "m + h must be below 2^30");
    if (m < 0 || h < 0 || k < 1 || rank < 0 || rank >= k || f_max < 1)
        return fail(nullptr, PGCN_ERR_INVALID, "bad sizes m=%d h=%d k=%d rank=%d f_max=%d", m, h, k, rank, f_max);
    if (recv_off[k] != h) return fail(nullptr, PGCN_ERR_INVALID, "recv_off[k]=%lld != h=%d", (long long)recv_off[k], h);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(nullptr, PGCN_ERR_NOGPU, "no CUDA device: the PGCN GPU path has no CPU fallback");
    }
    const int64_t nnz = rowptr[m];
    if (nnz > 0 && (!colidx || !vals || !t_colidx || !t_vals)) return fail(nullptr, PGCN_ERR_INVALID, "null colidx/vals");
    if (t_rowptr[m + h] != nnz) return fail(nullptr, PGCN_ERR_INVALID, "transpose nnz mismatch");
    for (int64_t e = 0; e < nnz; ++e) {
        if (colidx[e] < 0 || colidx[e] >= m + h) return fail(nullptr, PGCN_ERR_INVALID, "colidx[%lld]=%d out of [0,%d)", (long long)e, colidx[e], m + h);
        if (t_colidx[e] < 0 || t_colidx[e] >= m) return fail(nullptr, PGCN_ERR_INVALID, "t_colidx[%lld]=%d out of [0,%d)", (long long)e, t_colidx[e], m);
    }
    const int64_t S = send_off[k];
    for (int64_t j = 0; j < S; ++j)
        if (!send_idx || send_idx[j] < 0 || send_idx[j] >= m) return fail(nullptr, PGCN_ERR_INVALID, "send_idx[%lld] out of range", (long long)j);

    pgcn_plan* p = new pgcn_plan();
    p->m = m; p->h = h; p->k = k; p->rank = rank; p->f_max = f_max; p->S = S;
    p->send_off.assign(send_off, send_off + k + 1);
    p->recv_off.assign(recv_off, recv_off + k + 1);
    cudaGetDevice(&p->device);

#define TRY(expr) do { int rc__ = (expr); if (rc__) { g_lib_error = p->err; pgcn_plan_destroy(p); return rc__; } } while (0)
    // column reference counts: forward columns = rows of the transpose and vice versa
    std::vector<int> refs_fwd((size_t)m + h), refs_tr((size_t)m);
    for (int r = 0; r < m + h; ++r) refs_fwd[r] = t_rowptr[r + 1] - t_rowptr[r];
    for (int r = 0; r < m; ++r) refs_tr[r] = rowptr[r + 1] - rowptr[r];
    // rows of H kept hot in L2: about half of the H100's 50 MB L2, the rest is left to the streams
    if (const char* e = getenv("PGCN_HOT_MB")) p->opt_hot_mb = std::max<long long>(0, atoll(e));   // tuning knob
    // Two hot sets: one for full-width rows (f_max floats) and one for 64-float slices, which holds as many more rows
    // as the slice is narrower (the ring kernel gathers one slice of every row before the next slice).
    auto cold_threshold = [&](const std::vector<int>& refs, int64_t row_bytes) -> int {
        const int64_t hot_rows = std::max<int64_t>(1, (p->opt_hot_mb << 20) / row_bytes);
        const int64_t ncols = (int64_t)refs.size();
        if (ncols <= hot_rows) return -1;                  // everything fits: nothing is cold
        std::vector<int> sorted(refs);
        std::nth_element(sorted.begin(), sorted.begin() + (ncols - hot_rows), sorted.end());
        return sorted[ncols - hot_rows];
    };
    const int64_t full_bytes = (int64_t)f_max * 4, slice_bytes = std::min<int64_t>(full_bytes, 64 * 4);
    const int cold_fwd[2] = {cold_threshold(refs_fwd, full_bytes), cold_threshold(refs_fwd, slice_bytes)};
    const int cold_tr[2] = {cold_threshold(refs_tr, full_bytes), cold_threshold(refs_tr, slice_bytes)};
    TRY(csr_upload(p, p->fwd, m, rowptr, colidx, vals, nullptr, refs_fwd.data(), cold_fwd));
    TRY(csr_upload(p, p->tr, m + h, t_rowptr, t_colidx, t_vals, nullptr, refs_tr.data(), cold_tr, true));

    // distinct referenced columns / transposed rows (for the roofline's compulsory bytes)
    for (int r = 0; r < m + h; ++r) if (t_rowptr[r + 1] > t_rowptr[r]) ++p->cols_ref;
    p->rows_ref_t = 0;
    for (int r = 0; r < m; ++r) if (rowptr[r + 1] > rowptr[r]) ++p->rows_ref_t;

    // split A_local = [A_own | A_halo(peer) ...] (Parallel-GCN/main.c:271 then :295 per received block) so that
    // A_own * H_own overlaps the exchange and each peer's block is accumulated as soon as it has landed
    if (h > 0 && k > 1) {
        std::vector<int> o_rp(m + 1, 0), o_ci; std::vector<float> o_v;
        o_ci.reserve(nnz); o_v.reserve(nnz);
        std::vector<std::vector<int>> q_rp((size_t)k, std::vector<int>(1, 0)), q_ci((size_t)k), q_map((size_t)k);
        std::vector<std::vector<float>> q_v((size_t)k);
        std::vector<int> col_peer((size_t)h);
        for (int q = 0; q < k; ++q)
            for (int64_t c = recv_off[q]; c < recv_off[q + 1]; ++c) col_peer[(size_t)c] = q;
        std::vector<char> touched((size_t)k, 0);
        for (int r = 0; r < m; ++r) {
            for (int e = rowptr[r]; e < rowptr[r + 1]; ++e) {
                if (colidx[e] < m) { o_ci.push_back(colidx[e]); o_v.push_back(vals[e]); }
                else {
                    const int q = col_peer[(size_t)(colidx[e] - m)];
                    q_ci[q].push_back(colidx[e] - m);                    // slab-relative column
                    q_v[q].push_back(vals[e]);
                    touched[q] = 1;
                }
            }
            o_rp[r + 1] = (int)o_ci.size();
            for (int q = 0; q < k; ++q)
                if (touched[q]) { q_map[q].push_back(r); q_rp[q].push_back((int)q_ci[q].size()); touched[q] = 0; }
        }
        TRY(csr_upload(p, p->own, m, o_rp.data(), o_ci.data(), o_v.data(), nullptr, refs_fwd.data(), cold_fwd, true));
        p->halo_q.resize((size_t)k);
        for (int q = 0; q < k; ++q) {
            if (q_map[q].empty()) continue;
            TRY(csr_upload(p, p->halo_q[q], (int)q_map[q].size(), q_rp[q].data(), q_ci[q].data(), q_v[q].data(), &q_map[q],
                           refs_fwd.data() + m, cold_fwd));
        }
        // fused ReLU epilogue: a row is clamped by the launch of the pipelined forward that writes it last — the
        // own-columns launch for rows without halo entries, else the last peer block (in this rank's step order)
        {
            std::vector<int> last_step((size_t)m, 0);
            for (int i = 1; i < k; ++i) {
                const int src = (rank - i + k) % k;
                for (int r : q_map[src]) last_step[(size_t)r] = i;
            }
            std::vector<unsigned char> fin;
            fin.resize((size_t)std::max(p->own.nrows_c, 1));
            for (int c = 0; c < p->own.nrows_c; ++c) {
                const int r = p->own.d_rowids ? p->own.h_rowids[(size_t)c] : c;
                fin[(size_t)c] = last_step[(size_t)r] == 0;
            }
            TRY(upload(p, &p->own.d_final, fin.data(), fin.size()));
            for (int i = 1; i < k; ++i) {
                const int src = (rank - i + k) % k;
                if (q_map[src].empty()) continue;
                fin.resize(q_map[src].size());
                for (size_t j = 0; j < q_map[src].size(); ++j) fin[j] = last_step[(size_t)q_map[src][j]] == i;
                TRY(upload(p, &p->halo_q[(size_t)src].d_final, fin.data(), fin.size()));
            }
        }
        csr_view(p->tr, p->tr_own, 0, m);
        p->tr_halo_q.resize((size_t)k);
        for (int q = 0; q < k; ++q)
            if (recv_off[q + 1] > recv_off[q]) csr_view(p->tr, p->tr_halo_q[q], m + (int)recv_off[q], m + (int)recv_off[q + 1]);
        p->have_split = true;
    }

    {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, p->device) == cudaSuccess) p->num_sms = prop.multiProcessorCount;
        std::vector<unsigned int> zeros(64, 0u);
        TRY(upload(p, &p->d_counter, zeros.data(), zeros.size()));
        TRY(upload(p, &p->d_done, zeros.data(), zeros.size()));
        const unsigned long long epoch0 = 0;
        TRY(upload(p, &p->d_epoch, &epoch0, 1));
    }
    TRY(upload(p, &p->d_send_idx, send_idx, (size_t)S));
    // boundary CSR: for every owned row that appears in some send list, the slab positions
    {
        std::vector<std::pair<int, int>> pr((size_t)S);
        for (int64_t j = 0; j < S; ++j) pr[j] = std::make_pair(send_idx[j], (int)j);
        std::stable_sort(pr.begin(), pr.end(), [](const std::pair<int,int>& a, const std::pair<int,int>& b) { return a.first < b.first; });
        std::vector<int> brow, bptr(1, 0), bpos((size_t)S);
        for (int64_t j = 0; j < S; ++j) {
            if (j == 0 || pr[j].first != pr[j - 1].first) { if (j) bptr.push_back((int)j); brow.push_back(pr[j].first); }
            bpos[j] = pr[j].second;
        }
        if (S) bptr.push_back((int)S);
        p->nb = (int)brow.size();
        TRY(upload(p, &p->d_brow, brow.data(), brow.size()));
        TRY(upload(p, &p->d_bptr, bptr.data(), bptr.size()));
        TRY(upload(p, &p->d_bpos, bpos.data(), bpos.size()));
    }
    auto slab = [&](float** d, int64_t rows) -> int {
        CU(p, cudaMalloc((void**)d, std::max<size_t>((size_t)rows * f_max, 1) * sizeof(float)));
        return 0;
    };
    TRY(slab(&p->d_send_slab, S));
    TRY(slab(&p->d_halo_slab, h));
    TRY(slab(&p->d_rrecv_slab, S));
    TRY(slab(&p->d_hsend_slab, h));
    {
        // the exchange stream outranks the compute stream: its (small) kernels must get SM slots while an SpMM
        // grid is draining, because a neighbour is waiting for their stores
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        cudaError_t e1 = cudaStreamCreateWithPriority(&p->comm_stream, cudaStreamNonBlocking, prio_hi);
        if (e1 == cudaSuccess) e1 = cudaStreamCreateWithFlags(&p->host_stream, cudaStreamNonBlocking);
        cudaError_t e2 = cudaEventCreateWithFlags(&p->ev_a, cudaEventDisableTiming);
        cudaError_t e3 = cudaEventCreateWithFlags(&p->ev_b, cudaEventDisableTiming);
        p->ev_step.assign((size_t)k, nullptr);
        for (int q = 0; q < k && e3 == cudaSuccess; ++q) e3 = cudaEventCreateWithFlags(&p->ev_step[(size_t)q], cudaEventDisableTiming);
        if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) {
            fail(p, PGCN_ERR_CUDA, "stream/event creation failed");
            g_lib_error = p->err; pgcn_plan_destroy(p); return PGCN_ERR_CUDA;
        }
    }
#undef TRY
    *out = p;
    return 0;
}

int pgcn_plan_destroy(pgcn_plan* p)
{
    if (!p) return 0;
    cudaSetDevice(p->device);
    cudaDeviceSynchronize();
    if (p->comm && g_nccl.ok && !p->comm_borrowed) g_nccl.CommDestroy(p->comm);
    for (int q = 0; q < kMaxPeers; ++q)
        if (p->peer_arena[q] && q != p->rank && !p->peer_local[q]) cudaIpcCloseMemHandle(p->peer_arena[q]);
    cudaFree(p->arena);
    csr_free(p->tr_own);
    for (auto& c : p->tr_halo_q) csr_free(c);
    for (auto& c : p->halo_q) csr_free(c);
    csr_free(p->fwd); csr_free(p->tr); csr_free(p->own);
    for (cudaEvent_t e : p->ev_step) if (e) cudaEventDestroy(e);
    cudaFree(p->d_done);
    cudaFree(p->d_send_idx);
    cudaFree(p->d_brow); cudaFree(p->d_bptr); cudaFree(p->d_bpos);
    cudaFree(p->d_send_slab); cudaFree(p->d_halo_slab); cudaFree(p->d_rrecv_slab); cudaFree(p->d_hsend_slab);
    for (int i = 0; i < 2; ++i) {
        cudaFree(p->d_hostH[i]); cudaFree(p->d_hostZ[i]);
        if (p->ev_in[i]) cudaEventDestroy(p->ev_in[i]);
        if (p->ev_comp[i]) cudaEventDestroy(p->ev_comp[i]);
        if (p->ev_out[i]) cudaEventDestroy(p->ev_out[i]);
    }
    if (p->s_in) cudaStreamDestroy(p->s_in);
    if (p->s_out) cudaStreamDestroy(p->s_out);
    cudaFree(p->d_counter);
    cudaFree(p->d_epoch);
    cudaFree(p->d_vals0); cudaFree(p->d_vsets); cudaFree(p->d_rowptr); cudaFree(p->d_long_rows);
    for (void* q : p->retired) cudaFree(q);
    if (p->comm_stream) cudaStreamDestroy(p->comm_stream);
    if (p->host_stream) cudaStreamDestroy(p->host_stream);
    if (p->ev_a) cudaEventDestroy(p->ev_a);
    if (p->ev_b) cudaEventDestroy(p->ev_b);
    cudaGetLastError();
    delete p;
    return 0;
}

int pgcn_plan_set_option(pgcn_plan* p, const char* name, int64_t value)
{
    if (!p || !name) return fail(p, PGCN_ERR_INVALID, "null argument");
    const std::string n(name);
    if (n == "edges_per_block" || n == "ring_edges_per_block" || n == "ring_slots")   // explicit beats tuned
        for (DevCsr* c : plan_matrices(p)) {
            c->tuned_epb[0] = c->tuned_epb[1] = 0; c->tuned_slots = 0; c->tuned_tile = 0;
        }
    if (n == "edges_per_block") p->opt_epb = value;
    else if (n == "kernel") p->opt_kernel = value;
    else if (n == "ring_slots") p->opt_ring_slots = value;
    else if (n == "ring_edges_per_block") p->opt_ring_epb = value;
    else if (n == "ring_long_row") p->opt_ring_long = value;
    else if (n == "persistent") p->opt_persistent = value;
    else if (n == "persistent_multi") p->opt_persistent_multi = value;
    else if (n == "ring_groups") p->opt_ring_groups = value;
    else if (n == "ring_tile_floats") {
        if (value != 0 && value != 64 && value != 128 && value != 256)
            return fail(p, PGCN_ERR_INVALID, "ring_tile_floats must be 0 (tuned), 64, 128 or 256, not %lld", (long long)value);
        p->opt_ring_tile = value;
    }
    else if (n == "long_row") p->opt_long = value;
    else if (n == "tile_floats") p->opt_tile = value;
    else if (n == "hot_mb")
        // the cold-column marks are baked into the pair arrays at pgcn_plan_create: a later change would be a
        // silent no-op, so it is refused (use the PGCN_HOT_MB environment variable before creating the plan)
        return fail(p, PGCN_ERR_STATE, "hot_mb is fixed at plan creation (set PGCN_HOT_MB before pgcn_plan_create)");
    else if (n == "overlap") p->opt_overlap = value;
    else if (n == "relu") p->opt_relu = value ? 1 : 0;
    else if (n == "p2p") {
        // 0 = never use the peer transport even though pgcn_p2p_import succeeded here (another rank could not map
        // its peers: every rank must then fall back to NCCL together); 1 re-enables it when the arenas are mapped.
        p->opt_p2p = value ? 1 : 0;
        p->p2p = p->opt_p2p && p->arena && p->peer_arena[p->rank];
    }
    else return fail(p, PGCN_ERR_INVALID, "unknown option '%s'", name);
    return 0;
}

int64_t pgcn_plan_get_option(const pgcn_plan* p, const char* name)
{
    if (!p || !name) return PGCN_ERR_INVALID;
    const std::string n(name);
    if (n == "edges_per_block") return p->fwd.tuned_epb[0] > 0 ? p->fwd.tuned_epb[0] : p->opt_epb;
    if (n == "kernel") return p->opt_kernel;
    if (n == "ring_slots") return p->fwd.tuned_slots > 0 ? p->fwd.tuned_slots : p->opt_ring_slots;
    if (n == "ring_edges_per_block") return p->fwd.tuned_epb[1] > 0 ? p->fwd.tuned_epb[1] : p->opt_ring_epb;
    if (n == "ring_long_row") return p->opt_ring_long;
    if (n == "persistent") return p->opt_persistent;
    if (n == "persistent_multi") return p->opt_persistent_multi;
    if (n == "ring_groups") return p->opt_ring_groups;
    if (n == "ring_tile_floats") return p->opt_ring_tile > 0 ? p->opt_ring_tile : p->fwd.tuned_tile;
    if (n == "long_row") return p->opt_long;
    if (n == "tile_floats") return p->opt_tile;
    if (n == "hot_mb") return p->opt_hot_mb;
    if (n == "overlap") return p->opt_overlap;
    if (n == "relu") return p->opt_relu;
    if (n == "p2p") return p->p2p ? 1 : 0;
    if (n == "nccl") return p->comm ? 1 : 0;
    if (n == "blocks_fwd") return p->fwd.sched[0].nblocks;
    if (n == "long_rows_fwd") return p->fwd.sched[0].nlong;
    if (n == "ring_blocks_fwd") return p->fwd.sched[1].nblocks;
    if (n == "ring_long_rows_fwd") return p->fwd.sched[1].nlong;
    if (n == "retired_schedules") return p->nretired;
    if (n == "epoch") {                                   // synchronous read (tests); not while a stream is captured
        unsigned long long e = 0;
        if (cudaMemcpy(&e, p->d_epoch, sizeof e, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); return PGCN_ERR_CUDA; }
        return (int64_t)e;
    }
    return PGCN_ERR_INVALID;
}

int64_t pgcn_debug_schedule(const int32_t* rowptr, int32_t nrows, int64_t edges_per_block, int64_t long_row,
                            int32_t* blocks_out, int64_t cap_blocks, int32_t* nlong_out, int32_t* nslots_out)
{
    if (!rowptr || nrows < 0 || edges_per_block < 8) return fail(nullptr, PGCN_ERR_INVALID, "bad schedule arguments");
    std::vector<int4> blocks, longs;
    int nslots = 0;
    make_schedule(rowptr, nrows, edges_per_block, long_row > 0 ? long_row : 4 * edges_per_block, blocks, longs, nslots);
    if (nlong_out) *nlong_out = (int32_t)longs.size();
    if (nslots_out) *nslots_out = nslots;
    if (blocks_out) {
        const int64_t n = std::min<int64_t>((int64_t)blocks.size(), cap_blocks);
        for (int64_t i = 0; i < n; ++i) {
            blocks_out[4 * i] = blocks[i].x; blocks_out[4 * i + 1] = blocks[i].y;
            blocks_out[4 * i + 2] = blocks[i].z; blocks_out[4 * i + 3] = blocks[i].w;
        }
    }
    return (int64_t)blocks.size();
}

// Scratch features for the autotune: values in [-1, 1) from an integer hash. All-zero operands move the same bytes
// but cost less energy, so a power-limited card runs them at higher clocks than real features.
__global__ void fill_hash_kernel(float* x, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t h = (uint32_t)i * 0x9e3779b1u;
        h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13;
        x[i] = (float)(h >> 8) * (2.0f / 16777216.0f) - 1.0f;
    }
}

// Autotune: every matrix of the plan (forward, transposed, and — for k > 1 — the own-column part, each peer's halo
// block and the transposed row ranges the pipelined backward launches) gets its own schedule parameters, timed on
// zero-filled scratch operands of the right shapes. Returns the edges-per-block chosen for the forward matrix.
int pgcn_plan_autotune(pgcn_plan* p, int32_t f)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->fwd.nnz == 0) return (int)p->opt_epb;
    CU(p, cudaSetDevice(p->device));
    float *H0 = nullptr, *H1 = nullptr, *Z0 = nullptr, *Z1 = nullptr;
    const size_t bm = std::max<size_t>((size_t)p->m * f, 1) * 4, bh = std::max<size_t>((size_t)p->h * f, 1) * 4;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    auto cleanup = [&]() {
        cudaFree(H0); cudaFree(H1); cudaFree(Z0); cudaFree(Z1);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    };
    if (cudaMalloc((void**)&H0, bm) != cudaSuccess || cudaMalloc((void**)&H1, bh) != cudaSuccess ||
        cudaMalloc((void**)&Z0, bm) != cudaSuccess || cudaMalloc((void**)&Z1, bh) != cudaSuccess) {
        cleanup(); cudaGetLastError();
        return fail(p, PGCN_ERR_CUDA, "autotune: scratch allocation failed");
    }
    cudaStream_t st = p->host_stream;
    fill_hash_kernel<<<4 * p->num_sms, 256, 0, st>>>(H0, bm / 4);
    fill_hash_kernel<<<4 * p->num_sms, 256, 0, st>>>(H1, bh / 4);
    cudaMemsetAsync(Z0, 0, bm, st); cudaMemsetAsync(Z1, 0, bh, st);
    cudaEventCreate(&e0); cudaEventCreate(&e1);

    struct Cand { int64_t epb; int slots; };
    // Ring blocks stay at 512 edges (256 and 1024 never won by more than the run-to-run spread). The block size sets
    // how long rows are split, and so the order of their sums: with one block size, Z does not depend on the timing.
    static const Cand ring_cand[] = {{512, 16}, {512, 32}};
    static const Cand reg_cand[] = {{96, 0}, {128, 0}, {144, 0}, {160, 0}, {192, 0}, {256, 0}};
    // one matrix: h0/h1/split = gathered operand(s), z0/z1/zsplit = outputs
    auto tune = [&](DevCsr& c, const float* h0, const float* h1, int split, float* z0, float* z1, int zsplit, int beta) -> int {
        if (c.nnz == 0 || c.nrows == 0) return 0;
        const bool ring = use_ring(p, h0, h1, f);
        const Cand* cand = ring ? ring_cand : reg_cand;
        const int ncand = ring ? (int)(sizeof ring_cand / sizeof ring_cand[0]) : (int)(sizeof reg_cand / sizeof reg_cand[0]);
        const int which = ring ? 1 : 0;
        const int64_t keep_epb = c.tuned_epb[which];
        const int keep_slots = c.tuned_slots, keep_tile = c.tuned_tile;
        // ring row tile: the full width (tuned_tile 0) and 64-float slices, unless the option fixes it
        const int ntile = (ring && p->opt_ring_tile == 0) ? 2 : 1;
        const int npts = ntile * ncand;
        auto select = [&](int j) {
            c.tuned_epb[which] = cand[j % ncand].epb;
            if (ring) { c.tuned_slots = cand[j % ncand].slots; c.tuned_tile = j >= ncand ? 64 : 0; }
        };
        // n launches of point j, timed together (-1 on error)
        auto run = [&](int j, int n) -> float {
            select(j);
            cudaEventRecord(e0, st);
            for (int it = 0; it < n; ++it)
                if (int r2 = launch_spmm(p, c, h0, h1, split, z0, z1, zsplit, f, beta, st)) { rc = r2; return -1.f; }
            cudaEventRecord(e1, st);
            if (cudaEventSynchronize(e1) != cudaSuccess) { rc = fail(p, PGCN_ERR_CUDA, "autotune: kernel failed"); return -1.f; }
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0, e1);
            return ms / n;
        };
        // A power-limited card lowers its clocks after a few milliseconds of load, and which point is fastest can
        // change with the clock. So: build every schedule, keep the card busy until clocks settle, then time the
        // points in interleaved rounds and keep the lowest median.
        constexpr int kRounds = 7, kLaunches = 4;
        std::vector<float> t((size_t)npts * kRounds);
        bool ok = true;
        for (int j = 0; j < npts && ok; ++j) ok = run(j, 1) >= 0.f;
        float warm = 0.f;                                    // about 100 ms of launches (at most 200 timed runs)
        for (int i = 0; i < 200 && ok && warm < 100.f; ++i) { const float ms = run(i % npts, 2); ok = ms >= 0.f; warm += 2 * ms; }
        for (int r = 0; r < kRounds && ok; ++r)
            for (int j = 0; j < npts && ok; ++j) { t[(size_t)j * kRounds + r] = run(j, kLaunches); ok = t[(size_t)j * kRounds + r] >= 0.f; }
        if (!ok) {
            c.tuned_epb[which] = keep_epb; c.tuned_slots = keep_slots; c.tuned_tile = keep_tile;
            return rc;
        }
        int best = 0;
        float best_ms = 1e30f;
        for (int j = 0; j < npts; ++j) {
            std::nth_element(t.begin() + (size_t)j * kRounds, t.begin() + (size_t)j * kRounds + kRounds / 2, t.begin() + (size_t)(j + 1) * kRounds);
            const float med = t[(size_t)j * kRounds + kRounds / 2];
            if (med < best_ms) { best_ms = med; best = j; }
        }
        select(best);
        return 0;
    };
#define TUNE(...) do { if ((rc = tune(__VA_ARGS__))) { cleanup(); return rc; } } while (0)
    TUNE(p->fwd, H0, p->h ? H1 : nullptr, p->m, Z0, nullptr, p->m, 0);
    TUNE(p->tr, H0, nullptr, p->m, Z0, Z1, p->m, 0);
    if (p->have_split) {
        TUNE(p->own, H0, nullptr, p->m, Z0, nullptr, p->m, 0);
        TUNE(p->tr_own, H0, nullptr, p->m, Z0, Z1, p->m, 0);
        for (int q = 0; q < p->k; ++q) {
            TUNE(p->halo_q[(size_t)q], H1, nullptr, p->h, Z0, nullptr, p->m, 1);
            TUNE(p->tr_halo_q[(size_t)q], H0, nullptr, p->m, Z0, Z1, p->m, 0);
        }
    }
#undef TUNE
    cleanup();
    const int which = use_ring(p, H0, nullptr, f) ? 1 : 0;     // H0 was cudaMalloc'ed: aligned
    return (int)(p->fwd.tuned_epb[which] > 0 ? p->fwd.tuned_epb[which] : (which ? p->opt_ring_epb : p->opt_epb));
}

// Everything a fused forward / backward at width f would otherwise set up on its first call: the schedules of every
// matrix those calls launch, for the register kernel and (f a multiple of 128: the operands' alignment decides at
// run time) the ring kernel; the shared-memory opt-in and occupancy of every ring instance; the kernel modules.
int pgcn_plan_prepare(pgcn_plan* p, int32_t f)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    CU(p, cudaSetDevice(p->device));
    preload_kernels();
    cudaStream_t st = p->host_stream;
    const bool ring = p->opt_kernel != 4 && f % 128 == 0;
    DevCsr::Sched* sc;
    for (DevCsr* c : plan_matrices(p))
        if (c->nrows > 0 && ((rc = schedule(p, *c, false, st, &sc)) || (ring && (rc = schedule(p, *c, true, st, &sc)))))
            return rc;
    auto ring_opt_in = [&](const RingInst& ri) { return opt_in(p, ri.fn, ri.smem, ri.warps * 32, st, nullptr); };
    if (ring && (rc = for_each_ring(ring_opt_in))) return rc;
    // the ring instances of the edge calls at width f (they walk the forward matrix's schedules, built above)
    auto edge_opt_in = [&](const void* fn) {
        return opt_in(p, fn, sddmm_smem_bytes(f / 128), kSddmmWarps * 32, st, nullptr);
    };
    // pgcn_sddmm
    if (ring && f <= 512 && (rc = edge_opt_in((const void*)pick_sddmm(f / 128)))) return rc;
    // the multi-head SDDMM
    if (ring && (f == 128 || f == 256 || f == 512))
        for (int k = 2; k <= 8; k *= 2)
            if ((f / k) % 4 == 0 && (rc = edge_opt_in((const void*)pick_sddmm_heads(f / 128, k)))) return rc;
    // the max calls of a bound plan: the register schedules (built above) and the entries of the forward's split rows
    if (p->bound && (rc = max_partial(p, p->fwd.sched[0], st))) return rc;
    // the GATv2 calls: the score ring instances of width f and the datt partials of a bound plan
    if (ring && (f == 128 || f == 256))
        for (int k = 1; k <= 8; k *= 2)
            if ((rc = edge_opt_in((const void*)pick_gatv2_ring(f / 128, k)))) return rc;
    if (p->bound && (rc = gatv2_partial(p, p->fwd.sched[0], st))) return rc;
    p->prepared = true;
    return 0;
}

int pgcn_plan_bind_values(pgcn_plan* p)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (p->bound) return 0;
    CU(p, cudaSetDevice(p->device));
    const int64_t nnz = p->fwd.nnz;
    const int64_t ncol = (int64_t)p->m + p->h;
    std::vector<int> fcol, fval, frow, tcol, tval, trow;
    int rc;
    if ((rc = decode_records(p, p->fwd, fcol, fval, frow))) return rc;
    if ((rc = decode_records(p, p->tr, tcol, tval, trow))) return rc;
    if (p->tr.nnz != nnz) return fail(p, PGCN_ERR_INVALID, "transposed CSR holds %lld entries, the forward CSR %lld",
                                      (long long)p->tr.nnz, (long long)nnz);
    // forward entries in (column, row) order: a stable counting sort by column of the row-major entries (duplicates
    // keep their order of appearance)
    std::vector<int64_t> cstart((size_t)ncol + 1, 0);
    for (int64_t e = 0; e < nnz; ++e) ++cstart[(size_t)fcol[(size_t)e] + 1];
    for (int64_t c = 0; c < ncol; ++c) cstart[(size_t)c + 1] += cstart[(size_t)c];
    std::vector<int> fsorted((size_t)nnz);
    {
        std::vector<int64_t> pos(cstart.begin(), cstart.end() - 1);
        for (int64_t e = 0; e < nnz; ++e) fsorted[(size_t)pos[(size_t)fcol[(size_t)e]]++] = (int)e;
    }
    // transposed entries: row-major over the forward columns already; order each row by forward row (stable)
    std::vector<int> tsorted((size_t)nnz);
    for (int64_t e = 0; e < nnz; ++e) tsorted[(size_t)e] = (int)e;
    for (int64_t s = 0; s < nnz;) {
        int64_t t = s + 1;
        while (t < nnz && trow[(size_t)t] == trow[(size_t)s]) ++t;
        std::stable_sort(tsorted.begin() + s, tsorted.begin() + t, [&](int x, int y) { return tcol[(size_t)x] < tcol[(size_t)y]; });
        s = t;
    }
    std::vector<int> tmap((size_t)nnz);
    for (int64_t i = 0; i < nnz; ++i) {
        const int fe = fsorted[(size_t)i], te = tsorted[(size_t)i];
        if (fcol[(size_t)fe] != trow[(size_t)te] || frow[(size_t)fe] != tcol[(size_t)te])
            return fail(p, PGCN_ERR_INVALID, "the transposed CSR does not hold the forward entries: transposed entry %d (row %d, "
                        "column %d) has no forward entry (row %d, column %d) to match", te, trow[(size_t)te], tcol[(size_t)te],
                        tcol[(size_t)te], trow[(size_t)te]);
        if (fval[(size_t)fe] != tval[(size_t)te])
            return fail(p, PGCN_ERR_INVALID, "transposed entry %d (row %d, column %d) has another value than its forward entry %d",
                        te, trow[(size_t)te], tcol[(size_t)te], fe);
        tmap[(size_t)te] = fe;
    }
    // own-column and per-peer blocks: the forward entries in forward order, split by column (as pgcn_plan_create did)
    std::vector<int> omap;
    std::vector<std::vector<int>> qmap;
    if (p->have_split) {
        std::vector<int> col_peer((size_t)p->h);
        for (int q = 0; q < p->k; ++q)
            for (int64_t c = p->recv_off[(size_t)q]; c < p->recv_off[(size_t)q + 1]; ++c) col_peer[(size_t)c] = q;
        qmap.resize((size_t)p->k);
        for (int64_t e = 0; e < nnz; ++e) {
            const int c = fcol[(size_t)e];
            if (c < p->m) omap.push_back((int)e);
            else qmap[(size_t)col_peer[(size_t)(c - p->m)]].push_back((int)e);
        }
        if ((int64_t)omap.size() != p->own.nnz) return fail(p, PGCN_ERR_STATE, "own-column block does not match the forward CSR");
        for (int q = 0; q < p->k; ++q)
            if ((int64_t)qmap[(size_t)q].size() != p->halo_q[(size_t)q].nnz)
                return fail(p, PGCN_ERR_STATE, "halo block of peer %d does not match the forward CSR", q);
    }
    // device side: maps, creation values, the set table of the rewrite kernel
    std::vector<ValueSet> sets;
    long long total = 0;
    auto add = [&](DevCsr& c, const std::vector<int>* map) -> int {
        if (c.nnz == 0) return 0;
        if (map) { int r2 = upload_setup(p, &c.d_vmap, map->data(), map->size()); if (r2) return r2; }
        ValueSet s;
        s.cw = c.d_cw; s.map = map ? c.d_vmap : nullptr; s.nnz = c.nnz; s.start = total;
        total += c.nnz;
        sets.push_back(s);
        return 0;
    };
    if ((rc = add(p->fwd, nullptr))) return rc;
    if ((rc = add(p->tr, &tmap))) return rc;
    if (p->have_split) {
        if ((rc = add(p->own, &omap))) return rc;
        for (int q = 0; q < p->k; ++q)
            if ((rc = add(p->halo_q[(size_t)q], &qmap[(size_t)q]))) return rc;
    }
    if ((rc = upload_setup(p, &p->d_vals0, reinterpret_cast<const float*>(fval.data()), fval.size()))) return rc;
    if ((rc = upload_setup(p, &p->d_vsets, sets.data(), sets.size()))) return rc;
    // the edge softmax walks the forward rows: their rowptr, and the rows long enough for a CTA each
    std::vector<int> rowptr((size_t)p->m + 1, 0), long_rows;
    for (int64_t e = 0; e < nnz; ++e) ++rowptr[(size_t)frow[(size_t)e] + 1];
    for (int i = 0; i < p->m; ++i) {
        if (rowptr[(size_t)i + 1] > kAttnLongRow) long_rows.push_back(i);
        rowptr[(size_t)i + 1] += rowptr[(size_t)i];
    }
    if ((rc = upload_setup(p, &p->d_rowptr, rowptr.data(), rowptr.size()))) return rc;
    if ((rc = upload_setup(p, &p->d_long_rows, long_rows.data(), long_rows.size()))) return rc;
    p->nlong_rows = (int)long_rows.size();
    p->nvsets = (int)sets.size();
    p->vtotal = total;
    p->bound = true;
    return 0;
}

int pgcn_plan_set_values(pgcn_plan* p, const float* vals, void* stream)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "pgcn_plan_set_values needs the value maps: call pgcn_plan_bind_values first");
    if (p->vtotal == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    set_values_kernel<<<grid_for(p->vtotal, p->num_sms), 256, 0, st>>>(p->d_vsets, p->nvsets, p->vtotal, vals ? vals : p->d_vals0);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

void* pgcn_plan_slab(pgcn_plan* p, int which)
{
    if (!p) return nullptr;
    switch (which) {
        case 0: return p->d_send_slab;
        case 1: return p->d_halo_slab;
        case 2: return p->d_rrecv_slab;
        case 3: return p->d_hsend_slab;
        default: return nullptr;
    }
}

int pgcn_algorithmic_bytes(const pgcn_plan* p, int32_t f, pgcn_bytes* o)
{
    if (!p || !o) return PGCN_ERR_INVALID;
    const int64_t nnz = p->fwd.nnz, m = p->m, h = p->h, S = p->S, F = f;
    o->nnz = nnz; o->m = m; o->h = h; o->cols_ref = p->cols_ref;
    o->spmm_fwd = 8 * nnz + 4 * (m + 1) + 4 * F * p->cols_ref + 4 * F * m;
    o->spmm_bwd = 8 * nnz + 4 * (m + h + 1) + 4 * F * p->rows_ref_t + 4 * F * (m + h);
    o->gather_fwd = nnz * (8 + 4 * F) + 4 * (m + 1) + 4 * F * m;
    o->xchg_out = 4 * F * S;
    o->xchg_in = 4 * F * h;
    o->pack = 2 * 4 * F * S;
    return 0;
}

int64_t pgcn_launch_count(const pgcn_plan* p) { return p ? p->launches : 0; }

// ---- communicator --------------------------------------------------------------------------

int pgcn_comm_unique_id(void* id128)
{
    if (!id128) return fail(nullptr, PGCN_ERR_INVALID, "null id buffer");
    if (!load_nccl()) return fail(nullptr, PGCN_ERR_NCCL, "libnccl.so.2 not found in this process");
    ncclUniqueId id;
    NC(nullptr, g_nccl.GetUniqueId(&id));
    memcpy(id128, &id, sizeof id);
    return 0;
}

int pgcn_comm_init(pgcn_plan* p, const void* id128)
{
    if (!p || !id128) return fail(p, PGCN_ERR_INVALID, "null argument");
    if (!load_nccl()) return fail(p, PGCN_ERR_NCCL, "libnccl.so.2 not found in this process");
    if (p->comm) return 0;
    ncclUniqueId id;
    memcpy(&id, id128, sizeof id);
    CU(p, cudaSetDevice(p->device));
    NC(p, g_nccl.CommInitRank(&p->comm, p->k, id, p->rank));
    return 0;
}

int pgcn_comm_share(pgcn_plan* p, pgcn_plan* owner)
{
    if (!p || !owner) return fail(p, PGCN_ERR_INVALID, "null argument");
    if (!owner->comm) return fail(p, PGCN_ERR_STATE, "the owner plan has no communicator (pgcn_comm_init first)");
    if (p->k != owner->k || p->rank != owner->rank || p->device != owner->device)
        return fail(p, PGCN_ERR_INVALID, "plans of different rank / size / device cannot share a communicator");
    if (p->comm && !p->comm_borrowed) return fail(p, PGCN_ERR_STATE, "plan already owns a communicator");
    p->comm = owner->comm;
    p->comm_borrowed = true;
    return 0;
}

int pgcn_p2p_export(pgcn_plan* p, void* handle_out)
{
    if (!p || !handle_out) return fail(p, PGCN_ERR_INVALID, "null argument");
    if (p->k > kMaxPeers) return fail(p, PGCN_ERR_INVALID, "peer transport supports k <= %d", kMaxPeers);
    if (!p->arena) {
        auto align = [](int64_t x) { return (x + 255) / 256 * 256; };
        int64_t off = 0;
        p->off_flags = off; off = align(off + (int64_t)kMaxPeers * 8);
        const int64_t fwd_bytes = align((int64_t)p->h * p->f_max * 4), bwd_bytes = align((int64_t)p->S * p->f_max * 4);
        for (int i = 0; i < 2; ++i) { p->off_fwd[i] = off; off += std::max<int64_t>(fwd_bytes, 256); }
        for (int i = 0; i < 2; ++i) { p->off_bwd[i] = off; off += std::max<int64_t>(bwd_bytes, 256); }
        p->arena_bytes = off;
        CU(p, cudaMalloc(&p->arena, (size_t)off));
        CU(p, cudaMemset(p->arena, 0, (size_t)off));
        CU(p, cudaDeviceSynchronize());
    }
    P2PBlob b;
    memset(&b, 0, sizeof b);
    CU(p, cudaIpcGetMemHandle(&b.ipc, p->arena));
    b.arena_bytes = p->arena_bytes; b.off_flags = p->off_flags;
    for (int i = 0; i < 2; ++i) { b.off_fwd[i] = p->off_fwd[i]; b.off_bwd[i] = p->off_bwd[i]; }
    b.k = p->k; b.rank = p->rank; b.f_max = p->f_max;
    b.pid = (int64_t)getpid(); b.local_ptr = p->arena;
    for (int i = 0; i <= p->k; ++i) { b.send_off[i] = p->send_off[i]; b.recv_off[i] = p->recv_off[i]; }
    memset(handle_out, 0, PGCN_P2P_HANDLE_BYTES);
    memcpy(handle_out, &b, sizeof b);
    return 0;
}

int pgcn_p2p_import(pgcn_plan* p, const void* handles_k)
{
    if (!p || !handles_k) return fail(p, PGCN_ERR_INVALID, "null argument");
    if (!p->arena) return fail(p, PGCN_ERR_STATE, "call pgcn_p2p_export first");
    const char* base = static_cast<const char*>(handles_k);
    for (int q = 0; q < p->k; ++q) {
        memcpy(&p->peer_blob[q], base + (size_t)q * PGCN_P2P_HANDLE_BYTES, sizeof(P2PBlob));
        const P2PBlob& b = p->peer_blob[q];
        if (b.k != p->k || b.rank != q || b.f_max != p->f_max)
            return fail(p, PGCN_ERR_INVALID, "peer blob %d inconsistent (k=%d rank=%d f_max=%d)", q, b.k, b.rank, b.f_max);
        // wire-order invariant: what I send to q is what q expects from me (GPU/PGCN.py:47-48)
        if (b.recv_off[p->rank + 1] - b.recv_off[p->rank] != p->send_off[q + 1] - p->send_off[q])
            return fail(p, PGCN_ERR_INVALID, "send/recv count mismatch with peer %d", q);
        if (q == p->rank) { p->peer_arena[q] = p->arena; continue; }
        if (p->peer_arena[q]) continue;                     // already mapped (import called twice)
        if (b.pid == (int64_t)getpid()) {                   // a plan of this very process: plain device pointer
            p->peer_arena[q] = b.local_ptr;
            p->peer_local[q] = true;
            continue;
        }
        CU(p, cudaIpcOpenMemHandle(&p->peer_arena[q], b.ipc, cudaIpcMemLazyEnablePeerAccess));
    }
    preload_kernels();
    p->p2p = p->opt_p2p != 0;
    return 0;
}

// ---- hot path --------------------------------------------------------------------------------

int pgcn_spmm(pgcn_plan* p, int transpose, const float* H_own, const float* H_halo,
              float* Z, float* Z_halo, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (transpose == 2 || transpose == 3) {
        // the two halves of the overlapped forward, individually callable (k > 1 plans only)
        if (!p->have_split) return fail(p, PGCN_ERR_STATE, "plan has no own/halo split (k == 1 or h == 0)");
        if (!Z) return fail(p, PGCN_ERR_INVALID, "null Z");
        if (transpose == 2) {
            if (!H_own) return fail(p, PGCN_ERR_INVALID, "null H_own");
            return launch_spmm(p, p->own, H_own, nullptr, p->m, Z, nullptr, p->m, f, 0, st);
        }
        if (!H_halo) return fail(p, PGCN_ERR_INVALID, "null H_halo");
        for (int q = 0; q < p->k; ++q) {                  // Z += A_halo(q) * H_halo, one source peer after the other
            if (p->halo_q[(size_t)q].nrows == 0) continue;
            int rc2 = launch_spmm(p, p->halo_q[(size_t)q], H_halo, nullptr, p->h, Z, nullptr, p->m, f, 1, st);
            if (rc2) return rc2;
        }
        return 0;
    }
    if (!transpose) {
        if (p->m > 0 && (!H_own || !Z)) return fail(p, PGCN_ERR_INVALID, "null H_own/Z");
        if (p->h > 0 && !H_halo) return fail(p, PGCN_ERR_INVALID, "h=%d but H_halo is null", p->h);
        return launch_spmm(p, p->fwd, H_own, p->h > 0 ? H_halo : nullptr, p->m, Z, nullptr, p->m, f, 0, st);
    }
    if (p->m > 0 && (!H_own || !Z)) return fail(p, PGCN_ERR_INVALID, "null gZ/G");
    if (p->h > 0 && !Z_halo) return fail(p, PGCN_ERR_INVALID, "h=%d but Z_halo is null", p->h);
    return launch_spmm(p, p->tr, H_own, nullptr, p->m, Z, Z_halo, p->m, f, 0, st);
}

int pgcn_pack(pgcn_plan* p, const float* H, float* send_slab, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->S > 0 && (!H || !send_slab)) return fail(p, PGCN_ERR_INVALID, "null H/send_slab");
    return launch_pack(p, H, send_slab, f, (cudaStream_t)stream);
}

int pgcn_exchange(pgcn_plan* p, const float* send_slab, float* recv_slab, int32_t f, int reverse, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    return nccl_exchange(p, send_slab, recv_slab, f, reverse, (cudaStream_t)stream);
}

int pgcn_unpack_add(pgcn_plan* p, const float* recv_slab, float* G_own, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->S > 0 && (!recv_slab || !G_own)) return fail(p, PGCN_ERR_INVALID, "null recv_slab/G_own");
    return launch_unpack(p, recv_slab, G_own, f, (cudaStream_t)stream);
}

int pgcn_forward(pgcn_plan* p, const float* H_own, float* Z, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->m > 0 && (!H_own || !Z)) return fail(p, PGCN_ERR_INVALID, "null H_own/Z");
    cudaStream_t st = (cudaStream_t)stream;
    const int relu = (int)p->opt_relu;
    if (!p->have_split || !p->opt_overlap)
        // one rank, no overlap requested or nothing to split: every block has landed before one pass over [own | halo]
        return unsplit_forward(p, H_own, f, st, [&](float* halo, const float* halo_odd) {
            return launch_spmm(p, p->fwd, H_own, p->h > 0 ? halo : nullptr, p->m, Z, nullptr, p->m, f, 0, st, relu, false,
                               p->h > 0 ? halo_odd : nullptr);
        });
    Transport x;
    if ((rc = transport(p, f, &x)) || (rc = forward_send(p, H_own, f, x.p2p, true, st))) return rc;
    // ---- compute side: own columns while the rows travel, then each source's block as soon as it has landed
    if ((rc = launch_spmm(p, p->own, H_own, nullptr, p->m, Z, nullptr, p->m, f, 0, st, relu, true))) return rc;
    for (int i = 1; i < p->k; ++i) {
        const int src = step_src(p, i);
        if (x.p2p) { if ((rc = p2p_wait(p, src, st))) return rc; }
        else CU(p, cudaStreamWaitEvent(st, p->ev_step[(size_t)i], 0));
        if (p->halo_q[(size_t)src].nrows == 0) continue;
        if ((rc = launch_spmm(p, p->halo_q[(size_t)src], x.halo, nullptr, p->h, Z, nullptr, p->m, f, 1, st, relu, true,
                              x.halo_odd)))
            return rc;
    }
    if (x.p2p) CU(p, cudaStreamWaitEvent(st, p->ev_b, 0));
    return 0;
}

int pgcn_backward(pgcn_plan* p, const float* gZ, float* G_own, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->m > 0 && (!gZ || !G_own)) return fail(p, PGCN_ERR_INVALID, "null gZ/G_own");
    cudaStream_t st = (cudaStream_t)stream;
    // A^T g : rows [0,m) -> G_own, rows [m,m+h) -> halo partials, already in reverse wire order
    if (!p->have_split || !p->opt_overlap)
        return unsplit_backward(p, G_own, f, st, [&]() {
            return launch_spmm(p, p->tr, gZ, nullptr, p->m, G_own, p->d_hsend_slab, p->m, f, 0, st);
        });
    Transport x;
    if ((rc = transport(p, f, &x))) return rc;
    if (x.p2p && (rc = advance_epoch(p, st))) return rc;
    // ---- pipelined: the partials owed to each peer are computed first (in step order) and leave on the exchange
    // stream while the next peer's rows, and finally the own rows of A^T g, are still being computed
    cudaStream_t cs = p->comm_stream;
    for (int i = 1; i < p->k; ++i) {
        const int dst = step_dst(p, i);
        if (p->tr_halo_q[(size_t)dst].nrows > 0)
            if ((rc = launch_spmm(p, p->tr_halo_q[(size_t)dst], gZ, nullptr, p->m, G_own, p->d_hsend_slab, p->m, f, 0, st))) return rc;
        CU(p, cudaEventRecord(p->ev_step[(size_t)i], st));
        CU(p, cudaStreamWaitEvent(cs, p->ev_step[(size_t)i], 0));
        if (x.p2p) { if ((rc = p2p_put(p, dst, p->d_hsend_slab, f, true, cs))) return rc; }
        else if ((rc = nccl_step(p, p->d_hsend_slab, x.rrecv, f, 1, i, cs))) return rc;
    }
    CU(p, cudaEventRecord(p->ev_b, cs));
    if ((rc = launch_spmm(p, p->tr_own, gZ, nullptr, p->m, G_own, p->d_hsend_slab, p->m, f, 0, st))) return rc;
    if (x.p2p && (rc = p2p_wait_all(p, st))) return rc;
    CU(p, cudaStreamWaitEvent(st, p->ev_b, 0));      // NCCL: all blocks received; p2p: the send slab is free again
    return launch_unpack(p, x.rrecv, G_own, f, st, x.rrecv_odd);
}

int pgcn_forward_keep_halo(pgcn_plan* p, const float* H_own, float* Z, float* H_halo_out, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->k > 1 && p->h > 0 && !H_halo_out) return fail(p, PGCN_ERR_INVALID, "h=%d but H_halo_out is null", p->h);
    if ((rc = pgcn_forward(p, H_own, Z, f, stream))) return rc;
    if (p->k == 1 || p->h == 0) return 0;
    // the stream has waited for every source's rows; the peer transport's rows sit in the slab of this call's parity,
    // which the next fused call of the same parity overwrites: copy them now, picking the slab from the device epoch
    Transport x;
    if ((rc = transport(p, f, &x))) return rc;
    return copy_halo(p, x.halo, x.halo_odd, H_halo_out, f, (cudaStream_t)stream);
}

int pgcn_sddmm(pgcn_plan* p, const float* gZ, const float* H_own, const float* H_halo, float* dvals, int32_t f, void* stream)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->fwd.nnz > 0 && (!gZ || !H_own || !dvals)) return fail(p, PGCN_ERR_INVALID, "null gZ/H_own/dvals");
    if (p->h > 0 && !H_halo) return fail(p, PGCN_ERR_INVALID, "h=%d but H_halo is null", p->h);
    return launch_sddmm(p, gZ, H_own, p->h > 0 ? H_halo : nullptr, dvals, f, (cudaStream_t)stream);
}

// ---- sparse graph attention --------------------------------------------------------------------

int pgcn_halo_rows(pgcn_plan* p, const float* X_own, float* X_halo_out, int32_t w, void* stream)
{
    int rc = check_f(p, w);
    if (rc) return rc;
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "pgcn_halo_rows: call pgcn_plan_bind_values first");
    if (p->k == 1) return 0;
    if (p->m > 0 && !X_own) return fail(p, PGCN_ERR_INVALID, "null X_own");
    if (p->h > 0 && !X_halo_out) return fail(p, PGCN_ERR_INVALID, "h=%d but X_halo_out is null", p->h);
    cudaStream_t st = (cudaStream_t)stream;
    return unsplit_forward(p, X_own, w, st, [&](float* halo, const float* halo_odd) {
        return copy_halo(p, halo, halo_odd, X_halo_out, w, st);
    });
}

// The reverse of pgcn_halo_rows: the unsplit backward exchange with X_halo copied into the reverse send slab.
int pgcn_halo_rows_add(pgcn_plan* p, const float* X_halo, float* G_own, int32_t w, void* stream)
{
    int rc = check_f(p, w);
    if (rc) return rc;
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "pgcn_halo_rows_add: call pgcn_plan_bind_values first");
    if (p->k == 1) return 0;
    if (p->m > 0 && !G_own) return fail(p, PGCN_ERR_INVALID, "null G_own");
    if (p->h > 0 && !X_halo) return fail(p, PGCN_ERR_INVALID, "h=%d but X_halo is null", p->h);
    cudaStream_t st = (cudaStream_t)stream;
    return unsplit_backward(p, G_own, w, st, [&]() -> int {
        if (p->h > 0)
            CU(p, cudaMemcpyAsync(p->d_hsend_slab, X_halo, (size_t)p->h * w * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return 0;
    });
}

static int attn_check(pgcn_plan* p, const char* what, const float* el, const float* er_own, const float* er_halo)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "%s walks the forward rows: call pgcn_plan_bind_values first", what);
    if (p->m > 0 && (!el || !er_own)) return fail(p, PGCN_ERR_INVALID, "%s: null el/er_own", what);
    if (p->h > 0 && !er_halo) return fail(p, PGCN_ERR_INVALID, "%s: h=%d but er_halo is null", what, p->h);
    return 0;
}

// k heads; vec: every [., k] operand is aligned to the vector loads of its k values (attn_vec)
static int launch_attn(pgcn_plan* p, bool backward, const AttnArgs& a, cudaStream_t st, int k = 1, bool vec = false)
{
    const unsigned grid = (unsigned)p->nlong_rows + (unsigned)((p->m + kAttnWarps - 1) / kAttnWarps);
    pick_softmax(k, vec, backward)<<<grid, kAttnThreads, 0, st>>>(a);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

static AttnArgs attn_args(const pgcn_plan* p, const float* el, const float* er_own, const float* er_halo, float slope)
{
    AttnArgs a;
    a.rowptr = p->d_rowptr; a.long_rows = p->d_long_rows; a.nlong = p->nlong_rows; a.m = p->m;
    a.pieces = p->fwd.d_cw;
    a.el = el; a.er_own = er_own; a.er_halo = p->h > 0 ? er_halo : nullptr; a.slope = slope;
    a.alpha = a.dalpha = nullptr; a.out = a.d_el = nullptr;
    return a;
}

int pgcn_edge_softmax(pgcn_plan* p, const float* el, const float* er_own, const float* er_halo, float negative_slope,
                      float* alpha, void* stream)
{
    int rc = attn_check(p, "pgcn_edge_softmax", el, er_own, er_halo);
    if (rc) return rc;
    if (p->m == 0) return 0;
    if (p->fwd.nnz > 0 && !alpha) return fail(p, PGCN_ERR_INVALID, "null alpha");
    AttnArgs a = attn_args(p, el, er_own, er_halo, negative_slope);
    a.out = alpha;
    return launch_attn(p, false, a, (cudaStream_t)stream);
}

int pgcn_edge_softmax_backward(pgcn_plan* p, const float* el, const float* er_own, const float* er_halo,
                               const float* alpha, const float* dalpha, float negative_slope, float* dpre, float* d_el,
                               void* stream)
{
    int rc = attn_check(p, "pgcn_edge_softmax_backward", el, er_own, er_halo);
    if (rc) return rc;
    if (p->m == 0) return 0;
    if (!d_el || (p->fwd.nnz > 0 && (!alpha || !dalpha || !dpre)))
        return fail(p, PGCN_ERR_INVALID, "null alpha/dalpha/dpre/d_el");
    AttnArgs a = attn_args(p, el, er_own, er_halo, negative_slope);
    a.alpha = alpha; a.dalpha = dalpha; a.out = dpre; a.d_el = d_el;
    return launch_attn(p, true, a, (cudaStream_t)stream);
}

// ---- multi-head sparse graph attention ------------------------------------------------------------------------------

static int heads_check(pgcn_plan* p, const char* what, int heads)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (heads != 1 && heads != 2 && heads != 4 && heads != 8)
        return fail(p, PGCN_ERR_INVALID, "%s: heads=%d, not 1, 2, 4 or 8", what, heads);
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "%s reads the value maps: call pgcn_plan_bind_values first", what);
    return 0;
}

static int heads_check_f(pgcn_plan* p, const char* what, int heads, int f)
{
    int rc = heads_check(p, what, heads);
    if (rc) return rc;
    if ((rc = check_f(p, f))) return rc;
    if (f % heads != 0) return fail(p, PGCN_ERR_INVALID, "%s: f=%d is not a multiple of heads=%d", what, f, heads);
    return 0;
}

// Vector loads of the k values of a row or entry: k floats (4 .. 32 bytes) need alignment to min(4 k, 16) bytes
static bool attn_vec(int k, std::initializer_list<const void*> ops)
{
    const uintptr_t mask = (uintptr_t)std::min(4 * k, 16) - 1;
    for (const void* q : ops)
        if (q && (reinterpret_cast<uintptr_t>(q) & mask)) return false;
    return k > 1;
}

int pgcn_edge_softmax_heads(pgcn_plan* p, int32_t heads, const float* el, const float* er_own, const float* er_halo,
                            float negative_slope, float* alpha, void* stream)
{
    int rc = heads_check(p, "pgcn_edge_softmax_heads", heads);
    if (rc || (rc = attn_check(p, "pgcn_edge_softmax_heads", el, er_own, er_halo))) return rc;
    if (p->m == 0) return 0;
    if (p->fwd.nnz > 0 && !alpha) return fail(p, PGCN_ERR_INVALID, "null alpha");
    AttnArgs a = attn_args(p, el, er_own, er_halo, negative_slope);
    a.out = alpha;
    return launch_attn(p, false, a, (cudaStream_t)stream, heads, attn_vec(heads, {el, er_own, a.er_halo, alpha}));
}

int pgcn_edge_softmax_backward_heads(pgcn_plan* p, int32_t heads, const float* el, const float* er_own,
                                     const float* er_halo, const float* alpha, const float* dalpha, float negative_slope,
                                     float* dpre, float* d_el, void* stream)
{
    int rc = heads_check(p, "pgcn_edge_softmax_backward_heads", heads);
    if (rc || (rc = attn_check(p, "pgcn_edge_softmax_backward_heads", el, er_own, er_halo))) return rc;
    if (p->m == 0) return 0;
    if (!d_el || (p->fwd.nnz > 0 && (!alpha || !dalpha || !dpre)))
        return fail(p, PGCN_ERR_INVALID, "null alpha/dalpha/dpre/d_el");
    AttnArgs a = attn_args(p, el, er_own, er_halo, negative_slope);
    a.alpha = alpha; a.dalpha = dalpha; a.out = dpre; a.d_el = d_el;
    return launch_attn(p, true, a, (cudaStream_t)stream, heads,
                       attn_vec(heads, {el, er_own, a.er_halo, alpha, dalpha, dpre, d_el}));
}

// The unsplit forward exchange, then one multi-head launch over [H_own | halo slab of the call's parity], then the halo
// copy. The plan's resident values are not read.
int pgcn_forward_heads(pgcn_plan* p, int32_t heads, const float* alpha, const float* H_own, float* Z, float* H_halo_out,
                       int32_t f, void* stream)
{
    int rc = heads_check_f(p, "pgcn_forward_heads", heads, f);
    if (rc) return rc;
    if (p->m > 0 && (!H_own || !Z)) return fail(p, PGCN_ERR_INVALID, "null H_own/Z");
    if (p->fwd.nnz > 0 && !alpha) return fail(p, PGCN_ERR_INVALID, "null alpha");
    cudaStream_t st = (cudaStream_t)stream;
    const HeadArgs ha = {alpha, nullptr, heads};
    return unsplit_forward(p, H_own, f, st, [&](float* halo, const float* halo_odd) -> int {
        int rc2 = launch_spmm(p, p->fwd, H_own, p->h > 0 ? halo : nullptr, p->m, Z, nullptr, p->m, f, 0, st, 0, false,
                              p->h > 0 ? halo_odd : nullptr, &ha);
        return rc2 ? rc2 : copy_halo(p, halo, halo_odd, H_halo_out, f, st);
    });
}

// The unsplit backward with multi-head weights on the transposed records (through their value map).
int pgcn_backward_heads(pgcn_plan* p, int32_t heads, const float* alpha, const float* gZ, float* G_own, int32_t f,
                        void* stream)
{
    int rc = heads_check_f(p, "pgcn_backward_heads", heads, f);
    if (rc) return rc;
    if (p->m > 0 && (!gZ || !G_own)) return fail(p, PGCN_ERR_INVALID, "null gZ/G_own");
    if (p->fwd.nnz > 0 && !alpha) return fail(p, PGCN_ERR_INVALID, "null alpha");
    cudaStream_t st = (cudaStream_t)stream;
    const HeadArgs ha = {alpha, p->tr.d_vmap, heads};
    return unsplit_backward(p, G_own, f, st, [&]() {
        return launch_spmm(p, p->tr, gZ, nullptr, p->m, G_own, p->d_hsend_slab, p->m, f, 0, st, 0, false, nullptr, &ha);
    });
}

int pgcn_sddmm_heads(pgcn_plan* p, int32_t heads, const float* gZ, const float* H_own, const float* H_halo,
                     float* dalpha, int32_t f, void* stream)
{
    int rc = heads_check_f(p, "pgcn_sddmm_heads", heads, f);
    if (rc) return rc;
    if (p->fwd.nnz > 0 && (!gZ || !H_own || !dalpha)) return fail(p, PGCN_ERR_INVALID, "null gZ/H_own/dalpha");
    if (p->h > 0 && !H_halo) return fail(p, PGCN_ERR_INVALID, "h=%d but H_halo is null", p->h);
    return launch_sddmm_heads(p, heads, gZ, H_own, p->h > 0 ? H_halo : nullptr, dalpha, f, (cudaStream_t)stream);
}

// ---- max aggregation ------------------------------------------------------------------------------------------------

static int max_check(pgcn_plan* p, const char* what, int f)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (!p->bound) return fail(p, PGCN_ERR_STATE, "%s reads the value maps: call pgcn_plan_bind_values first", what);
    return check_f(p, f);
}

// The unsplit forward exchange, then one max launch over [H_own | halo slab of the call's parity].
int pgcn_forward_max(pgcn_plan* p, const float* H_own, float* Z, int32_t* arg, int32_t f, void* stream)
{
    int rc = max_check(p, "pgcn_forward_max", f);
    if (rc) return rc;
    if (p->m > 0 && (!H_own || !Z || !arg)) return fail(p, PGCN_ERR_INVALID, "pgcn_forward_max: null H_own/Z/arg");
    cudaStream_t st = (cudaStream_t)stream;
    return unsplit_forward(p, H_own, f, st, [&](float* halo, const float* halo_odd) {
        return launch_max(p, H_own, p->h > 0 ? halo : nullptr, p->h > 0 ? halo_odd : nullptr, Z, arg, f, st);
    });
}

// The transposed max launch (gZ routed by arg through the value map), then the unsplit backward exchange.
int pgcn_backward_max(pgcn_plan* p, const int32_t* arg, const float* gZ, float* G_own, int32_t f, void* stream)
{
    int rc = max_check(p, "pgcn_backward_max", f);
    if (rc) return rc;
    if (p->m > 0 && (!arg || !gZ || !G_own)) return fail(p, PGCN_ERR_INVALID, "pgcn_backward_max: null arg/gZ/G_own");
    cudaStream_t st = (cudaStream_t)stream;
    return unsplit_backward(p, G_own, f, st, [&]() {
        return launch_max_backward(p, arg, gZ, G_own, p->d_hsend_slab, f, st);
    });
}

// ---- GATv2 attention ------------------------------------------------------------------------------------------------

static int launch_softmax_raw(pgcn_plan* p, bool backward, int k, const float* alpha, float* io, cudaStream_t st)
{
    if (p->m == 0 || p->fwd.nnz == 0) return 0;
    AttnArgs a = attn_args(p, nullptr, nullptr, nullptr, 0.f);
    a.alpha = backward ? alpha : nullptr;
    a.dalpha = backward ? io : nullptr;
    a.out = io;
    const unsigned grid = (unsigned)p->nlong_rows + (unsigned)((p->m + kAttnWarps - 1) / kAttnWarps);
    pick_softmax_raw(k, attn_vec(k, {alpha, io}), backward)<<<grid, kAttnThreads, 0, st>>>(a);
    ++p->launches;
    CU(p, cudaGetLastError());
    return 0;
}

// The unsplit forward exchange of xl, then in one launch sequence: the scores into alpha, their softmax in place, the
// multi-head aggregation of xl with alpha over [xl_own | halo slab of the call's parity], and the halo copy.
int pgcn_forward_gatv2(pgcn_plan* p, int32_t heads, const float* xl_own, const float* xr, const float* att,
                       float negative_slope, float* alpha, float* Z, float* xl_halo_out, int32_t f, void* stream)
{
    int rc = heads_check_f(p, "pgcn_forward_gatv2", heads, f);
    if (rc) return rc;
    if (!att || (p->m > 0 && (!xl_own || !xr || !Z)))
        return fail(p, PGCN_ERR_INVALID, "pgcn_forward_gatv2: null xl_own/xr/att/Z");
    if (p->fwd.nnz > 0 && !alpha) return fail(p, PGCN_ERR_INVALID, "pgcn_forward_gatv2: null alpha");
    cudaStream_t st = (cudaStream_t)stream;
    const HeadArgs ha = {alpha, nullptr, heads};
    return unsplit_forward(p, xl_own, f, st, [&](float* halo, const float* halo_odd) -> int {
        const float* H1 = p->h > 0 ? halo : nullptr;
        const float* H1_odd = p->h > 0 ? halo_odd : nullptr;
        int rc2 = launch_gatv2_score(p, heads, xr, xl_own, H1, H1_odd, att, negative_slope, alpha, f, st);
        if (rc2 || (rc2 = launch_softmax_raw(p, false, heads, nullptr, alpha, st))) return rc2;
        if ((rc2 = launch_spmm(p, p->fwd, xl_own, H1, p->m, Z, nullptr, p->m, f, 0, st, 0, false, H1_odd, &ha)))
            return rc2;
        return copy_halo(p, halo, halo_odd, xl_halo_out, f, st);
    });
}

// dalpha = SDDMM(gZ, xl) into work, dscore over it in place, dxr and datt on the forward records, then dxl on the
// transposed records inside the unsplit backward exchange.
int pgcn_backward_gatv2(pgcn_plan* p, int32_t heads, const float* alpha, const float* gZ, const float* xl_own,
                        const float* xl_halo, const float* xr, const float* att, float negative_slope, float* work,
                        float* dxl, float* dxr, float* datt, int32_t f, void* stream)
{
    int rc = heads_check_f(p, "pgcn_backward_gatv2", heads, f);
    if (rc) return rc;
    if (!att || !datt || (p->m > 0 && (!gZ || !xl_own || !xr || !dxl || !dxr)))
        return fail(p, PGCN_ERR_INVALID, "pgcn_backward_gatv2: null gZ/xl_own/xr/att/dxl/dxr/datt");
    if (p->fwd.nnz > 0 && (!alpha || !work)) return fail(p, PGCN_ERR_INVALID, "pgcn_backward_gatv2: null alpha/work");
    if (p->h > 0 && !xl_halo) return fail(p, PGCN_ERR_INVALID, "pgcn_backward_gatv2: h=%d but xl_halo is null", p->h);
    cudaStream_t st = (cudaStream_t)stream;
    const float* xh = p->h > 0 ? xl_halo : nullptr;
    if ((rc = launch_sddmm_heads(p, heads, gZ, xl_own, xh, work, f, st))) return rc;
    if ((rc = launch_softmax_raw(p, true, heads, alpha, work, st))) return rc;
    if ((rc = launch_gatv2_rows(p, heads, work, xl_own, xh, xr, att, negative_slope, dxr, datt, f, st))) return rc;
    return unsplit_backward(p, dxl, f, st, [&]() {
        return launch_gatv2_cols(p, heads, alpha, work, gZ, xl_own, xh, xr, att, negative_slope, dxl, p->d_hsend_slab,
                                 f, st);
    });
}

static int host_slots(pgcn_plan* p, int64_t need)
{
    if (!p->s_in) {
        CU(p, cudaStreamCreateWithFlags(&p->s_in, cudaStreamNonBlocking));
        CU(p, cudaStreamCreateWithFlags(&p->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CU(p, cudaEventCreateWithFlags(&p->ev_in[i], cudaEventDisableTiming));
            CU(p, cudaEventCreateWithFlags(&p->ev_comp[i], cudaEventDisableTiming));
            CU(p, cudaEventCreateWithFlags(&p->ev_out[i], cudaEventDisableTiming));
        }
    }
    if (need > p->host_cap) {
        CU(p, cudaDeviceSynchronize());
        for (int i = 0; i < 2; ++i) {
            cudaFree(p->d_hostH[i]); cudaFree(p->d_hostZ[i]);
            p->d_hostH[i] = p->d_hostZ[i] = nullptr;
        }
        p->host_cap = 0;
        for (int i = 0; i < 2; ++i) {
            CU(p, cudaMalloc((void**)&p->d_hostH[i], std::max<size_t>((size_t)need, 1) * 4));
            CU(p, cudaMalloc((void**)&p->d_hostZ[i], std::max<size_t>((size_t)need, 1) * 4));
        }
        p->host_cap = need;
        p->host_steps = 0;
    }
    return 0;
}

int pgcn_forward_host_async(pgcn_plan* p, const float* H_host, float* Z_host, int32_t f)
{
    int rc = check_f(p, f);
    if (rc) return rc;
    if (p->m > 0 && (!H_host || !Z_host)) return fail(p, PGCN_ERR_INVALID, "null host buffer");
    CU(p, cudaSetDevice(p->device));
    const int64_t need = (int64_t)p->m * f;
    if ((rc = host_slots(p, need))) return rc;
    const int s = (int)(p->host_steps & 1);
    const bool reuse = p->host_steps >= 2;
    cudaStream_t cs = p->host_stream;
    // copy-in: the slot's H is free once the aggregation two steps ago has read it
    if (reuse) CU(p, cudaStreamWaitEvent(p->s_in, p->ev_comp[s], 0));
    CU(p, cudaMemcpyAsync(p->d_hostH[s], H_host, (size_t)need * 4, cudaMemcpyHostToDevice, p->s_in));
    CU(p, cudaEventRecord(p->ev_in[s], p->s_in));
    // compute: needs this step's H, and the slot's Z must have left for the host (two steps ago)
    CU(p, cudaStreamWaitEvent(cs, p->ev_in[s], 0));
    if (reuse) CU(p, cudaStreamWaitEvent(cs, p->ev_out[s], 0));
    if ((rc = pgcn_forward(p, p->d_hostH[s], p->d_hostZ[s], f, cs))) return rc;
    CU(p, cudaEventRecord(p->ev_comp[s], cs));
    // copy-out
    CU(p, cudaStreamWaitEvent(p->s_out, p->ev_comp[s], 0));
    CU(p, cudaMemcpyAsync(Z_host, p->d_hostZ[s], (size_t)need * 4, cudaMemcpyDeviceToHost, p->s_out));
    CU(p, cudaEventRecord(p->ev_out[s], p->s_out));
    ++p->host_steps;
    return 0;
}

int pgcn_forward_host_wait(pgcn_plan* p)
{
    if (!p) return fail(nullptr, PGCN_ERR_INVALID, "null plan");
    if (!p->s_out) return 0;
    CU(p, cudaStreamSynchronize(p->s_out));
    CU(p, cudaStreamSynchronize(p->host_stream));
    return 0;
}

int pgcn_forward_host(pgcn_plan* p, const float* H_host, float* Z_host, int32_t f)
{
    int rc = pgcn_forward_host_async(p, H_host, Z_host, f);
    if (rc) return rc;
    return pgcn_forward_host_wait(p);
}

}  // extern "C"
