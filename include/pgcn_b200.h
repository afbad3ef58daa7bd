/*
 * pgcn_b200.h — C-ABI of the H100-native PGCN aggregation path.
 *
 * This is the drop-in boundary for ONE hot path of the reference
 * (gunduzvd/Scalable-Graph-Convolutional-Network-Training-on-Distributed-Memory-Systems):
 * the per-layer sparse neighbour aggregation  Z = A_local * H  plus the boundary-row
 * (halo) exchange that the 1-D row partition induces.  In the reference that path is
 *
 *     GPU/PGCN.py:85-119   communicate_fgm(H, backward)     (pack / send / recv / unpack / H+X)
 *     GPU/PGCN.py:121-134  PSpMM.forward / PSpMM.backward   (torch.sparse.mm(A, H), torch.sparse.mm(A.t(), g))
 *     GPU/PGCN.py:37-64    compute_communication_maps, get_partitiont_of_adjacency_matrix (plan inputs)
 *     Parallel-GCN/main.c:269-299 / :374-404   GrB_mxm PLUS_TIMES_FP32 aggregation (CPU twin)
 *
 * Conventions
 *   - every entry point is extern "C", returns 0 on success or a negative pgcn_status,
 *     never throws, never calls exit(); the text of the last error is pgcn_last_error().
 *   - index arrays handed to pgcn_plan_create are HOST pointers and are copied; feature
 *     matrices (H, Z, G, slabs) are DEVICE pointers owned by the caller (torch), row-major
 *     fp32 with a leading dimension equal to f.
 *   - all compute entry points are asynchronous on the cudaStream_t passed in (as void*).
 *   - no torch types appear here.
 *
 * Column space of the local matrix (SURVEY.md §8e): rank r renumbers columns to
 *     [ own rows (m) | halo rows received from peer 0 | ... | from peer k-1 ]
 * each halo group sorted by global vertex id — the same order as the reference's
 * sorted send/recv maps (GPU/PGCN.py:47-48), so sender order == receiver order.
 */
#ifndef PGCN_B200_H
#define PGCN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pgcn_plan pgcn_plan;

typedef enum pgcn_status {
    PGCN_OK = 0,
    PGCN_ERR_INVALID = -1,   /* bad argument (null pointer, negative size, f > f_max, ...) */
    PGCN_ERR_CUDA = -2,      /* a CUDA runtime call failed                                   */
    PGCN_ERR_NCCL = -3,      /* NCCL missing or an NCCL call failed                          */
    PGCN_ERR_NOGPU = -4,     /* no CUDA device visible: there is NO CPU fallback             */
    PGCN_ERR_STATE = -5      /* call made in the wrong state (no communicator, ...)          */
} pgcn_status;

/* Byte counts for the roofline (SURVEY.md §8d "Algorithmic bytes"). All per call, this rank. */
typedef struct pgcn_bytes {
    int64_t nnz;            /* nnz_loc of the forward matrix                                  */
    int64_t m;              /* owned rows                                                      */
    int64_t h;              /* halo rows                                                       */
    int64_t cols_ref;       /* distinct columns referenced (own + halo)                        */
    int64_t spmm_fwd;       /* 8*nnz + 4*(m+1) + 4*f*cols_ref + 4*f*m                          */
    int64_t spmm_bwd;       /* 8*nnz + 4*(m+h+1) + 4*f*rows_ref_t + 4*f*(m+h)                  */
    int64_t gather_fwd;     /* no-reuse bound: nnz*(8+4f) + 4*(m+1) + 4*f*m                    */
    int64_t xchg_out;       /* 4*f*S   bytes this rank sends in a forward exchange             */
    int64_t xchg_in;        /* 4*f*h   bytes this rank receives in a forward exchange          */
    int64_t pack;           /* 2*4*f*S HBM bytes of the pack kernel                            */
} pgcn_bytes;

/* ---- library-level ---------------------------------------------------------------------- */

/* Version / build string, e.g. "pgcn_b200 0.1 sm_90a". Never NULL. */
const char* pgcn_version(void);

/* Number of visible CUDA devices, or a negative pgcn_status. */
int pgcn_device_count(void);

/* Text of the last error raised on `plan` (or on the library when plan == NULL). Never NULL. */
const char* pgcn_last_error(const pgcn_plan* plan);

/* ---- plan: replaces GPU/PGCN.py:37-64 (maps + local matrix) and :178-182 (buffers) ------- */

/*
 * Build the per-rank plan on the CURRENT CUDA device.
 *   rowptr/colidx/vals        forward CSR of the owned rows: m rows, columns in [0, m+h)
 *   t_rowptr/t_colidx/t_vals  CSR of its transpose: m+h rows, columns in [0, m)
 *                             (replaces the per-call A.t() + re-coalesce of GPU/PGCN.py:132)
 *   send_idx                  S = send_off[k] local row ids; rows for peer p are
 *                             send_idx[send_off[p] .. send_off[p+1])   (GPU/PGCN.py:47 send_map)
 *   recv_off                  halo rows from peer p live at columns m+recv_off[p] .. m+recv_off[p+1);
 *                             h = recv_off[k]                          (GPU/PGCN.py:48 recv_map)
 *   f_max                     largest feature width that will be used (sizes the slabs)
 * Duplicated (row, col) entries are allowed and are summed, like the uncoalesced COO of
 * GPU/PGCN.py:60-63.
 */
int pgcn_plan_create(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                     int32_t m, int32_t h,
                     const int32_t* t_rowptr, const int32_t* t_colidx, const float* t_vals,
                     const int32_t* send_idx, const int64_t* send_off, const int64_t* recv_off,
                     int32_t k, int32_t rank, int32_t f_max,
                     pgcn_plan** out);

int pgcn_plan_destroy(pgcn_plan* plan);

/*
 * Plan options (take effect at the next compute call). Names:
 *   "kernel"               0 = automatic (default): widths that are multiples of 128 floats with 16-byte aligned
 *                          operands take the shared-memory ring kernel fed by 2-D tensor-map TMA, everything else the
 *                          register-pipeline kernel; 4 = always the register kernel; 5 / 6 / 7 = ring kernel fed by
 *                          1-D cp.async.bulk / cp.async / 2-D tensor-map TMA (one row per copy). Under every setting
 *                          an operand that is not 16-byte aligned takes the register kernel with scalar accesses:
 *                          slower, same bits as the register kernel on aligned copies
 *   "ring_slots"           row slots per warp of the ring kernel: 16 (default), 32, 64; "ring_groups" 2 | 4 (64 slots)
 *   "ring_tile_floats"     floats of H one ring slot holds: 0 = tuned by pgcn_plan_autotune, else the full width
 *                          (256 when f % 256 == 0, else 128) (default); 64 = 256-byte slices, gathered one slice of
 *                          every row after the other so that less of H competes for L2; 128, 256. A width that does
 *                          not divide f, and 64 with "kernel" 6, take the full width. Results do not depend on it.
 *   "ring_edges_per_block" target nnz of one row block = one warp's unit of work          (default 512)
 *   "ring_long_row"        rows with more nnz than this are split into segments           (default 2 * block)
 *   "persistent"           1 = persistent CTAs fetch row blocks dynamically (default; single-rank plans and plans
 *                          without overlap), "persistent_multi" 1 = also for overlapped multi-rank plans (default 0:
 *                          persistent CTAs would hold the SMs the exchange kernels need)
 *   "edges_per_block", "long_row", "tile_floats"   the same for the register kernel (defaults 128, 4 * block, 0)
 *   "overlap"              1 = split A_local into own / per-peer halo blocks and pipeline the exchange with them
 *                          (Parallel-GCN/main.c:271 then :275-299)                         (default 1)
 *   "relu"                 1 = pgcn_forward writes relu(A_local * H); NaN stays NaN, as in torch.relu (default 0)
 *   "p2p"                  0 = never use the peer-memory transport (all ranks must agree)  (default 1)
 * pgcn_plan_autotune overrides block sizes / ring depth / ring tile width per matrix; setting a block size or the
 * ring depth explicitly clears the tuned values, a non-zero "ring_tile_floats" overrides the tuned width. "hot_mb" (L2-resident hot set of H rows) is fixed at plan creation: environment variable PGCN_HOT_MB.
 * Split rows are always reduced in a fixed order: results are run-to-run deterministic.
 * Read-only names for pgcn_plan_get_option: "nccl", "blocks_fwd", "long_rows_fwd", "ring_blocks_fwd",
 * "ring_long_rows_fwd", "retired_schedules" (see pgcn_plan_prepare), "epoch" (the peer transport's exchange epoch =
 * fused calls over peer memory so far; a synchronous device read, not to be called while a stream is captured).
 */
int pgcn_plan_set_option(pgcn_plan* plan, const char* name, int64_t value);
int64_t pgcn_plan_get_option(const pgcn_plan* plan, const char* name);

/*
 * Time the forward SpMM of this plan at feature width f for a few "edges_per_block" values on
 * scratch buffers and keep the fastest (set-up work, like the reference's untimed plan building,
 * GPU/PGCN.py:171-200). Synchronous. Returns the chosen value (>0) or a negative pgcn_status.
 */
int pgcn_plan_autotune(pgcn_plan* plan, int32_t f);

/*
 * CUDA graphs. Synchronous set-up work for width f under the current options: builds every row-block schedule the
 * fused calls can use at f (register and ring kernel: which one runs depends on the operands' alignment), sets every
 * ring kernel instance's shared-memory attribute and occupancy, and loads the kernels. Afterwards pgcn_forward and
 * pgcn_backward at width f make only stream-ordered CUDA calls and can be captured (cudaStreamBeginCapture,
 * torch.cuda.graph). A call that would still need set-up work while its stream is being captured returns
 * PGCN_ERR_STATE, before any unsafe call, and names this function; change f or an option, then prepare again.
 * Schedules replaced after the first prepare (a new option, pgcn_plan_autotune) are kept until pgcn_plan_destroy,
 * so a graph captured earlier never reads freed memory (read-only option "retired_schedules" counts them).
 * A captured graph fixes f, the options, the "relu" epilogue and the operand addresses of the capture: replay it on
 * new inputs by copying them into the captured buffers. The peer transport's exchange epoch lives in device memory
 * and advances with every replay, so eager calls and replays may be mixed in any order, as long as all ranks make
 * the same sequence of fused calls. pgcn_launch_count does not count replays.
 */
int pgcn_plan_prepare(pgcn_plan* plan, int32_t f);

/*
 * Host-only (no GPU needed): the row-block schedule the SpMM walks, for inspection and tests.
 * rowptr must describe NON-EMPTY rows only (the plan squeezes empty rows out first). Writes up to cap_blocks
 * blocks as 4 int32 each {first row, nrows | -(slot+1), e_begin, e_end}; returns the number of blocks.
 */
int64_t pgcn_debug_schedule(const int32_t* rowptr, int32_t nrows, int64_t edges_per_block, int64_t long_row,
                            int32_t* blocks_out, int64_t cap_blocks, int32_t* nlong_out, int32_t* nslots_out);

/* Plan-owned device slabs (f_max floats per row), for callers that want zero-copy access:
 * which = 0 send slab (S rows), 1 halo/recv slab (h rows), 2 reverse recv slab (S rows),
 * 3 reverse send slab (h rows: halo partials of A^T g). */
void* pgcn_plan_slab(pgcn_plan* plan, int which);

int pgcn_algorithmic_bytes(const pgcn_plan* plan, int32_t f, pgcn_bytes* out);

/* Number of kernels launched by this plan since creation (bench.py's "gpu_launches"). */
int64_t pgcn_launch_count(const pgcn_plan* plan);

/* ---- communicator: replaces dist.init_process_group + dist.send/recv (GPU/PGCN.py:107,112,242) */

/* Fill `id128` (128 bytes) with an NCCL unique id (rank 0 calls this, then ships the bytes). */
int pgcn_comm_unique_id(void* id128);
/* Collective over the k ranks of the plan. */
int pgcn_comm_init(pgcn_plan* plan, const void* id128);

/*
 * Peer-memory transport (single NVSwitch box): the pack kernel stores boundary rows straight
 * into the peer's halo slab over NVLink, no staging copy and no NCCL on the data path.
 *   pgcn_p2p_export : writes PGCN_P2P_HANDLE_BYTES: this rank's CUDA IPC handle for its exchange arena + layout
 *   pgcn_p2p_import : takes the k handles/layouts gathered from all ranks (rank-major)
 */
#define PGCN_P2P_HANDLE_BYTES 512
/* Many plans, one communicator (mini-batch training: one plan per pre-sampled batch, GPU/PGCN-Mini-batch.py:220-230
 * swaps [bA, send_map, recv_map] per batch over the same process group): `plan` borrows `owner`'s NCCL communicator
 * (same rank / size / device); the owner must outlive the borrowers. */
int pgcn_comm_share(pgcn_plan* plan, pgcn_plan* owner);
int pgcn_p2p_export(pgcn_plan* plan, void* handle_out);
int pgcn_p2p_import(pgcn_plan* plan, const void* handles_k);

/* ---- the hot path ------------------------------------------------------------------------ */

/*
 * Z = op(A_local) * [H_own ; H_halo]         (GPU/PGCN.py:127 and :132 without the exchange)
 *   transpose = 0 : A (m rows). H_own is m x f, H_halo is h x f (may be NULL when h == 0).
 *                   Z is m x f; Z_halo is ignored.
 *   transpose = 1 : A^T (m+h rows). H_own is the m x f upstream gradient, H_halo ignored.
 *                   Rows [0,m) go to Z (m x f), rows [m, m+h) go to Z_halo (h x f), already in
 *                   the wire order of the reverse exchange.
 *   transpose = 2 : own-columns half of the overlapped forward, Z  = A_own  * H_own
 *   transpose = 3 : halo-columns half,                          Z += A_halo * H_halo
 *                   (Parallel-GCN/main.c:271 then :295; plans with k > 1 and h > 0 only)
 * Operands need 4-byte alignment only. When one of them is not 16-byte aligned (or f % 4 != 0) the call takes the
 * register kernel with scalar accesses, which is slower; the same holds for every entry point below.
 */
int pgcn_spmm(pgcn_plan* plan, int transpose,
              const float* H_own, const float* H_halo,
              float* Z, float* Z_halo, int32_t f, void* stream);

/* send_slab[j, :] = H[send_idx[j], :]  for all peers in one launch   (GPU/PGCN.py:104) */
int pgcn_pack(pgcn_plan* plan, const float* H, float* send_slab, int32_t f, void* stream);

/*
 * All-to-all-v of row slabs (GPU/PGCN.py:99-115, both phases, all peers, one grouped call).
 *   reverse = 0 : send send_slab rows [send_off[p], send_off[p+1]) to p; receive halo rows
 *                 [recv_off[p], recv_off[p+1]) from p.
 *   reverse = 1 : the gradient direction (maps swapped, GPU/PGCN.py:93-97).
 * Zero-length messages are skipped on the wire (they are still counted by the host stats).
 */
int pgcn_exchange(pgcn_plan* plan, const float* send_slab, float* recv_slab,
                  int32_t f, int reverse, void* stream);

/*
 * G_own[send_idx[j], :] += recv_slab[j, :]   summed over ALL j in a fixed order
 * (the intended semantics of GPU/PGCN.py:115 in backward; the reference ASSIGNS — quirk Q3).
 */
int pgcn_unpack_add(pgcn_plan* plan, const float* recv_slab, float* G_own, int32_t f, void* stream);

/*
 * Fused convenience entry points = PSpMM.forward / PSpMM.backward (GPU/PGCN.py:123-134).
 *   forward : pack -> exchange (NCCL, or peer stores when p2p was imported) overlapped with
 *             the own-columns part of the SpMM -> halo-columns part. Z (m x f) = A_local * H.
 *   backward: G (m x f) = (A_local^T * gZ)[own] + contributions received from the peers.
 * With k == 1 no communicator is needed.
 */
/* Plan option "relu" = 1 fuses the layer epilogue into the forward: Z = max(0, A_local * H), clamped in the store of
 * whichever launch writes a row last (no extra pass over Z). With the dense step applied first — relu(A (H W)) — it is
 * the reference layer relu(linear(PSpMM(A, H))) of GPU/PGCN.py:144-148 up to fp32 association. Forward only. */
int pgcn_forward(pgcn_plan* plan, const float* H_own, float* Z, int32_t f, void* stream);
int pgcn_backward(pgcn_plan* plan, const float* gZ, float* G_own, int32_t f, void* stream);

/* ---- edge values: the aggregation's values set per call, and their gradient ------------------ */
/*
 * torch.sparse.mm(A, H) (GPU/PGCN.py:127) takes new values of A on every call and, when they require grad, returns
 * dA.values = < gZ[row(e)], H[col(e)] >. These entry points give the plan the same two abilities (learned edge
 * weights, per-step edge masks such as DropEdge, attention scores), without changing the exchange or the kernels.
 *
 * pgcn_plan_bind_values: synchronous set-up, like pgcn_plan_autotune and pgcn_plan_prepare. For every record set of
 *   the plan (forward, transposed, and on split multi-rank plans the own-column block and each peer's block) it builds
 *   a device map from each stored entry to its forward entry (an index into the colidx / vals arrays given to
 *   pgcn_plan_create), reading the plan's own records back; it also keeps a device copy of the creation values.
 *   Transposed entries are matched to the forward entry of the same (row, column), duplicates in order of appearance;
 *   a transposed CSR that does not hold the same entries with the same values returns PGCN_ERR_INVALID and names the
 *   first mismatch. Cost: 4 B per entry per record set that is not the forward matrix itself, plus 4 B per entry of
 *   creation values: 12 B per edge on a split multi-rank plan, 8 B on one rank. Plans that are never bound pay nothing.
 *   Binding twice is a no-op. Its copies run on a stream of the plan and wait for that stream only (never for the
 *   device), so it may be called while other plans of the process have exchange kernels waiting on the device.
 * pgcn_plan_set_values: `vals` is a DEVICE array of nnz floats in forward CSR order; NULL restores the creation values.
 *   One kernel rewrites the value words of every record set, stream-ordered on `stream`: every later compute call on
 *   that stream (pgcn_spmm, pgcn_forward / pgcn_backward, the _host variants, every kernel and layout) aggregates with
 *   these values. Masks, schedules and the hot / cold marking do not depend on values and do not change. Capturable.
 *   Before pgcn_plan_bind_values it returns PGCN_ERR_STATE.
 * pgcn_sddmm: dvals[e] = sum_c gZ[row(e), c] * [H_own ; H_halo][col(e), c] for every forward entry e, written in
 *   forward CSR order (nnz floats). gZ and H_own are m x f, H_halo h x f (may be NULL when h == 0): the halo rows of
 *   the forward, see pgcn_forward_keep_halo. Local only (no exchange); every output is reduced in one fixed order, so
 *   runs are bit-identical. Needs no binding. f = 128, 256, 384 or 512 with 16-byte aligned operands takes a
 *   shared-memory ring kernel fed by TMA bulk copies, every other case a plain kernel. Like pgcn_forward it refuses,
 *   with PGCN_ERR_STATE, set-up work while its stream is being captured: pgcn_plan_prepare(plan, f) does that set-up.
 * pgcn_forward_keep_halo: pgcn_forward, and in addition the h halo rows this call received are copied into
 *   H_halo_out (h x f, caller-owned) on `stream` before it returns, out of the slab of the call's exchange parity (the
 *   next fused call of the same parity overwrites that slab). With k == 1 it is pgcn_forward (H_halo_out unused).
 */
int pgcn_plan_bind_values(pgcn_plan* plan);
int pgcn_plan_set_values(pgcn_plan* plan, const float* vals, void* stream);
int pgcn_sddmm(pgcn_plan* plan, const float* gZ, const float* H_own, const float* H_halo, float* dvals, int32_t f,
               void* stream);
int pgcn_forward_keep_halo(pgcn_plan* plan, const float* H_own, float* Z, float* H_halo_out, int32_t f, void* stream);

/* ---- sparse graph attention: the edge softmax of GPU/PGAT.py:139-148 over the stored pattern ---------------------- */
/*
 * With el (m floats, one per owned row) and er (one per column: er_own, m floats, then er_halo, h floats, the halo
 * rows' values from pgcn_halo_rows; er_halo may be NULL when h == 0):
 *   s_e = LeakyReLU(el[row(e)] + er[col(e)], negative_slope)          for every forward entry e
 *   alpha_e = exp(s_e - max_row s) / sum_row exp(s - max_row s)        over the stored entries of row(e) only
 * pgcn_edge_softmax writes alpha (nnz floats, forward CSR order: what pgcn_plan_set_values takes). Rows without entries
 *   write nothing. Full-precision expf with the row maximum subtracted: no overflow for any row length or score.
 * pgcn_edge_softmax_backward: given alpha and dalpha (nnz, e.g. pgcn_sddmm of the output gradient against the
 *   aggregated rows), writes dpre_e = alpha_e (dalpha_e - sum_row alpha dalpha) * (s_e > 0 ? 1 : negative_slope)
 *   (nnz floats) and d_el[i] = sum over row i of dpre (m floats, 0 for empty rows). The gradient of er is the column
 *   sum of dpre over all ranks: pgcn_plan_set_values(dpre), then pgcn_backward on an m x 4 matrix of ones (column 0).
 *   Both kernels give a warp to each row and a CTA to each row of more than 1024 entries; every output is reduced in
 *   one fixed order, so runs are bit-identical.
 * pgcn_halo_rows: the forward exchange of pgcn_forward without the SpMM. X_own is m x w (this rank's owned rows), the
 *   h halo rows it receives are copied into X_halo_out (h x w) on `stream`. Peer transport when imported and
 *   w % 4 == 0 (the device epoch advances as in every fused call), NCCL otherwise. k == 1: nothing to do.
 * All three need pgcn_plan_bind_values (PGCN_ERR_STATE before) and do no set-up work of their own: they are capturable
 *   once the plan is bound (and, for the exchange, wired). A null plan or a null argument returns PGCN_ERR_INVALID.
 */
int pgcn_edge_softmax(pgcn_plan* plan, const float* el, const float* er_own, const float* er_halo, float negative_slope,
                      float* alpha, void* stream);
int pgcn_edge_softmax_backward(pgcn_plan* plan, const float* el, const float* er_own, const float* er_halo,
                               const float* alpha, const float* dalpha, float negative_slope, float* dpre, float* d_el,
                               void* stream);
int pgcn_halo_rows(pgcn_plan* plan, const float* X_own, float* X_halo_out, int32_t w, void* stream);

/* ---- multi-head sparse graph attention: K = heads in {1, 2, 4, 8} heads of width d = f / K ------------------------ */
/*
 * Every array is row-major and head-minor: el, er_own and d_el are m x K, er_halo is h x K, alpha, dalpha and dpre are
 * nnz x K in forward CSR order (the order of pgcn_plan_set_values). Head h of the output is
 *   Z[:, h d:(h+1) d] = A(alpha[:, h]) [H_own ; H_halo][:, h d:(h+1) d]
 * and the heads are concatenated. None of these calls reads or writes the plan's resident values (pgcn_plan_set_values
 * is never needed): the aggregation takes its weights from alpha.
 * pgcn_edge_softmax_heads / pgcn_edge_softmax_backward_heads: pgcn_edge_softmax / _backward for every head at once (one
 *   gather of a column brings its K er values). heads == 1 launches the single-head kernels: the same bits.
 * pgcn_forward_heads: the exchange of pgcn_forward without its per-source overlap (both transports), then one launch of
 *   the register SpMM with the heads' weights over [H_own | halo rows]; with H_halo_out (h x f, may be NULL) the halo
 *   rows received are copied out as in pgcn_forward_keep_halo. The device epoch advances as in every fused call.
 * pgcn_backward_heads: G_own = A(alpha)^T gZ with the halo partials summed at their owners (pgcn_backward without its
 *   per-peer pipelining). With alpha[:, h] equal to the plan's creation values for every head, both calls give the bits of
 *   pgcn_forward / pgcn_backward with the plan option kernel = 4 (the same schedule and summation order).
 * pgcn_sddmm_heads: dalpha[e, h] = < gZ[row(e), h d:(h+1) d], [H_own ; H_halo][col(e), h d:(h+1) d] >. f = 128, 256 or
 *   512 with d % 4 == 0 and 16-byte aligned operands takes a ring kernel, every other case a plain kernel; heads == 1 is
 *   pgcn_sddmm.
 * All five need pgcn_plan_bind_values (PGCN_ERR_STATE before). heads outside {1, 2, 4, 8}, f % heads != 0 and null
 * arguments return PGCN_ERR_INVALID. After pgcn_plan_prepare(plan, f) they are capturable.
 */
int pgcn_edge_softmax_heads(pgcn_plan* plan, int32_t heads, const float* el, const float* er_own, const float* er_halo,
                            float negative_slope, float* alpha, void* stream);
int pgcn_edge_softmax_backward_heads(pgcn_plan* plan, int32_t heads, const float* el, const float* er_own,
                                     const float* er_halo, const float* alpha, const float* dalpha, float negative_slope,
                                     float* dpre, float* d_el, void* stream);
int pgcn_forward_heads(pgcn_plan* plan, int32_t heads, const float* alpha, const float* H_own, float* Z,
                       float* H_halo_out, int32_t f, void* stream);
int pgcn_backward_heads(pgcn_plan* plan, int32_t heads, const float* alpha, const float* gZ, float* G_own, int32_t f,
                        void* stream);
int pgcn_sddmm_heads(pgcn_plan* plan, int32_t heads, const float* gZ, const float* H_own, const float* H_halo,
                     float* dalpha, int32_t f, void* stream);

/* ---- max aggregation: the element-wise maximum over each row's neighbours (GraphSAGE "pool", PyG aggr="max") ------- */
/*
 * For every owned row i and feature c, with X = [H_own ; H_halo]:
 *   Z[i, c] = X[col(e*), c],  arg[i, c] = e*
 * e* is the FIRST stored entry of row i in forward CSR order whose value is >= every other entry's, NaN counting as
 * larger than any number (numpy.argmax over the row's entries); Z is copied from the winner bit for bit (its sign of
 * zero, its NaN payload). arg indexes the colidx / vals arrays given to pgcn_plan_create (colidx[arg] is the local
 * column). Rows without an entry give Z = 0 and arg = -1. The values of A are not read, only its pattern: of duplicated
 * (row, column) entries the first copy wins. A max is exact, so Z does not depend on the block size, width, alignment or
 * long-row split. On several ranks Z is the same on every partition; where values tie, the winner follows the local
 * column order [own | halo by peer], so arg may name another (equal-valued) global column than on one rank.
 * Z and gZ are m x f fp32, arg is m x f int32, all row-major with row stride f.
 * pgcn_forward_max: the exchange of pgcn_forward without its per-source overlap (both transports), then one launch of
 *   the max kernel over [H_own | halo rows]. The device epoch advances as in every fused call.
 * pgcn_backward_max: G_own[j, c] = sum of gZ[i, c] over every row i, on every rank, whose arg[i, c] is an entry of
 *   column j: one launch over the transposed records, then the exchange of pgcn_backward without its per-peer
 *   pipelining, the halo partials summed at their owners in a fixed order. Run-to-run identical, like the forward.
 * Both need pgcn_plan_bind_values (PGCN_ERR_STATE before). f outside [1, f_max] and null arguments return
 * PGCN_ERR_INVALID. After pgcn_plan_prepare(plan, f) they are capturable.
 */
int pgcn_forward_max(pgcn_plan* plan, const float* H_own, float* Z, int32_t* arg, int32_t f, void* stream);
int pgcn_backward_max(pgcn_plan* plan, const int32_t* arg, const float* gZ, float* G_own, int32_t f, void* stream);

/* ---- GATv2 attention: dynamic attention (Brody et al.) over the stored pattern, K = heads in {1, 2, 4, 8} ---------- */
/*
 * Inputs: xl (source side, m x f; the halo rows come from their owners), xr (destination side, m x f; only owned rows
 * are read, so only xl is exchanged), att (K x d, d = f / K, row-major: att[h, c] is float h d + c) and negative_slope.
 * For every stored entry e = (i, j) of the local matrix (j a local column in [own | halo by peer]) and head h:
 *   s_eh      = sum_{c < d} att[h, c] * LeakyReLU(xl[j, h d + c] + xr[i, h d + c])
 *   alpha_.h  = the softmax of s_.h over the stored entries of each row, row maximum subtracted, full-precision expf
 *   Z[i, h d:(h+1) d] = sum_e alpha_eh xl[j, h d:(h+1) d]                 (heads concatenated)
 * This is PyG GATv2Conv(share_weights=False, concat=True, bias=False, add_self_loops=False, dropout=0) over the stored
 * pattern; share_weights=True is xl == xr. Rows without entries give Z = 0 and write no alpha. alpha and work are
 * nnz x K in forward CSR order (the order pgcn_plan_set_values takes). Every sum is added in a fixed order: two runs
 * give the same bits, and so do the ring and plain score kernels and the 4-wide and scalar backward kernels.
 * Backward, with dalpha = pgcn_sddmm_heads(gZ, xl), dscore_eh = alpha_eh (dalpha_eh - sum_row alpha_.h dalpha_.h),
 * t = xl[j] + xr[i] and g_ec = dscore_e,h(c) * att_c * LeakyReLU'(t_c):
 *   dxr[i]    = sum_{e in row i} g_e
 *   dxl[j]    = sum_{e in column j} alpha_e,h(c) gZ[i, c] + g_ec     (halo columns summed at their owners)
 *   datt[h, c] = sum_e dscore_eh * LeakyReLU(t_c)                    (no atomics: per-chunk partials, fixed order)
 * pgcn_forward_gatv2: the exchange of xl as in pgcn_forward_heads (once), then the score kernel writes the scores into
 *   alpha, the edge softmax turns them into alpha in place, the multi-head aggregation writes Z, and with xl_halo_out
 *   (h x f, may be NULL) the received halo rows of xl are copied out for the backward. The device epoch advances as in
 *   every fused call.
 * pgcn_backward_gatv2: work (nnz x K, caller-owned) receives dalpha and then dscore in place; dxr (m x f) and datt (K x d)
 *   from the forward records; dxl (m x f) from the transposed records, with the exchange of pgcn_backward_heads.
 *   xl_halo: the rows pgcn_forward_gatv2 returned in xl_halo_out (h x f; unused when h == 0).
 * Both need pgcn_plan_bind_values (PGCN_ERR_STATE before) and never read or write the plan's resident values. heads
 * outside {1, 2, 4, 8}, f % heads != 0 and null arguments return PGCN_ERR_INVALID. After pgcn_plan_prepare(plan, f)
 * both are capturable. The plan keeps f_max floats per 8 row blocks of its forward schedule for the datt partials.
 */
int pgcn_forward_gatv2(pgcn_plan* plan, int32_t heads, const float* xl_own, const float* xr, const float* att,
                       float negative_slope, float* alpha, float* Z, float* xl_halo_out, int32_t f, void* stream);
int pgcn_backward_gatv2(pgcn_plan* plan, int32_t heads, const float* alpha, const float* gZ, const float* xl_own,
                        const float* xl_halo, const float* xr, const float* att, float negative_slope, float* work,
                        float* dxl, float* dxr, float* datt, int32_t f, void* stream);

/* ---- host-buffer variant: what a non-torch host (the reference's C path) would bind -------- */
/*
 * Same as pgcn_forward but H and Z are HOST pointers (pinned or pageable): copies H to the
 * device, runs the path, copies Z back, synchronises. This is the call bench.py times as "e2e".
 */
int pgcn_forward_host(pgcn_plan* plan, const float* H_host, float* Z_host, int32_t f);
/*
 * Software-pipelined form for a host that streams many aggregations (layers, mini-batches, timesteps):
 * pgcn_forward_host_async enqueues  H_host -> device slot (copy-in stream) ; pgcn_forward (compute stream) ;
 * device slot -> Z_host (copy-out stream)  on one of TWO device slots and returns at once, so the upload of
 * step i+1 and the download of step i-1 run under the aggregation of step i (PCIe is full duplex).
 * H_host must stay untouched and Z_host unread until pgcn_forward_host_wait returns; it waits for everything
 * enqueued so far. Pinned host buffers are needed for the copies to overlap. Replaces nothing in the reference
 * (it has no host-resident path, GPU/PGCN.py:186-196 keeps H on the device): it is the C-trainer-facing form of
 * the PSpMM.forward boundary (GPU/PGCN.py:123-127).
 * On a multi-rank plan the call advances the exchange epoch on the plan's own stream, which is not ordered with the
 * caller's streams: every earlier call of the plan must have completed before it (synchronise the caller's stream),
 * and no other call of the plan may be enqueued between it and pgcn_forward_host_wait.
 */
int pgcn_forward_host_async(pgcn_plan* plan, const float* H_host, float* Z_host, int32_t f);
int pgcn_forward_host_wait(pgcn_plan* plan);

#ifdef __cplusplus
}
#endif
#endif /* PGCN_B200_H */
