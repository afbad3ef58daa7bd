/*
 * pgcn_gine.h — C-ABI of the GINE library (lib/libpgcn_gine.so), sm_90a.
 *
 * The edge-feature sum aggregation of GINE (Hu et al., "Strategies for Pre-training Graph Neural Networks"; PyG's
 * GINEConv) over the stored pattern of a rank's local matrix. For every stored entry e = (i, j) of row i and every
 * feature, with X [m + h, f] (own rows, then halo rows) and E [nnz_local, f]:
 *
 *     pre_e  = X[j] + E_e                       one fp32 add (__fadd_rn)
 *     msg_e  = pre_e < 0 ? +0 : pre_e           torch.relu's rule: NaN propagates, -0 stays -0
 *     Z[i]   = sum_{e in row i} msg_e           fp32, starting at +0, in CSR entry order; split rows in chunk order
 *     dE_e   = !(pre_e <= 0) ? gZ[i] : 0        torch's relu backward: the gradient passes for pre > 0 and for NaN
 *     dX[j]  = sum_{e in column j} dE_e         in transposed-entry order (the stable column sort), j in [0, m + h)
 *
 * The values of A are not read; every stored entry contributes, duplicates included. A row with no entries gives
 * Z = 0. Round-to-nearest keeps the sign of a sum, so fl(x + e) > 0 exactly when x + e > 0: the mask is the exact one,
 * and dE is either gZ[i] or 0, to the bit. GIN's self term (1 + eps) x_i is not part of these kernels.
 *
 * A per-entry tensor (E, dE) is nnz x f, row-major, in the local forward CSR's entry order (the order of
 * PgcnPlan.edge_pairs()); every per-entry offset is 64-bit, so nnz * f may exceed 2^31. It never crosses ranks: under
 * the 1-D row partition every entry belongs to the rank that owns its row.
 *
 * Operands (fp32, row-major, DEVICE pointers):
 *   X_own    m x f          the owned rows of X
 *   X_halo   h x f          the halo rows of X ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   perm     int32 [nnz]    for every transposed entry t, the forward entry it is (PgcnPlan.transposed_entries())
 * The walks are the gated aggregation's (pgcn_gated.h, PgcnPlan.gated_walks()): the forward CSR's work table for the
 * forward, the transposed CSR's for the backward. Split rows' chunk partials are summed in chunk order by a fixup
 * launch. work: nslots x f floats of the walk's table (NULL when nslots == 0).
 *
 * No atomics: every output element is a sum in one fixed order, so runs give the same bits. f % 4 == 0 with every
 * operand 16-byte aligned takes the float4 instances, anything else the scalar ones; both sum in the same order and
 * give the same bits. Calls are asynchronous on `stream`, allocate nothing and do no set-up: they are capturable in a
 * CUDA graph. Conventions as pgcn_b200.h: extern "C", 0 or a negative status, never throws. Arguments are checked
 * before any device work; with no device visible every call returns PGCN_GINE_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_GINE_H
#define PGCN_GINE_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_gine_status {
    PGCN_GINE_OK = 0,
    PGCN_GINE_ERR_INVALID = -1,   /* null pointer, bad width, inconsistent walk  */
    PGCN_GINE_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed       */
    PGCN_GINE_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path  */
} pgcn_gine_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_gine_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_gine_last_error(void);

/*
 * Load every kernel of this library on the current device; later calls on that device return at once. CUDA loads a
 * kernel lazily, at its first launch, and that load waits for the device. When several ranks share one process, a rank
 * whose stream holds an exchange waiting for a peer must not launch a kernel that is not loaded yet, or the peer's half
 * of the exchange is never enqueued: call this before the first exchange of a GINE layer (op.aggregate_gine does). Not
 * a stream operation: it may be called during a CUDA-graph capture.
 */
int pgcn_gine_load(void);

/*
 * Forward over the forward walk: Z (m x f) from X (own and halo rows) and E. Nothing per entry is written.
 */
int pgcn_gine_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* X_own, const float* X_halo,
                      const float* E, float* Z, float* work, int32_t f, void* stream);

/*
 * Backward, one column walk over the transposed walk: dX ((m + h) x f) for every column j in [0, m + h) and, unless
 * dE is NULL, dE (nnz x f), from X, E and gZ (m x f); the ReLU mask is recomputed from X and E. Rows [0, m) of dX are
 * the owned rows, rows [m, m + h) the halo partials in [halo by peer] order, what pgcn_halo_rows_add
 * (pgcn_b200_halo.h) returns to their owners. A NULL dE leaves dX's bits unchanged.
 */
int pgcn_gine_backward(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, const float* X_own,
                       const float* X_halo, const float* E, const float* gZ, float* dE, float* dX, float* work,
                       int32_t f, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_GINE_H */
