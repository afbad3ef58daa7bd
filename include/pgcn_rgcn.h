/*
 * pgcn_rgcn.h — C-ABI of the relational-aggregation library (lib/libpgcn_rgcn.so), sm_90a.
 *
 * The per-relation aggregation of R-GCN (Schlichtkrull et al., "Modeling Relational Data with Graph Convolutional
 * Networks"; PyG's RGCNConv, DGL's RelGraphConv) over the stored pattern of a rank's local matrix. Every stored entry
 * e = (i, j) carries a relation rel_e in [0, R) and a weight w_e; with X [m + h, f] (own rows, then halo rows):
 *
 *     Z[i, r]  = sum_{e in row i, rel_e = r} w_e * X[j]        Z [m, R, f], i.e. [m R, f] with virtual row v = i R + r
 *     dX[j]    = sum_{e in column j} w_e * gZ[i, rel_e]           j in [0, m + h)
 *
 * Each product is one rounded multiply (__fmul_rn) and each sum a chain of rounded adds (__fadd_rn) from +0; a NULL w
 * means w_e = 1, and then nothing is multiplied: the terms are X[j] and gZ[i, rel_e] themselves. The values of A are
 * not read; every stored entry contributes, duplicates included. A (row, relation) pair with no entries gives zeros.
 * +-inf and NaN propagate as IEEE arithmetic on these formulas.
 *
 * Both directions are one kernel: out[v] = sum_{e in item of v} w[perm[e]] * src[idx[e]], with src split into own rows
 * [0, split) and halo rows [split, ...). The caller's walks (pgcn_gated.h's struct and work tables,
 * PgcnPlan.relation_walks()) put R into the indices, so the kernel never sees it:
 *   forward   a CSR over the m R virtual rows: the forward entries sorted stably by (row, relation), perm = perm_f
 *             (the forward entry of each sorted entry), idx = colidx[perm_f] in [0, m + h); src = X_own, X_halo,
 *             split = m. A virtual row sums its entries in forward CSR order.
 *   backward  the transposed CSR over the m + h columns (perm = PgcnPlan.transposed_entries()), with
 *             idx = t_colidx R + rel[perm] in [0, m R); src = gZ as [m R, f], no halo rows. A column sums its entries in
 *             transposed-entry order (the stable column sort).
 * Rows longer than pgcn_gated_chunk() entries are split into chunks whose partial sums are added in chunk order by a
 * fixup launch. work: nslots x f floats of the walk's table (NULL when nslots == 0).
 *
 * w is fp32 [nnz], in the local forward CSR's entry order (the order of PgcnPlan.edge_pairs()), read as w[perm[e]].
 * Per-row and per-entry offsets are 64-bit, so m R f and nnz f may exceed 2^31; m R itself must fit in int32.
 *
 * Operands (fp32, row-major, DEVICE pointers):
 *   X_own    m x f          the owned rows of X
 *   X_halo   h x f          the halo rows of X ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   gZ       m R x f        the gradient of Z
 *   w        fp32 [nnz]     the entries' weights, or NULL (every weight 1)
 *   perm     int32 [nnz]    see above; may be NULL when w is NULL
 *
 * No atomics: every output element is a sum in one fixed order, so runs give the same bits. f % 4 == 0 with every
 * operand 16-byte aligned takes the float4 instances, anything else the scalar ones; both sum in the same order and
 * give the same bits. Calls are asynchronous on `stream`, allocate nothing and do no set-up: they are capturable in a
 * CUDA graph. Conventions as pgcn_b200.h: extern "C", 0 or a negative status, never throws. Arguments are checked
 * before any device work; with no device visible every call returns PGCN_RGCN_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_RGCN_H
#define PGCN_RGCN_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_rgcn_status {
    PGCN_RGCN_OK = 0,
    PGCN_RGCN_ERR_INVALID = -1,   /* null pointer, bad size or width, inconsistent walk */
    PGCN_RGCN_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed              */
    PGCN_RGCN_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path         */
} pgcn_rgcn_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_rgcn_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_rgcn_last_error(void);

/*
 * Load every kernel of this library on the current device; later calls on that device return at once. CUDA loads a
 * kernel lazily, at its first launch, and that load waits for the device. When several ranks share one process, a rank
 * whose stream holds an exchange waiting for a peer must not launch a kernel that is not loaded yet, or the peer's half
 * of the exchange is never enqueued: call this before the first exchange of a relational layer (op.aggregate_rgcn
 * does). Not a stream operation: it may be called during a CUDA-graph capture.
 */
int pgcn_rgcn_load(void);

/*
 * Forward over the relation walk (fwd->rows == m R): Z (m R x f) from X (own and halo rows).
 */
int pgcn_rgcn_forward(const pgcn_gated_walk* fwd, const int32_t* perm, int32_t m, int32_t h, int32_t R,
                      const float* X_own, const float* X_halo, const float* w, float* Z, float* work, int32_t f,
                      void* stream);

/*
 * Backward over the transposed relation walk (tr->rows == m + h): dX ((m + h) x f) for every column j in [0, m + h)
 * from gZ (m R x f). Rows [0, m) of dX are the owned rows, rows [m, m + h) the halo partials in [halo by peer] order,
 * what pgcn_halo_rows_add (pgcn_b200_halo.h) returns to their owners.
 */
int pgcn_rgcn_backward(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, int32_t R,
                       const float* gZ, const float* w, float* dX, float* work, int32_t f, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_RGCN_H */
