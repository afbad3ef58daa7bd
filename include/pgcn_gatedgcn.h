/*
 * pgcn_gatedgcn.h — C-ABI of the GatedGCN library (lib/libpgcn_gatedgcn.so), sm_90a.
 *
 * The edge-gated aggregation of GatedGCN (Bresson & Laurent, "Residual Gated Graph ConvNets", in the form of Dwivedi et
 * al., "Benchmarking Graph Neural Networks") over the stored pattern of a rank's local matrix, with an edge-feature
 * stream. For every stored entry e = (i, j) of row i and every feature:
 *
 *     ehat_e = (Dx[i] + Ex[j]) + Ce_e            fp32, summed in exactly this order
 *     s_e    = sigmoid(ehat_e)                   the gated aggregation's gate (pgcn_gated.h): rcp_rn(1 + expf(-x))
 *     num_i  = sum_{e in row i} s_e Bx[j],   den_i = sum_{e in row i} s_e
 *     Z[i]   = num_i / (den_i + eps)
 *
 * and its gradients from gZ (m x f) and gEhat (nnz x f, NULL meaning zero), with U[i] = gZ[i] / (den_i + eps):
 *
 *     dCe_e  = gEhat_e + U[i] (Bx[j] - Z[i]) s_e (1 - s_e)        (= d ehat_e)
 *     dDx[i] = sum_{e in row i} dCe_e,   dEx[j] = sum_{e in col j} dCe_e,   dBx[j] = sum_{e in col j} s_e U[i]
 *
 * s (1 - s) is evaluated as the gated aggregation evaluates it. A row without entries gives Z = 0 / eps (NaN when
 * eps == 0). The values of A are not read; every stored entry contributes, duplicates included. +-inf and NaN propagate
 * as IEEE arithmetic on these formulas.
 *
 * A per-entry tensor (Ce, ehat, gEhat, dCe) is nnz x f, row-major, in the local forward CSR's entry order (the order of
 * PgcnPlan.edge_pairs()); every per-entry offset is 64-bit, so nnz * f may exceed 2^31. It never crosses ranks: under
 * the 1-D row partition every entry belongs to the rank that owns its row.
 *
 * Operands (fp32, row-major, DEVICE pointers):
 *   Dx_own   m x f          destination side; only owned rows are read
 *   EB_own   m x 2f         Ex in columns [0, f), Bx in [f, 2f)
 *   EB_halo  h x 2f         the halo rows of EB ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   perm     int32 [nnz]    for every transposed entry t, the forward entry it is (PgcnPlan.transposed_entries())
 * The walks are the gated aggregation's (pgcn_gated.h, PgcnPlan.gated_walks()): the forward CSR's work table for the
 * forward and the row walk, the transposed CSR's for the column walk. Split rows' chunk partials are summed in chunk
 * order by a fixup launch. eps must be finite and >= 0.
 *
 * No atomics: every output element is a sum in one fixed order, so runs give the same bits. f % 4 == 0 with every
 * operand 16-byte aligned takes the float4 instances, anything else the scalar ones; both sum in the same order and
 * give the same bits. Calls are asynchronous on `stream`, allocate nothing and do no set-up: they are capturable in a
 * CUDA graph. Conventions as pgcn_b200.h: extern "C", 0 or a negative status, never throws. Arguments are checked
 * before any device work; with no device visible every call returns PGCN_GATEDGCN_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_GATEDGCN_H
#define PGCN_GATEDGCN_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_gatedgcn_status {
    PGCN_GATEDGCN_OK = 0,
    PGCN_GATEDGCN_ERR_INVALID = -1,   /* null pointer, bad width or eps, inconsistent walk */
    PGCN_GATEDGCN_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed            */
    PGCN_GATEDGCN_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path       */
} pgcn_gatedgcn_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_gatedgcn_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_gatedgcn_last_error(void);

/*
 * Load every kernel of this library on the current device; later calls on that device return at once. CUDA loads a
 * kernel lazily, at its first launch, and that load waits for the device. When several ranks share one process, a rank
 * whose stream holds an exchange waiting for a peer must not launch a kernel that is not loaded yet, or the peer's half
 * of the exchange is never enqueued: call this before the first exchange of a GatedGCN layer (op.aggregate_gatedgcn
 * does). Not a stream operation: it may be called during a CUDA-graph capture.
 */
int pgcn_gatedgcn_load(void);

/*
 * Forward over the forward walk: Ehat (nnz x f), Z (m x f) and den (m x f, the sums of the gates, without eps) from
 * Dx, [Ex | Bx] and Ce. work: nslots x 2f floats, the split rows' [num | den] chunk partials (NULL when nslots == 0).
 */
int pgcn_gatedgcn_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* Dx_own, const float* EB_own,
                          const float* EB_halo, const float* Ce, float eps, float* Z, float* den, float* Ehat,
                          float* work, int32_t f, void* stream);

/*
 * Backward, row walk over the forward walk: dCe (nnz x f), dDx (m x f) and U = gZ / (den + eps) (m x f), from the
 * forward's Ehat, Z and den, gZ (m x f) and gEhat (nnz x f, or NULL for zero). U is formed once per row, here, and the
 * column walk reads it. work: nslots x f floats.
 */
int pgcn_gatedgcn_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* EB_own,
                                const float* EB_halo, const float* Ehat, const float* gEhat, const float* Z,
                                const float* den, const float* gZ, float eps, float* U, float* dCe, float* dDx,
                                float* work, int32_t f, void* stream);

/*
 * Backward, column walk over the transposed walk: dEB ((m + h) x 2f) = [dEx | dBx] for every column j in [0, m + h),
 * from Ehat, dCe and U (pgcn_gatedgcn_backward_rows); perm names each transposed entry's forward entry. Rows [0, m) are
 * the owned rows, rows [m, m + h) the halo partials in [halo by peer] order, what pgcn_halo_rows_add
 * (pgcn_b200_halo.h) returns to their owners. The halo rows of EB are not read. work: nslots x 2f floats.
 */
int pgcn_gatedgcn_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h,
                                const float* Ehat, const float* dCe, const float* U, float* dEB, float* work,
                                int32_t f, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_GATEDGCN_H */
