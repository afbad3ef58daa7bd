/*
 * pgcn_gated.h — C-ABI of the gated-aggregation library (lib/libpgcn_gated.so), sm_90a.
 *
 * The message of PyG's ResGatedGraphConv (Bresson & Laurent, "Residual Gated Graph ConvNets") over the stored pattern
 * of a rank's local matrix, with a gate per entry and per feature:
 *
 *     eta_e = sigmoid(K[i] + Q[j])                 sigmoid(x) = 1 / (1 + expf(-x)), full-precision expf
 *     Z[i]  = sum over the stored entries e = (i, j) of row i of  eta_e * V[j]           (element-wise in the features)
 *
 * and its gradients, recomputed from K, Q and V instead of stored per entry:
 *
 *     dK[i] = gZ[i] * sum_{e in row i} V[j] * eta_e (1 - eta_e)
 *     dV[j] = sum_{e in col j} eta_e * gZ[i]
 *     dQ[j] = V[j] * sum_{e in col j} gZ[i] * eta_e (1 - eta_e)
 *
 * eta (1 - eta) is evaluated as eta * sigma(-x), with sigma(-x) = expf(-x) * eta (1 where expf(-x) overflows), so it
 * keeps its relative accuracy where eta rounds to 1. The values of A are not read; every stored entry contributes,
 * duplicates included. +-inf and NaN propagate as IEEE arithmetic on these formulas.
 *
 * Operands (fp32, row-major, DEVICE pointers):
 *   K_own   m x f          destination side; only owned rows are read
 *   QV_own  m x 2f         Q in columns [0, f), V in [f, 2f)
 *   QV_halo h x 2f         the halo rows of QV ([halo by peer], e.g. from pgcn_halo_rows); may be NULL when h == 0
 * A walk is a CSR's entries (idx) over `rows` rows plus its work table: `items` int32 [nitems, 4] of
 * (row, e0, e1, slot), one per row of at most pgcn_gated_chunk() entries (slot -1: written straight to the output) and
 * one per chunk of a longer row (slot >= 0: written to work[slot]); `splits` int32 [nsplits, 3] of (row, slot0, count):
 * the split rows, whose chunks' partials are summed in chunk order by a fixup launch. Every row appears in the table,
 * empty rows included. The forward and row walks take the local forward CSR (rows = m, columns in [0, m + h) laid out
 * [own | halo by peer]); the column walk takes the transposed CSR (rows = m + h, entries in [0, m)).
 *
 * No atomics: every output element is a sum in one fixed order, so runs give the same bits. f % 4 == 0 with every
 * operand 16-byte aligned takes the float4 instances, anything else the scalar ones; both sum in the same order and
 * give the same bits. Calls are asynchronous on `stream`, allocate nothing and do no set-up: they are capturable in a
 * CUDA graph. Conventions as pgcn_b200.h: extern "C", 0 or a negative status, never throws. Arguments are checked
 * before any device work; with no device visible every call returns PGCN_GATED_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_GATED_H
#define PGCN_GATED_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_gated_status {
    PGCN_GATED_OK = 0,
    PGCN_GATED_ERR_INVALID = -1,   /* null pointer, bad width or inconsistent walk   */
    PGCN_GATED_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed          */
    PGCN_GATED_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path     */
} pgcn_gated_status;

/* A walk: host struct of device pointers (see above). */
typedef struct pgcn_gated_walk {
    const int32_t* idx;        /* the CSR's entries: column ids (forward) or row ids (transposed) */
    const int32_t* items;      /* nitems x 4, 16-byte aligned  */
    const int32_t* splits;     /* nsplits x 3                  */
    int32_t rows;
    int32_t nitems;            /* at least rows                */
    int32_t nsplits;
    int32_t nslots;            /* rows of the caller's work buffer */
} pgcn_gated_walk;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_gated_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_gated_last_error(void);

/* Entries per work item: rows longer than this are split into chunks of this many entries. */
int32_t pgcn_gated_chunk(void);

/*
 * Forward: Z (m x f) from the forward walk. work: nslots x f floats (NULL when nslots == 0).
 */
int pgcn_gated_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* K_own, const float* QV_own,
                       const float* QV_halo, float* Z, float* work, int32_t f, void* stream);

/*
 * Backward, row walk: dK (m x f) from gZ (m x f) over the forward walk. work: nslots x f floats.
 */
int pgcn_gated_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, const float* K_own,
                             const float* QV_own, const float* QV_halo, const float* gZ, float* dK, float* work,
                             int32_t f, void* stream);

/*
 * Backward, column walk over the transposed walk: dQV ((m + h) x 2f) = [dQ | dV] for every column j in [0, m + h).
 * Rows [0, m) are the owned rows, rows [m, m + h) the halo partials in [halo by peer] order, what
 * pgcn_halo_rows_add (pgcn_b200_halo.h) returns to their owners. work: nslots x 2f floats.
 */
int pgcn_gated_backward_cols(const pgcn_gated_walk* tr, int32_t m, int32_t h, const float* K_own,
                             const float* QV_own, const float* QV_halo, const float* gZ, float* dQV, float* work,
                             int32_t f, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_GATED_H */
