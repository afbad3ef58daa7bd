/*
 * pgcn_transformer.h — C-ABI of the graph-transformer attention library (lib/libpgcn_transformer.so), sm_90a.
 *
 * Scaled dot-product attention over the stored pattern of a rank's local matrix, the attention of PyG's
 * TransformerConv (Shi et al., "Masked Label Prediction", UniMP) and of the graph transformer layer of Dwivedi &
 * Bresson, with K heads of width C = f / K concatenated:
 *
 *     s_eh     = scale * < q[i, h], k[j, h] >                 for every stored entry e = (i, j) of row i
 *     alpha_.h = softmax of s_.h over row i's stored entries
 *     Z[i, h]  = sum_e  M_eh alpha_eh v[j, h]
 *
 * M is the attention-dropout factor: keep_scale where the mask keeps (e, h), 0 where it drops, 1 without dropout.
 * The mask is the one pgcn_edge_dropout (pgcn_dropout.h) draws: entry (gid[i], gid[j]), head h is kept iff word h & 3
 * of Philox4x32-10(counter = (gid[i], gid[j], c, h >> 2), key) >= threshold, with [key, c] read from the device
 * int64[2] `drop`; so every partition of a graph draws the same mask. The forward is one pass per row with an online
 * softmax (a running max, a running sum and an accumulator rescaled as entries arrive) and saves only
 * L[i, h] = max + log(sum), the log-sum-exp of the row's scores. The backward recomputes p = expf(s - L) per entry:
 *
 *     D[i, h]  = < gZ[i, h], Z[i, h] >
 *     ds_eh    = p_eh (M_eh dp_eh - D[i, h]),   dp_eh = < gZ[i, h], v[j, h] >
 *     dQ[i]    = scale * sum_{e in row i} ds_e k[j]
 *     dK[j]    = scale * sum_{e in col j} ds_e q[i],     dV[j] = sum_{e in col j} M_e p_e gZ[i]
 *
 * The values of A are not read; every stored entry contributes, duplicates included. A row without entries gives
 * Z = 0 (its L is -inf and never read). +-inf and NaN propagate as IEEE arithmetic on these formulas, evaluated in
 * the order the kernels use (tests/transformer_oracle.py restates it).
 *
 * Operands (fp32, row-major, DEVICE pointers); heads in {1, 2, 4, 8}, f % heads == 0, 1 <= f <= 256 (a row's q and its
 * accumulators live in registers):
 *   Q_own    m x f          the destination rows' queries
 *   KV_own   m x 2f         k in columns [0, f), v in [f, 2f)
 *   KV_halo  h x 2f         the halo rows of KV ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   gid      int32 [m + h]  global ids of the owned rows, then of the halo rows; read only when drop != NULL
 *   drop     NULL (no dropout) or a device int64 [key, c]; threshold and keep_scale as op.dropout_constants(p)
 * The walks are the gated aggregation's (pgcn_gated.h, PgcnPlan.gated_walks()): the forward CSR's work table for the
 * forward and the row walk, the transposed CSR's for the column walk. The kernels take the chunking from the table.
 *
 * No atomics: every output element is reduced in one fixed order, so runs give the same bits. Each head's features
 * sit on 32 / K lanes of a warp, 4 consecutive features per lane per pass; with C % 4 == 0 and every feature operand
 * 16-byte aligned the float4 instances load them, otherwise the scalar instances load the same features one by one
 * onto the same lanes and reduce them in the same order: both give the same bits. Calls are asynchronous on `stream`,
 * allocate nothing and do no set-up: they are capturable in a CUDA graph. Conventions as pgcn_b200.h: extern "C",
 * 0 or a negative status, never throws. Arguments are checked before any device work; with no device visible every
 * call returns PGCN_TRANSFORMER_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_TRANSFORMER_H
#define PGCN_TRANSFORMER_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_transformer_status {
    PGCN_TRANSFORMER_OK = 0,
    PGCN_TRANSFORMER_ERR_INVALID = -1,   /* null pointer, bad width or head count, inconsistent walk */
    PGCN_TRANSFORMER_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed                   */
    PGCN_TRANSFORMER_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path              */
} pgcn_transformer_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_transformer_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_transformer_last_error(void);

/*
 * Forward over the forward walk: Z (m x f) and L (m x heads). work: nslots x (f + 2 heads) floats, the split rows'
 * chunk partials (accumulator, running max, running sum), merged in chunk order (NULL when nslots == 0).
 */
int pgcn_transformer_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* Q_own,
                             const float* KV_own, const float* KV_halo, float scale, const int32_t* gid,
                             const int64_t* drop, uint32_t threshold, float keep_scale, float* Z, float* L, float* work,
                             int32_t f, void* stream);

/*
 * Backward, row walk over the forward walk: dQ (m x f) and D (m x heads) from gZ, the forward's Z and L, and the same
 * drop snapshot as the forward. D is computed once per row. work: nslots x f floats.
 */
int pgcn_transformer_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                   const float* Q_own, const float* KV_own, const float* KV_halo, float scale,
                                   const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                   const float* gZ, const float* Z, const float* L, float* dQ, float* D, float* work,
                                   int32_t f, void* stream);

/*
 * Backward, column walk over the transposed walk: dKV ((m + h) x 2f) = [dK | dV] for every column j in [0, m + h),
 * from gZ, L and D (pgcn_transformer_backward_rows). Rows [0, m) are the owned rows, rows [m, m + h) the halo partials
 * in [halo by peer] order, what pgcn_halo_rows_add (pgcn_b200_halo.h) returns to their owners. work: nslots x 2f.
 */
int pgcn_transformer_backward_cols(const pgcn_gated_walk* tr, int32_t m, int32_t h, int32_t heads,
                                   const float* Q_own, const float* KV_own, const float* KV_halo, float scale,
                                   const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                   const float* gZ, const float* L, const float* D, float* dKV, float* work, int32_t f,
                                   void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_TRANSFORMER_H */
