/*
 * pgcn_transformer_edge.h — C-ABI of the graph-transformer attention with edge features
 * (lib/libpgcn_transformer_edge.so), sm_90a.
 *
 * The attention of PyG's TransformerConv(edge_dim=..., concat=True, beta=False) over the stored pattern of a rank's
 * local matrix, with E = lin_edge(edge_attr) already formed by the caller: K heads of width C = f / K concatenated, and
 * for every stored entry e = (i, j) of row i
 *
 *     kk_e     = k[j] + E_e,   vv_e = v[j] + E_e            (element-wise, each sum rounded to fp32 first)
 *     s_eh     = scale * < q[i, h], kk_e[h] >
 *     alpha_.h = softmax of s_.h over row i's stored entries
 *     Z[i, h]  = sum_e  M_eh alpha_eh vv_e[h]
 *
 * M is the attention-dropout factor of pgcn_transformer.h (the mask pgcn_edge_dropout draws from the entries' global
 * ids and the device int64[2] `drop`). The forward is one pass per row with an online softmax and saves only the
 * log-sum-exp L[i, h]. The row walk recomputes p = expf(s - L) per entry and, with P = M p, D = < gZ, Z > and
 * ds = p (M < gZ[i, h], vv_e[h] > - D), writes
 *
 *     dQ[i]    = scale * sum_{e in row i} ds_e kk_e
 *     dE_e     = P_e gZ[i] + scale ds_e q[i]                 (per head)
 *     PS_e     = [P_e | ds_e]                               (2K floats per entry)
 *
 * and the column walk reads PS through the transposed entries' forward entries, with no score recomputed:
 *
 *     dK[j]    = scale * sum_{e in col j} ds_e q[i],     dV[j] = sum_{e in col j} P_e gZ[i]
 *
 * The values of A are not read; every stored entry contributes, duplicates included. A row without entries gives
 * Z = 0. +-inf and NaN propagate as IEEE arithmetic on these formulas. With E = 0 every output has the bits of
 * pgcn_transformer.h's.
 *
 * Operands (fp32, row-major, DEVICE pointers); heads in {1, 2, 4, 8}, f % heads == 0, 1 <= f <= 256:
 *   Q_own    m x f          the destination rows' queries
 *   KV_own   m x 2f         k in columns [0, f), v in [f, 2f)
 *   KV_halo  h x 2f         the halo rows of KV ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   E        nnz x f        the edge term of every local entry, in the forward CSR's entry order (PgcnPlan.edge_pairs())
 *   gid      int32 [m + h]  global ids of the owned rows, then of the halo rows; read only when drop != NULL
 *   drop     NULL (no dropout) or a device int64 [key, c]; threshold and keep_scale as op.dropout_constants(p)
 *   perm     int32 [nnz]    the forward entry of every transposed entry (PgcnPlan.transposed_entries())
 * Per-entry offsets are 64-bit. The walks are the gated aggregation's (pgcn_gated.h, PgcnPlan.gated_walks()).
 *
 * No atomics: every output element is reduced in one fixed order, so runs give the same bits. With C % 4 == 0 and
 * every feature operand (E and dE included) 16-byte aligned the float4 instances load and store the features,
 * otherwise the scalar instances do the same work feature by feature, with the same bits. Calls are asynchronous on
 * `stream`, allocate nothing and do no set-up: they are capturable in a CUDA graph. Conventions as pgcn_b200.h:
 * extern "C", 0 or a negative status, never throws. Arguments are checked before any device work; with no device
 * visible every call returns PGCN_TRANSFORMER_EDGE_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_TRANSFORMER_EDGE_H
#define PGCN_TRANSFORMER_EDGE_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_transformer_edge_status {
    PGCN_TRANSFORMER_EDGE_OK = 0,
    PGCN_TRANSFORMER_EDGE_ERR_INVALID = -1,   /* null pointer, bad width or head count, inconsistent walk */
    PGCN_TRANSFORMER_EDGE_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed                   */
    PGCN_TRANSFORMER_EDGE_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path              */
} pgcn_transformer_edge_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_transformer_edge_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_transformer_edge_last_error(void);

/*
 * Load every kernel of this library on the current device now. CUDA loads a kernel at its first launch and that load
 * waits for the device; with several ranks in one process, a first launch queued behind an exchange that waits on a
 * later rank would never return. Call it before the first exchange; later calls return at once.
 */
int pgcn_transformer_edge_load(void);

/*
 * Forward over the forward walk: Z (m x f) and L (m x heads). work: nslots x (f + 2 heads) floats, the split rows'
 * chunk partials (accumulator, running max, running sum), merged in chunk order (NULL when nslots == 0).
 */
int pgcn_transformer_edge_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* Q_own,
                                  const float* KV_own, const float* KV_halo, const float* E, float scale,
                                  const int32_t* gid, const int64_t* drop, uint32_t threshold, float keep_scale,
                                  float* Z, float* L, float* work, int32_t f, void* stream);

/*
 * Backward, row walk over the forward walk: dQ (m x f), D (m x heads), PS (nnz x 2 heads: [P | ds] per entry) and dE
 * (nnz x f; NULL when E needs no gradient, and then nothing is written) from gZ, the forward's Z and L, and the same
 * drop snapshot as the forward. D is computed once per row. work: nslots x f floats.
 */
int pgcn_transformer_edge_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                        const float* Q_own, const float* KV_own, const float* KV_halo, const float* E,
                                        float scale, const int32_t* gid, const int64_t* drop, uint32_t threshold,
                                        float keep_scale, const float* gZ, const float* Z, const float* L, float* dQ,
                                        float* D, float* PS, float* dE, float* work, int32_t f, void* stream);

/*
 * Backward, column walk over the transposed walk: dKV ((m + h) x 2f) = [dK | dV] for every column j in [0, m + h), from
 * Q, gZ and the row walk's PS read through perm. Rows [0, m) are the owned rows, rows [m, m + h) the halo partials in
 * [halo by peer] order, what pgcn_halo_rows_add (pgcn_b200_halo.h) returns to their owners. work: nslots x 2f.
 */
int pgcn_transformer_edge_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h,
                                        int32_t heads, const float* Q_own, const float* gZ, const float* PS,
                                        float scale, float* dKV, float* work, int32_t f, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_TRANSFORMER_EDGE_H */
