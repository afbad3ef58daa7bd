/*
 * pgcn_gatv2_edge.h — C-ABI of GATv2 attention with edge features and attention dropout (lib/libpgcn_gatv2_edge.so),
 * sm_90a.
 *
 * The attention of PyG's GATv2Conv(edge_dim=..., dropout=p, concat=True, bias=False, add_self_loops=False) over the
 * stored pattern of a rank's local matrix, with XL = lin_l(x), XR = lin_r(x) and E = lin_edge(edge_attr) already
 * formed by the caller: K heads of width d = f / K concatenated, att[h, c] the flat feature h d + c, and for every
 * stored entry e = (i, j) of row i
 *
 *     t_e      = (XR[i] + XL[j]) + E_e                       (element-wise, each sum rounded to fp32, in this order)
 *     s_eh     = sum_c att[h, c] * LeakyReLU(t_e[h d + c])
 *     p_.h     = softmax of s_.h over row i's stored entries
 *     Z[i, h]  = sum_e  M_eh p_eh XL[j, h]                   (E enters the score only)
 *
 * M is the attention-dropout factor of pgcn_dropout.h (the mask pgcn_edge_dropout draws from the entries' global ids,
 * the head and the device int64[2] `drop`), 1 without dropout. The forward is one pass per row with an online softmax
 * and saves only the log-sum-exp L[i, h]. The row walk recomputes t, s and p = expf(s - L) per entry and, with
 * P = M p, D_ih = < gZ[i, h], Z[i, h] >, ds = p (M < gZ[i, h], XL[j, h] > - D) and
 * g_ec = ds_eh(c) att_c LeakyReLU'(t_ec) (LeakyReLU' is 1 for t > 0 and negative_slope otherwise), writes
 *
 *     G_e      = g_e                                         (dE; caller scratch when E needs no gradient)
 *     PS_e     = [P_e | ds_e]                                (2K floats per entry)
 *     dXR[i]   = sum_{e in row i} g_e
 *     datt[c]  = sum_e ds_eh(c) LeakyReLU(t_ec)              (per-CTA partials, then one ordered column reduction)
 *
 * and the column walk reads PS and G through the transposed entries' forward entries, with no score recomputed:
 *
 *     dXL[j]   = sum_{e in col j} (P_eh(c) gZ[i, c] + g_ec)
 *
 * The values of A are not read; every stored entry contributes, duplicates included. A row without entries gives
 * Z = 0. +-inf and NaN propagate as IEEE arithmetic on these formulas.
 *
 * Operands (fp32, row-major, DEVICE pointers); heads in {1, 2, 4, 8}, f % heads == 0, 1 <= f <= 256:
 *   XL_own   m x f          the source side of the owned rows
 *   XL_halo  h x f          its halo rows ([halo by peer], from pgcn_halo_rows); may be NULL when h == 0
 *   XR       m x f          the destination side of the owned rows
 *   att      f              [heads, d], row-major
 *   E        nnz x f        the edge term of every local entry, in the forward CSR's entry order (PgcnPlan.edge_pairs())
 *   gid      int32 [m + h]  global ids of the owned rows, then of the halo rows; read only when drop != NULL
 *   drop     NULL (no dropout) or a device int64 [key, c]; threshold and keep_scale as op.dropout_constants(p)
 *   perm     int32 [nnz]    the forward entry of every transposed entry (PgcnPlan.transposed_entries())
 * Per-entry offsets are 64-bit. The walks are the gated aggregation's (pgcn_gated.h, PgcnPlan.gated_walks()).
 * negative_slope must be finite.
 *
 * No atomics: every output element is reduced in one fixed order, so runs give the same bits. With d % 4 == 0 and
 * every feature operand (att, E and G included) 16-byte aligned the float4 instances load and store the features,
 * otherwise the scalar instances do the same work feature by feature, with the same bits. Calls are asynchronous on
 * `stream`, allocate nothing and do no set-up: they are capturable in a CUDA graph. Conventions as pgcn_b200.h:
 * extern "C", 0 or a negative status, never throws. Arguments are checked before any device work; with no device
 * visible every call returns PGCN_GATV2_EDGE_ERR_NOGPU (there is no CPU path).
 */
#ifndef PGCN_GATV2_EDGE_H
#define PGCN_GATV2_EDGE_H

#include <stdint.h>

#include "pgcn_gated.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_gatv2_edge_status {
    PGCN_GATV2_EDGE_OK = 0,
    PGCN_GATV2_EDGE_ERR_INVALID = -1,   /* null pointer, bad width or head count, inconsistent walk */
    PGCN_GATV2_EDGE_ERR_CUDA = -2,      /* a CUDA runtime call or a launch failed                   */
    PGCN_GATV2_EDGE_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path              */
} pgcn_gatv2_edge_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_gatv2_edge_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_gatv2_edge_last_error(void);

/*
 * Rows of f floats the row walk's `work` needs for the forward walk `fwd`: its nslots split-row partials, then one
 * datt partial per CTA of the walk. -1 for a NULL walk. Host only: no device is touched.
 */
int64_t pgcn_gatv2_edge_work_rows(const pgcn_gated_walk* fwd);

/*
 * Load every kernel of this library on the current device now. CUDA loads a kernel at its first launch and that load
 * waits for the device; with several ranks in one process, a first launch queued behind an exchange that waits on a
 * later rank would never return. Call it before the first exchange; later calls return at once.
 */
int pgcn_gatv2_edge_load(void);

/*
 * Forward over the forward walk: Z (m x f) and L (m x heads). work: nslots x (f + 2 heads) floats, the split rows'
 * chunk partials (accumulator, running max, running sum), merged in chunk order (NULL when nslots == 0).
 */
int pgcn_gatv2_edge_forward(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads, const float* XL_own,
                            const float* XL_halo, const float* XR, const float* att, const float* E,
                            float negative_slope, const int32_t* gid, const int64_t* drop, uint32_t threshold,
                            float keep_scale, float* Z, float* L, float* work, int32_t f, void* stream);

/*
 * Backward, row walk over the forward walk: dXR (m x f), D (m x heads), PS (nnz x 2 heads: [P | ds] per entry), G
 * (nnz x f: g per entry, read by the column walk) and datt (f) from gZ, the forward's Z and L, and the same drop
 * snapshot as the forward. D is computed once per row. work: pgcn_gatv2_edge_work_rows(fwd) x f floats.
 */
int pgcn_gatv2_edge_backward_rows(const pgcn_gated_walk* fwd, int32_t m, int32_t h, int32_t heads,
                                  const float* XL_own, const float* XL_halo, const float* XR, const float* att,
                                  const float* E, float negative_slope, const int32_t* gid, const int64_t* drop,
                                  uint32_t threshold, float keep_scale, const float* gZ, const float* Z,
                                  const float* L, float* dXR, float* D, float* PS, float* G, float* datt, float* work,
                                  int32_t f, void* stream);

/*
 * Backward, column walk over the transposed walk: dXL ((m + h) x f) for every column j in [0, m + h), from gZ and the
 * row walk's PS and G read through perm. Rows [0, m) are the owned rows, rows [m, m + h) the halo partials in
 * [halo by peer] order, what pgcn_halo_rows_add (pgcn_b200_halo.h) returns to their owners. work: nslots x f.
 */
int pgcn_gatv2_edge_backward_cols(const pgcn_gated_walk* tr, const int32_t* perm, int32_t m, int32_t h, int32_t heads,
                                  const float* gZ, const float* PS, const float* G, float* dXL, float* work, int32_t f,
                                  void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_GATV2_EDGE_H */
