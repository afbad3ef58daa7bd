/*
 * pgcn_b200_halo.h — the reverse halo exchange of the plan library (lib/libpgcn_b200.so), declared beside
 * pgcn_b200.h. pgcn_b200.h's list of functions is pinned (every one of them is classified, and the exchanging ones
 * are run out of step, by the test suite); entry points added to the plan library later are declared here.
 * Conventions as pgcn_b200.h.
 */
#ifndef PGCN_B200_HALO_H
#define PGCN_B200_HALO_H

#include "pgcn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * pgcn_halo_rows_add: the reverse of pgcn_halo_rows. X_halo is h x w, one row per halo row of this rank in [halo by
 * peer] order (e.g. partial gradients this rank computed for rows its peers own); each row goes back to the rank that
 * owns it, and every rank adds what it receives into G_own (m x w, in place). A row in several peers' send lists gets
 * every peer's partial, added in the fixed order of pgcn_backward's unpack. It is pgcn_backward's unsplit exchange
 * with a device-to-device copy of X_halo into the reverse send slab in place of the transposed SpMM: peer transport
 * when imported and w % 4 == 0 (the device epoch advances as in every fused call), NCCL otherwise. k == 1: nothing to
 * do. Needs pgcn_plan_bind_values (PGCN_ERR_STATE before); w outside (0, f_max] or a null argument returns
 * PGCN_ERR_INVALID. It does no set-up work of its own: after pgcn_plan_prepare(plan, w) it is capturable.
 */
int pgcn_halo_rows_add(pgcn_plan* plan, const float* X_halo, float* G_own, int32_t w, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_B200_HALO_H */
