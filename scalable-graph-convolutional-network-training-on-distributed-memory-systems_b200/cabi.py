"""ctypes binding of include/pgcn_b200.h — the C-ABI drop-in boundary (SURVEY.md §8b) — and of include/pgcn_b200_halo.h,
include/pgcn_dropout.h, include/pgcn_gated.h, include/pgcn_transformer.h, include/pgcn_gatedgcn.h,
include/pgcn_transformer_edge.h, include/pgcn_gine.h and include/pgcn_rgcn.h.

Nothing here computes: it loads lib/libpgcn_b200.so (load), lib/libpgcn_dropout.so (load_dropout) and
lib/libpgcn_gated.so (load_gated), lib/libpgcn_transformer.so (load_transformer), lib/libpgcn_gatedgcn.so
(load_gatedgcn), lib/libpgcn_transformer_edge.so (load_transformer_edge), lib/libpgcn_gine.so (load_gine) and lib/libpgcn_rgcn.so (load_rgcn), declares every exported symbol and turns negative status codes into RuntimeError. If the library is missing there is no fallback: the
product path fails loudly (the CPU oracle under oracle/ is test infrastructure only).
"""
import ctypes as C
import os

from . import build as _build

P2P_HANDLE_BYTES = 512
NCCL_ID_BYTES = 128

# every symbol declared in include/pgcn_b200.h
SYMBOLS = [
    "pgcn_version", "pgcn_device_count", "pgcn_last_error",
    "pgcn_plan_create", "pgcn_plan_destroy", "pgcn_plan_set_option", "pgcn_plan_get_option",
    "pgcn_plan_autotune", "pgcn_plan_prepare", "pgcn_debug_schedule", "pgcn_plan_slab", "pgcn_algorithmic_bytes", "pgcn_launch_count",
    "pgcn_comm_unique_id", "pgcn_comm_init", "pgcn_comm_share", "pgcn_p2p_export", "pgcn_p2p_import",
    "pgcn_spmm", "pgcn_pack", "pgcn_exchange", "pgcn_unpack_add",
    "pgcn_forward", "pgcn_backward", "pgcn_forward_host", "pgcn_forward_host_async", "pgcn_forward_host_wait",
    "pgcn_plan_bind_values", "pgcn_plan_set_values", "pgcn_sddmm", "pgcn_forward_keep_halo",
    "pgcn_edge_softmax", "pgcn_edge_softmax_backward", "pgcn_halo_rows",
    "pgcn_edge_softmax_heads", "pgcn_edge_softmax_backward_heads", "pgcn_forward_heads", "pgcn_backward_heads",
    "pgcn_sddmm_heads", "pgcn_forward_max", "pgcn_backward_max", "pgcn_forward_gatv2", "pgcn_backward_gatv2",
]

# every symbol declared in include/pgcn_b200_halo.h (exported by libpgcn_b200.so as well)
HALO_SYMBOLS = ["pgcn_halo_rows_add"]

# every symbol declared in include/pgcn_dropout.h
DROPOUT_SYMBOLS = ["pgcn_dropout_version", "pgcn_dropout_last_error", "pgcn_edge_dropout"]

# every symbol declared in include/pgcn_gated.h
GATED_SYMBOLS = ["pgcn_gated_version", "pgcn_gated_last_error", "pgcn_gated_chunk", "pgcn_gated_forward",
                 "pgcn_gated_backward_rows", "pgcn_gated_backward_cols"]

# every symbol declared in include/pgcn_transformer.h
TRANSFORMER_SYMBOLS = ["pgcn_transformer_version", "pgcn_transformer_last_error", "pgcn_transformer_forward",
                       "pgcn_transformer_backward_rows", "pgcn_transformer_backward_cols"]

# every symbol declared in include/pgcn_gatedgcn.h
GATEDGCN_SYMBOLS = ["pgcn_gatedgcn_version", "pgcn_gatedgcn_last_error", "pgcn_gatedgcn_load",
                    "pgcn_gatedgcn_forward", "pgcn_gatedgcn_backward_rows", "pgcn_gatedgcn_backward_cols"]

# every symbol declared in include/pgcn_transformer_edge.h
TRANSFORMER_EDGE_SYMBOLS = ["pgcn_transformer_edge_version", "pgcn_transformer_edge_last_error",
                            "pgcn_transformer_edge_load", "pgcn_transformer_edge_forward",
                            "pgcn_transformer_edge_backward_rows", "pgcn_transformer_edge_backward_cols"]

# every symbol declared in include/pgcn_gine.h
GINE_SYMBOLS = ["pgcn_gine_version", "pgcn_gine_last_error", "pgcn_gine_load", "pgcn_gine_forward",
                "pgcn_gine_backward"]

# every symbol declared in include/pgcn_rgcn.h
RGCN_SYMBOLS = ["pgcn_rgcn_version", "pgcn_rgcn_last_error", "pgcn_rgcn_load", "pgcn_rgcn_forward",
                "pgcn_rgcn_backward"]

# every symbol declared in include/pgcn_gatv2_edge.h
GATV2_EDGE_SYMBOLS = ["pgcn_gatv2_edge_version", "pgcn_gatv2_edge_last_error", "pgcn_gatv2_edge_work_rows",
                      "pgcn_gatv2_edge_load", "pgcn_gatv2_edge_forward", "pgcn_gatv2_edge_backward_rows",
                      "pgcn_gatv2_edge_backward_cols"]


class PgcnBytes(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        "nnz", "m", "h", "cols_ref", "spmm_fwd", "spmm_bwd", "gather_fwd", "xchg_out", "xchg_in", "pack")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class PgcnGatedWalk(C.Structure):
    """pgcn_gated_walk: a CSR's entries and its work table, device pointers."""
    _fields_ = [("idx", C.c_void_p), ("items", C.c_void_p), ("splits", C.c_void_p), ("rows", C.c_int32),
                ("nitems", C.c_int32), ("nsplits", C.c_int32), ("nslots", C.c_int32)]


_lib = None
_dropout = None
_gated = None
_transformer = None
_gatedgcn = None
_transformer_edge = None
_gine = None
_rgcn = None
_gatv2_edge = None


def lib_path():
    return _build.LIB


def dropout_lib_path():
    return _build.DROPOUT_LIB


def gated_lib_path():
    return _build.GATED_LIB


def transformer_lib_path():
    return _build.TRANSFORMER_LIB


def gatedgcn_lib_path():
    return _build.GATEDGCN_LIB


def transformer_edge_lib_path():
    return _build.TRANSFORMER_EDGE_LIB


def gine_lib_path():
    return _build.GINE_LIB


def rgcn_lib_path():
    return _build.RGCN_LIB


def gatv2_edge_lib_path():
    return _build.GATV2_EDGE_LIB


def _built(path, stale, build, build_if_missing):
    """path, rebuilt first when stale and nvcc is available; a missing library raises."""
    if build_if_missing and stale():
        try:
            build()
        except RuntimeError:
            if not os.path.exists(path):
                raise
    if not os.path.exists(path):
        raise RuntimeError("%s is missing (%s): build it with __graft_entry__.build(); there is no CPU fallback for "
                           "the PGCN hot path" % (os.path.basename(path), path))
    return path


def load(build_if_missing=True):
    """Load libpgcn_b200.so (building it first when stale and nvcc is available)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _built(_build.LIB, _build.is_stale, _build.build, build_if_missing)
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.pgcn_version.restype = C.c_char_p
    lib.pgcn_version.argtypes = []
    lib.pgcn_device_count.restype = C.c_int
    lib.pgcn_device_count.argtypes = []
    lib.pgcn_last_error.restype = C.c_char_p
    lib.pgcn_last_error.argtypes = [vp]
    lib.pgcn_plan_create.restype = C.c_int
    lib.pgcn_plan_create.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, i32, C.POINTER(vp)]
    lib.pgcn_plan_destroy.restype = C.c_int
    lib.pgcn_plan_destroy.argtypes = [vp]
    lib.pgcn_plan_set_option.restype = C.c_int
    lib.pgcn_plan_set_option.argtypes = [vp, C.c_char_p, i64]
    lib.pgcn_plan_get_option.restype = i64
    lib.pgcn_plan_get_option.argtypes = [vp, C.c_char_p]
    lib.pgcn_plan_autotune.restype = C.c_int
    lib.pgcn_plan_autotune.argtypes = [vp, i32]
    lib.pgcn_plan_prepare.restype = C.c_int
    lib.pgcn_plan_prepare.argtypes = [vp, i32]
    lib.pgcn_debug_schedule.restype = i64
    lib.pgcn_debug_schedule.argtypes = [vp, i32, i64, i64, vp, i64, vp, vp]
    lib.pgcn_plan_slab.restype = vp
    lib.pgcn_plan_slab.argtypes = [vp, C.c_int]
    lib.pgcn_algorithmic_bytes.restype = C.c_int
    lib.pgcn_algorithmic_bytes.argtypes = [vp, i32, C.POINTER(PgcnBytes)]
    lib.pgcn_launch_count.restype = i64
    lib.pgcn_launch_count.argtypes = [vp]
    lib.pgcn_comm_unique_id.restype = C.c_int
    lib.pgcn_comm_unique_id.argtypes = [vp]
    lib.pgcn_comm_init.restype = C.c_int
    lib.pgcn_comm_init.argtypes = [vp, vp]
    lib.pgcn_p2p_export.restype = C.c_int
    lib.pgcn_p2p_export.argtypes = [vp, vp]
    lib.pgcn_p2p_import.restype = C.c_int
    lib.pgcn_p2p_import.argtypes = [vp, vp]
    lib.pgcn_spmm.restype = C.c_int
    lib.pgcn_spmm.argtypes = [vp, C.c_int, vp, vp, vp, vp, i32, vp]
    lib.pgcn_pack.restype = C.c_int
    lib.pgcn_pack.argtypes = [vp, vp, vp, i32, vp]
    lib.pgcn_exchange.restype = C.c_int
    lib.pgcn_exchange.argtypes = [vp, vp, vp, i32, C.c_int, vp]
    lib.pgcn_unpack_add.restype = C.c_int
    lib.pgcn_unpack_add.argtypes = [vp, vp, vp, i32, vp]
    lib.pgcn_forward.restype = C.c_int
    lib.pgcn_forward.argtypes = [vp, vp, vp, i32, vp]
    lib.pgcn_backward.restype = C.c_int
    lib.pgcn_backward.argtypes = [vp, vp, vp, i32, vp]
    lib.pgcn_forward_host.restype = C.c_int
    lib.pgcn_forward_host.argtypes = [vp, vp, vp, i32]
    lib.pgcn_comm_share.restype = C.c_int
    lib.pgcn_comm_share.argtypes = [vp, vp]
    lib.pgcn_forward_host_async.restype = C.c_int
    lib.pgcn_forward_host_async.argtypes = [vp, vp, vp, i32]
    lib.pgcn_forward_host_wait.restype = C.c_int
    lib.pgcn_forward_host_wait.argtypes = [vp]
    lib.pgcn_plan_bind_values.restype = C.c_int
    lib.pgcn_plan_bind_values.argtypes = [vp]
    lib.pgcn_plan_set_values.restype = C.c_int
    lib.pgcn_plan_set_values.argtypes = [vp, vp, vp]
    lib.pgcn_sddmm.restype = C.c_int
    lib.pgcn_sddmm.argtypes = [vp, vp, vp, vp, vp, i32, vp]
    lib.pgcn_forward_keep_halo.restype = C.c_int
    lib.pgcn_forward_keep_halo.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.pgcn_edge_softmax.restype = C.c_int
    lib.pgcn_edge_softmax.argtypes = [vp, vp, vp, vp, C.c_float, vp, vp]
    lib.pgcn_edge_softmax_backward.restype = C.c_int
    lib.pgcn_edge_softmax_backward.argtypes = [vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    lib.pgcn_halo_rows.restype = C.c_int
    lib.pgcn_halo_rows.argtypes = [vp, vp, vp, i32, vp]
    lib.pgcn_edge_softmax_heads.restype = C.c_int
    lib.pgcn_edge_softmax_heads.argtypes = [vp, i32, vp, vp, vp, C.c_float, vp, vp]
    lib.pgcn_edge_softmax_backward_heads.restype = C.c_int
    lib.pgcn_edge_softmax_backward_heads.argtypes = [vp, i32, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    lib.pgcn_forward_heads.restype = C.c_int
    lib.pgcn_forward_heads.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp]
    lib.pgcn_backward_heads.restype = C.c_int
    lib.pgcn_backward_heads.argtypes = [vp, i32, vp, vp, vp, i32, vp]
    lib.pgcn_sddmm_heads.restype = C.c_int
    lib.pgcn_sddmm_heads.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp]
    lib.pgcn_forward_max.restype = C.c_int
    lib.pgcn_forward_max.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.pgcn_backward_max.restype = C.c_int
    lib.pgcn_backward_max.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.pgcn_forward_gatv2.restype = C.c_int
    lib.pgcn_forward_gatv2.argtypes = [vp, i32, vp, vp, vp, C.c_float, vp, vp, vp, i32, vp]
    lib.pgcn_backward_gatv2.restype = C.c_int
    lib.pgcn_backward_gatv2.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp, vp, i32, vp]
    lib.pgcn_halo_rows_add.restype = C.c_int
    lib.pgcn_halo_rows_add.argtypes = [vp, vp, vp, i32, vp]
    _lib = lib
    return lib


def check(rc, plan=None):
    """Raise RuntimeError carrying pgcn_last_error when a C-ABI call returned a negative status."""
    if rc < 0:
        msg = load().pgcn_last_error(plan)
        raise RuntimeError("pgcn_b200 error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_dropout(build_if_missing=True):
    """Load libpgcn_dropout.so (building it first when stale and nvcc is available)."""
    global _dropout
    if _dropout is not None:
        return _dropout
    lib = C.CDLL(_built(_build.DROPOUT_LIB, _build.dropout_is_stale, _build.build_dropout, build_if_missing))
    lib.pgcn_dropout_version.restype = C.c_char_p
    lib.pgcn_dropout_version.argtypes = []
    lib.pgcn_dropout_last_error.restype = C.c_char_p
    lib.pgcn_dropout_last_error.argtypes = []
    lib.pgcn_edge_dropout.restype = C.c_int
    lib.pgcn_edge_dropout.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_uint32, C.c_float, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]
    _dropout = lib
    return lib


def check_dropout(rc):
    """Raise RuntimeError carrying pgcn_dropout_last_error when a libpgcn_dropout call returned a negative status."""
    if rc < 0:
        msg = load_dropout().pgcn_dropout_last_error()
        raise RuntimeError("pgcn_dropout error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_gated(build_if_missing=True):
    """Load libpgcn_gated.so (building it first when stale and nvcc is available)."""
    global _gated
    if _gated is not None:
        return _gated
    lib = C.CDLL(_built(_build.GATED_LIB, _build.gated_is_stale, _build.build_gated, build_if_missing))
    vp, i32, walk = C.c_void_p, C.c_int32, C.POINTER(PgcnGatedWalk)
    lib.pgcn_gated_version.restype = C.c_char_p
    lib.pgcn_gated_version.argtypes = []
    lib.pgcn_gated_last_error.restype = C.c_char_p
    lib.pgcn_gated_last_error.argtypes = []
    lib.pgcn_gated_chunk.restype = i32
    lib.pgcn_gated_chunk.argtypes = []
    lib.pgcn_gated_forward.restype = C.c_int
    lib.pgcn_gated_forward.argtypes = [walk, i32, i32, vp, vp, vp, vp, vp, i32, vp]
    lib.pgcn_gated_backward_rows.restype = C.c_int
    lib.pgcn_gated_backward_rows.argtypes = [walk, i32, i32, vp, vp, vp, vp, vp, vp, i32, vp]
    lib.pgcn_gated_backward_cols.restype = C.c_int
    lib.pgcn_gated_backward_cols.argtypes = [walk, i32, i32, vp, vp, vp, vp, vp, vp, i32, vp]
    _gated = lib
    return lib


def check_gated(rc):
    """Raise RuntimeError carrying pgcn_gated_last_error when a libpgcn_gated call returned a negative status."""
    if rc < 0:
        msg = load_gated().pgcn_gated_last_error()
        raise RuntimeError("pgcn_gated error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_transformer(build_if_missing=True):
    """Load libpgcn_transformer.so (building it first when stale and nvcc is available)."""
    global _transformer
    if _transformer is not None:
        return _transformer
    lib = C.CDLL(_built(_build.TRANSFORMER_LIB, _build.transformer_is_stale, _build.build_transformer,
                        build_if_missing))
    vp, i32, u32, f32, walk = C.c_void_p, C.c_int32, C.c_uint32, C.c_float, C.POINTER(PgcnGatedWalk)
    lib.pgcn_transformer_version.restype = C.c_char_p
    lib.pgcn_transformer_version.argtypes = []
    lib.pgcn_transformer_last_error.restype = C.c_char_p
    lib.pgcn_transformer_last_error.argtypes = []
    # (walk, m, h, heads, Q_own, KV_own, KV_halo, scale, gid, drop, threshold, keep_scale, ...)
    head = [walk, i32, i32, i32, vp, vp, vp, f32, vp, vp, u32, f32]
    lib.pgcn_transformer_forward.restype = C.c_int
    lib.pgcn_transformer_forward.argtypes = head + [vp, vp, vp, i32, vp]
    lib.pgcn_transformer_backward_rows.restype = C.c_int
    lib.pgcn_transformer_backward_rows.argtypes = head + [vp, vp, vp, vp, vp, vp, i32, vp]
    lib.pgcn_transformer_backward_cols.restype = C.c_int
    lib.pgcn_transformer_backward_cols.argtypes = head + [vp, vp, vp, vp, vp, i32, vp]
    _transformer = lib
    return lib


def check_transformer(rc):
    """Raise RuntimeError carrying pgcn_transformer_last_error when a libpgcn_transformer call returned a negative
    status."""
    if rc < 0:
        msg = load_transformer().pgcn_transformer_last_error()
        raise RuntimeError("pgcn_transformer error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_gatedgcn(build_if_missing=True):
    """Load libpgcn_gatedgcn.so (building it first when stale and nvcc is available)."""
    global _gatedgcn
    if _gatedgcn is not None:
        return _gatedgcn
    lib = C.CDLL(_built(_build.GATEDGCN_LIB, _build.gatedgcn_is_stale, _build.build_gatedgcn, build_if_missing))
    vp, i32, f32, walk = C.c_void_p, C.c_int32, C.c_float, C.POINTER(PgcnGatedWalk)
    lib.pgcn_gatedgcn_version.restype = C.c_char_p
    lib.pgcn_gatedgcn_version.argtypes = []
    lib.pgcn_gatedgcn_last_error.restype = C.c_char_p
    lib.pgcn_gatedgcn_last_error.argtypes = []
    lib.pgcn_gatedgcn_load.restype = C.c_int
    lib.pgcn_gatedgcn_load.argtypes = []
    # (walk, m, h, Dx_own, EB_own, EB_halo, Ce, eps, Z, den, Ehat, work, f, stream)
    lib.pgcn_gatedgcn_forward.restype = C.c_int
    lib.pgcn_gatedgcn_forward.argtypes = [walk, i32, i32, vp, vp, vp, vp, f32, vp, vp, vp, vp, i32, vp]
    # (walk, m, h, EB_own, EB_halo, Ehat, gEhat, Z, den, gZ, eps, U, dCe, dDx, work, f, stream)
    lib.pgcn_gatedgcn_backward_rows.restype = C.c_int
    lib.pgcn_gatedgcn_backward_rows.argtypes = [walk, i32, i32, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, i32, vp]
    # (walk, perm, m, h, Ehat, dCe, U, dEB, work, f, stream)
    lib.pgcn_gatedgcn_backward_cols.restype = C.c_int
    lib.pgcn_gatedgcn_backward_cols.argtypes = [walk, vp, i32, i32, vp, vp, vp, vp, vp, i32, vp]
    _gatedgcn = lib
    return lib


def check_gatedgcn(rc):
    """Raise RuntimeError carrying pgcn_gatedgcn_last_error when a libpgcn_gatedgcn call returned a negative status."""
    if rc < 0:
        msg = load_gatedgcn().pgcn_gatedgcn_last_error()
        raise RuntimeError("pgcn_gatedgcn error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_transformer_edge(build_if_missing=True):
    """Load libpgcn_transformer_edge.so (building it first when stale and nvcc is available)."""
    global _transformer_edge
    if _transformer_edge is not None:
        return _transformer_edge
    lib = C.CDLL(_built(_build.TRANSFORMER_EDGE_LIB, _build.transformer_edge_is_stale, _build.build_transformer_edge,
                        build_if_missing))
    vp, i32, u32, f32, walk = C.c_void_p, C.c_int32, C.c_uint32, C.c_float, C.POINTER(PgcnGatedWalk)
    lib.pgcn_transformer_edge_version.restype = C.c_char_p
    lib.pgcn_transformer_edge_version.argtypes = []
    lib.pgcn_transformer_edge_last_error.restype = C.c_char_p
    lib.pgcn_transformer_edge_last_error.argtypes = []
    lib.pgcn_transformer_edge_load.restype = C.c_int
    lib.pgcn_transformer_edge_load.argtypes = []
    # (walk, m, h, heads, Q_own, KV_own, KV_halo, E, scale, gid, drop, threshold, keep_scale, ...)
    head = [walk, i32, i32, i32, vp, vp, vp, vp, f32, vp, vp, u32, f32]
    lib.pgcn_transformer_edge_forward.restype = C.c_int
    lib.pgcn_transformer_edge_forward.argtypes = head + [vp, vp, vp, i32, vp]
    # (..., gZ, Z, L, dQ, D, PS, dE, work, f, stream)
    lib.pgcn_transformer_edge_backward_rows.restype = C.c_int
    lib.pgcn_transformer_edge_backward_rows.argtypes = head + [vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    # (walk, perm, m, h, heads, Q_own, gZ, PS, scale, dKV, work, f, stream)
    lib.pgcn_transformer_edge_backward_cols.restype = C.c_int
    lib.pgcn_transformer_edge_backward_cols.argtypes = [walk, vp, i32, i32, i32, vp, vp, vp, f32, vp, vp, i32, vp]
    _transformer_edge = lib
    return lib


def check_transformer_edge(rc):
    """Raise RuntimeError carrying pgcn_transformer_edge_last_error when a libpgcn_transformer_edge call returned a
    negative status."""
    if rc < 0:
        msg = load_transformer_edge().pgcn_transformer_edge_last_error()
        raise RuntimeError("pgcn_transformer_edge error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_gine(build_if_missing=True):
    """Load libpgcn_gine.so (building it first when stale and nvcc is available)."""
    global _gine
    if _gine is not None:
        return _gine
    lib = C.CDLL(_built(_build.GINE_LIB, _build.gine_is_stale, _build.build_gine, build_if_missing))
    vp, i32, walk = C.c_void_p, C.c_int32, C.POINTER(PgcnGatedWalk)
    lib.pgcn_gine_version.restype = C.c_char_p
    lib.pgcn_gine_version.argtypes = []
    lib.pgcn_gine_last_error.restype = C.c_char_p
    lib.pgcn_gine_last_error.argtypes = []
    lib.pgcn_gine_load.restype = C.c_int
    lib.pgcn_gine_load.argtypes = []
    # (walk, m, h, X_own, X_halo, E, Z, work, f, stream)
    lib.pgcn_gine_forward.restype = C.c_int
    lib.pgcn_gine_forward.argtypes = [walk, i32, i32, vp, vp, vp, vp, vp, i32, vp]
    # (walk, perm, m, h, X_own, X_halo, E, gZ, dE, dX, work, f, stream)
    lib.pgcn_gine_backward.restype = C.c_int
    lib.pgcn_gine_backward.argtypes = [walk, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    _gine = lib
    return lib


def check_gine(rc):
    """Raise RuntimeError carrying pgcn_gine_last_error when a libpgcn_gine call returned a negative status."""
    if rc < 0:
        msg = load_gine().pgcn_gine_last_error()
        raise RuntimeError("pgcn_gine error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_rgcn(build_if_missing=True):
    """Load libpgcn_rgcn.so (building it first when stale and nvcc is available)."""
    global _rgcn
    if _rgcn is not None:
        return _rgcn
    lib = C.CDLL(_built(_build.RGCN_LIB, _build.rgcn_is_stale, _build.build_rgcn, build_if_missing))
    vp, i32, walk = C.c_void_p, C.c_int32, C.POINTER(PgcnGatedWalk)
    lib.pgcn_rgcn_version.restype = C.c_char_p
    lib.pgcn_rgcn_version.argtypes = []
    lib.pgcn_rgcn_last_error.restype = C.c_char_p
    lib.pgcn_rgcn_last_error.argtypes = []
    lib.pgcn_rgcn_load.restype = C.c_int
    lib.pgcn_rgcn_load.argtypes = []
    # (walk, perm, m, h, R, X_own, X_halo, w, Z, work, f, stream)
    lib.pgcn_rgcn_forward.restype = C.c_int
    lib.pgcn_rgcn_forward.argtypes = [walk, vp, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp]
    # (walk, perm, m, h, R, gZ, w, dX, work, f, stream)
    lib.pgcn_rgcn_backward.restype = C.c_int
    lib.pgcn_rgcn_backward.argtypes = [walk, vp, i32, i32, i32, vp, vp, vp, vp, i32, vp]
    _rgcn = lib
    return lib


def check_rgcn(rc):
    """Raise RuntimeError carrying pgcn_rgcn_last_error when a libpgcn_rgcn call returned a negative status."""
    if rc < 0:
        msg = load_rgcn().pgcn_rgcn_last_error()
        raise RuntimeError("pgcn_rgcn error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc


def load_gatv2_edge(build_if_missing=True):
    """Load libpgcn_gatv2_edge.so (building it first when stale and nvcc is available)."""
    global _gatv2_edge
    if _gatv2_edge is not None:
        return _gatv2_edge
    lib = C.CDLL(_built(_build.GATV2_EDGE_LIB, _build.gatv2_edge_is_stale, _build.build_gatv2_edge, build_if_missing))
    vp, i32, u32, f32, walk = C.c_void_p, C.c_int32, C.c_uint32, C.c_float, C.POINTER(PgcnGatedWalk)
    lib.pgcn_gatv2_edge_version.restype = C.c_char_p
    lib.pgcn_gatv2_edge_version.argtypes = []
    lib.pgcn_gatv2_edge_last_error.restype = C.c_char_p
    lib.pgcn_gatv2_edge_last_error.argtypes = []
    lib.pgcn_gatv2_edge_work_rows.restype = C.c_int64
    lib.pgcn_gatv2_edge_work_rows.argtypes = [walk]
    lib.pgcn_gatv2_edge_load.restype = C.c_int
    lib.pgcn_gatv2_edge_load.argtypes = []
    # (walk, m, h, heads, XL_own, XL_halo, XR, att, E, negative_slope, gid, drop, threshold, keep_scale, ...)
    head = [walk, i32, i32, i32, vp, vp, vp, vp, vp, f32, vp, vp, u32, f32]
    # (..., Z, L, work, f, stream)
    lib.pgcn_gatv2_edge_forward.restype = C.c_int
    lib.pgcn_gatv2_edge_forward.argtypes = head + [vp, vp, vp, i32, vp]
    # (..., gZ, Z, L, dXR, D, PS, G, datt, work, f, stream)
    lib.pgcn_gatv2_edge_backward_rows.restype = C.c_int
    lib.pgcn_gatv2_edge_backward_rows.argtypes = head + [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    # (walk, perm, m, h, heads, gZ, PS, G, dXL, work, f, stream)
    lib.pgcn_gatv2_edge_backward_cols.restype = C.c_int
    lib.pgcn_gatv2_edge_backward_cols.argtypes = [walk, vp, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp]
    _gatv2_edge = lib
    return lib


def check_gatv2_edge(rc):
    """Raise RuntimeError carrying pgcn_gatv2_edge_last_error when a libpgcn_gatv2_edge call returned a negative
    status."""
    if rc < 0:
        msg = load_gatv2_edge().pgcn_gatv2_edge_last_error()
        raise RuntimeError("pgcn_gatv2_edge error %d: %s" % (rc, (msg or b"").decode("utf-8", "replace")))
    return rc
