"""CPU-side checks of the edge-value entry points (pgcn_plan_bind_values, pgcn_plan_set_values, pgcn_sddmm,
pgcn_forward_keep_halo): the binding declares them, and null plans or arguments are reported, not crashed on."""
import ctypes as C

from pgcn_b200 import cabi

NEW = ["pgcn_plan_bind_values", "pgcn_plan_set_values", "pgcn_sddmm", "pgcn_forward_keep_halo"]


def test_binding_declares_the_new_symbols():
    lib = cabi.load()
    for name in NEW:
        assert name in cabi.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None, name


def test_null_plan_is_invalid_not_a_crash():
    lib = cabi.load()
    assert lib.pgcn_plan_bind_values(None) == -1
    assert b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_plan_set_values(None, None, None) == -1
    assert lib.pgcn_sddmm(None, None, None, None, None, 16, None) == -1
    assert lib.pgcn_forward_keep_halo(None, None, None, None, 16, None) == -1
