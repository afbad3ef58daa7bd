"""CPU-side check of pgcn_plan_prepare (the set-up call that makes the fused entry points capturable in a CUDA graph):
a null plan is an invalid argument, reported with a message, not a crash."""
from pgcn_b200 import cabi


def test_prepare_rejects_a_null_plan():
    lib = cabi.load()
    assert lib.pgcn_plan_prepare(None, 16) == -1
    assert b"null" in lib.pgcn_last_error(None)
