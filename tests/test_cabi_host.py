"""CPU-side checks of the drop-in boundary: the library loads, exports every symbol that
include/pgcn_b200.h declares, and FAILS LOUDLY without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
import pgcn_b200
from pgcn_b200 import cabi


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "pgcn_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(", txt)))


def test_header_and_binding_agree():
    assert header_symbols() == sorted(cabi.SYMBOLS)


def test_library_exports_every_declared_symbol():
    lib = cabi.load()
    for name in header_symbols():
        assert hasattr(lib, name), "libpgcn_b200.so does not export " + name
    assert b"sm_90a" in lib.pgcn_version()


def test_built_for_sm_90a():
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-lelf", cabi.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_invalid_arguments_are_reported_not_crashing():
    lib = cabi.load()
    out = C.c_void_p()
    rc = lib.pgcn_plan_create(None, None, None, 0, 0, None, None, None, None, None, None, 1, 0, 16, C.byref(out))
    assert rc == -1 and b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_plan_destroy(None) == 0
    assert lib.pgcn_forward(None, None, None, 16, None) == -1


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = cabi.load()
    rp = np.zeros(2, dtype=np.int32)
    off = np.zeros(2, dtype=np.int64)
    out = C.c_void_p()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.pgcn_plan_create(p(rp), None, None, 1, 0, p(rp), None, None, None, p(off), p(off), 1, 0, 16, C.byref(out))
    assert rc == -4 and not out.value                      # PGCN_ERR_NOGPU
    assert b"no CPU fallback" in lib.pgcn_last_error(None)
    with pytest.raises(RuntimeError):
        cabi.check(rc)


def test_op_rejects_cpu_tensors():
    import torch
    from pgcn_b200 import op

    class FakePlan:
        m = 4; f_max = 8
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_forward(FakePlan(), torch.zeros(4, 8))


def test_product_never_imports_oracle():
    pkg = os.path.dirname(pgcn_b200.__file__)
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), fn
                assert "liboracle" not in src, fn


@pytest.mark.parametrize("epb,long_row", [(8, 0), (64, 0), (128, 300), (144, 0), (256, 100000)])
def test_row_block_schedule_invariants(epb, long_row):
    """The native scheduler (host code of libpgcn_b200.so) on a skewed degree sequence: every edge is covered
    exactly once and in order, ordinary blocks hold whole rows (<= 128 of them, <= epb edges unless a single row
    is larger), rows longer than long_row become ceil(d/epb) single-row segments with consecutive slots."""
    rng = np.random.RandomState(epb)
    deg = np.concatenate([rng.zipf(1.6, 5000).clip(1, 40000), [1] * 300, [70000, 513, 4 * epb, 4 * epb + 1]])
    rng.shuffle(deg)
    rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    nrows = len(deg)
    cap = int(rowptr[-1] // 8 + nrows + 16)
    blocks = np.zeros((cap, 4), dtype=np.int32)
    nlong, nslots = C.c_int32(), C.c_int32()
    lib = cabi.load()
    nb = lib.pgcn_debug_schedule(rowptr.ctypes.data_as(C.c_void_p), nrows, epb, long_row,
                                 blocks.ctypes.data_as(C.c_void_p), cap, C.byref(nlong), C.byref(nslots))
    assert 0 < nb <= cap
    b = blocks[:nb]
    lr = long_row if long_row > 0 else 4 * epb
    # edges: contiguous cover of [0, nnz)
    assert b[0, 2] == 0 and b[-1, 3] == rowptr[-1]
    assert np.array_equal(b[1:, 2], b[:-1, 3]) and (b[:, 3] > b[:, 2]).all()
    seg = b[:, 1] < 0
    # ordinary blocks: whole rows, bounded size
    o = b[~seg]
    assert np.array_equal(rowptr[o[:, 0]], o[:, 2]) and np.array_equal(rowptr[o[:, 0] + o[:, 1]], o[:, 3])
    assert (o[:, 1] >= 1).all() and (o[:, 1] <= 128).all()
    multi = o[:, 1] > 1
    assert ((o[multi, 3] - o[multi, 2]) <= epb).all()
    assert (deg[o[:, 0]] <= lr).all()
    # split rows
    long_rows = np.flatnonzero(deg > lr)
    assert nlong.value == len(long_rows)
    s_ = b[seg]
    assert np.array_equal(np.unique(s_[:, 0]), long_rows)
    assert np.array_equal(-s_[:, 1] - 1, np.arange(len(s_)))               # slots are consecutive in block order
    assert nslots.value == len(s_) == int(sum(-(-deg[r] // epb) for r in long_rows))
    assert ((s_[:, 3] - s_[:, 2]) <= epb).all()
    for r in long_rows[:5]:
        mine = s_[s_[:, 0] == r]
        assert mine[0, 2] == rowptr[r] and mine[-1, 3] == rowptr[r + 1]


def test_debug_schedule_rejects_bad_arguments():
    lib = cabi.load()
    assert lib.pgcn_debug_schedule(None, 1, 128, 0, None, 0, None, None) == -1
