"""CPU-side checks of the gated aggregation: include/pgcn_gated.h and include/pgcn_b200_halo.h against their bindings,
libpgcn_gated.so's exports, architecture and kernel manifest, libpgcn_b200.so's unchanged manifest, the libraries'
separate dependency lists, the refusals of the C entry points (bad arguments, no GPU), the work table, the oracle's
analytic gradients against torch autograd in fp64, and PGATED.py's usage errors."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import gated_oracle as go
from conftest import ROOT
from pgcn_b200 import build, cabi, plan as planmod

MANIFEST = os.path.join(ROOT, "tests", "gated_kernel_instances.txt")


def header_functions(name):
    txt = open(os.path.join(ROOT, "include", name)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {fn: [a for a in args.split(",") if a.strip() not in ("", "void")]
            for fn, args in re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


@pytest.mark.parametrize("header,symbols,load", [("pgcn_gated.h", "GATED_SYMBOLS", "load_gated"),
                                                 ("pgcn_b200_halo.h", "HALO_SYMBOLS", "load")])
def test_header_and_binding_agree(header, symbols, load):
    fns = header_functions(header)
    assert sorted(fns) == sorted(getattr(cabi, symbols))
    lib = getattr(cabi, load)()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    assert not set(fns) & set(cabi.SYMBOLS)


def test_libraries_export_every_symbol_and_name_sm_90a():
    lib = cabi.load_gated()
    for name in cabi.GATED_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_gated.so does not export " + name
    assert b"sm_90a" in lib.pgcn_gated_version()
    assert os.path.basename(cabi.gated_lib_path()) == "libpgcn_gated.so"
    assert lib.pgcn_gated_chunk() >= 32
    assert hasattr(cabi.load(), "pgcn_halo_rows_add")


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_gated()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.gated_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifests():
    lk = _tools()
    cabi.load_gated()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.gated_lib_path()) == want
    cabi.load()
    with open(os.path.join(ROOT, "tests", "kernel_instances.txt")) as fh:
        assert lk.list_kernels() == [ln.strip() for ln in fh if ln.strip()]


def test_each_library_has_its_own_dependencies():
    here = {os.path.abspath(build.__file__)}
    assert not set(build.GATED_DEPS) & set(build.DEPS) - here
    assert not set(build.GATED_DEPS) & set(build.DROPOUT_DEPS) - here
    assert os.path.join(build.CSRC, "gated.cu") in build.GATED_DEPS
    assert os.path.join(ROOT, "include", "pgcn_b200_halo.h") in build.DEPS


def _walk(rows, nitems=None, items=1, nslots=0):
    return cabi.PgcnGatedWalk(8, items, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_gated()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)
    assert lib.pgcn_gated_forward(None, 4, 0, p, p, None, p, None, 8, None) == -1
    assert b"null walk" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_forward(C.byref(w), 5, 0, p, p, None, p, None, 8, None) == -1
    assert b"rows" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_forward(C.byref(w), 4, 0, p, p, None, p, None, 0, None) == -1
    assert b"f=0" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_forward(C.byref(w), 4, 0, None, p, None, p, None, 8, None) == -1
    assert lib.pgcn_gated_forward(C.byref(w), 4, 2, p, p, None, p, None, 8, None) == -1
    assert b"QV_halo" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_forward(C.byref(_walk(4, nitems=3)), 4, 0, p, p, None, p, None, 8, None) == -1
    assert lib.pgcn_gated_forward(C.byref(_walk(4, nslots=2)), 4, 0, p, p, None, p, None, 8, None) == -1
    assert b"work" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_backward_rows(C.byref(w), 4, 0, p, p, None, None, p, None, 8, None) == -1
    assert b"gZ" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_backward_cols(C.byref(w), 4, 2, p, p, p, p, p, None, 8, None) == -1     # rows != m + h
    assert b"rows" in lib.pgcn_gated_last_error()
    assert lib.pgcn_gated_backward_cols(C.byref(_walk(6)), 4, 2, p, p, p, p, None, None, 8, None) == -1
    assert b"output" in lib.pgcn_gated_last_error()
    assert cabi.load().pgcn_halo_rows_add(None, None, None, 8, None) == -1


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_gated(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_gated_forward(C.byref(w), 2, 0, p, p, None, p, None, 4, None),\n"
            "      lib.pgcn_gated_backward_rows(C.byref(w), 2, 0, p, p, None, p, p, None, 4, None),\n"
            "      lib.pgcn_gated_backward_cols(C.byref(w), 2, 0, p, p, None, p, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_gated_last_error().decode())\n" % ROOT)
    cabi.load_gated()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 3)
    assert [int(x) for x in parts[:3]] == [-4, -4, -4] and "no CUDA device" in parts[3]


@pytest.mark.parametrize("chunk", [1, 3, 512])
def test_work_table_covers_every_entry_once_in_chunk_order(chunk):
    deg = np.array([0, 5, 1, 7, 0, 3, 12, 2])
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    items, splits, nslots = planmod.gated_work_table(rowptr, chunk)
    assert items.dtype == splits.dtype == np.int32 and items.shape[1] == 4 and splits.shape[1] == 3
    assert sorted(items[:, 0][items[:, 3] < 0].tolist() + splits[:, 0].tolist()) == list(range(len(deg)))
    assert (items[:, 2] - items[:, 1] <= np.maximum(chunk, deg[items[:, 0]])).all()
    long_rows = np.flatnonzero(deg > chunk)
    assert splits[:, 0].tolist() == long_rows.tolist() and nslots == int(sum(-(-deg[long_rows] // chunk)))
    assert (items[:nslots, 3] == np.arange(nslots)).all() and (items[nslots:, 3] == -1).all()
    for r, s0, n in splits:
        ch = items[s0:s0 + n]
        assert (ch[:, 0] == r).all() and ch[0, 1] == rowptr[r] and ch[-1, 2] == rowptr[r + 1]
        assert (ch[1:, 1] == ch[:-1, 2]).all() and (ch[:, 2] - ch[:, 1] <= chunk).all()
    for r, e0, e1, _ in items[nslots:]:
        assert e0 == rowptr[r] and e1 == rowptr[r + 1]


def test_oracle_gradients_equal_torch_autograd_in_fp64():
    rs = np.random.RandomState(3)
    A = sp.random(40, 50, density=0.15, random_state=rs, format="csr")
    A.indices[::7] = A.indices[1::7][:len(A.indices[::7])]          # some repeated columns in a row
    rows, cols = (torch.from_numpy(a) for a in go._entries(A.indptr, A.indices))
    f = 6
    K, gZ = rs.standard_normal((40, f)) * 3, rs.standard_normal((40, f))
    Q, V = rs.standard_normal((50, f)) * 3, rs.standard_normal((50, f))
    got = go.terms(A.indptr, A.indices, 50, K, Q, V, gZ, round_x=False)
    Kt, Qt, Vt = (torch.tensor(x, requires_grad=True) for x in (K, Q, V))
    Z = go.torch_gated(rows, cols, Kt, Qt, Vt)
    Z.backward(torch.from_numpy(gZ))
    for name, want in (("Z", Z.detach()), ("dK", Kt.grad), ("dQ", Qt.grad), ("dV", Vt.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)
        assert (got[name][1] >= np.abs(got[name][0]) * (1 - 1e-12)).all(), name


def test_oracle_fp32_reference_propagates_special_values():
    rowptr, colidx = np.array([0, 2, 3]), np.array([0, 1, 1])
    f32 = lambda a: np.array(a, np.float32)
    K = f32([[np.inf], [-np.inf]])
    Q = f32([[-np.inf], [0.0]])
    V = f32([[1.0], [2.0]])
    out = go.fp32_reference(rowptr, colidx, 2, K, Q, V, f32([[1.0], [1.0]]))
    assert np.isnan(out["Z"][0, 0]) and out["Z"][1, 0] == 0.0       # inf - inf; sigmoid(-inf) = 0
    assert np.isnan(out["dV"][0, 0])


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import gated
    with pytest.raises(SystemExit) as e:
        gated.main(argv)
    assert e.value.code == 2
    assert "usage: PGATED.py" in capsys.readouterr().out


def test_cli_run_refuses_gloo():
    from pgcn_b200 import gated
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gated.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")


class _FakePlan:
    m, n, f_max, _bound, layout = 4, 4, 8, True, "local"

    def gated_walks(self):
        return None, None


def test_aggregate_gated_has_no_cpu_fallback_and_needs_f_max_2f():
    from pgcn_b200 import op
    x = torch.zeros((4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_gated(_FakePlan(), x, x, x)
    with pytest.raises(ValueError, match="f_max >= 2f"):
        op.aggregate_gated(_FakePlan(), torch.zeros((4, 5)), x, x)
