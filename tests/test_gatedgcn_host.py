"""CPU-side checks of GatedGCN: include/pgcn_gatedgcn.h against its binding, libpgcn_gatedgcn.so's exports,
architecture and kernel manifest, the other libraries' unchanged manifests, the libraries' separate dependency lists,
the refusals of the C entry points (bad arguments, no GPU), PgcnPlan.transposed_entries' permutation, the oracle's
analytic gradients against torch autograd in fp64 with and without an edge gradient, and PGATEDGCN.py's usage
errors."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import gatedgcn_oracle as gco
from conftest import ROOT
from pgcn_b200 import build, cabi, graphio, plan as planmod

MANIFEST = os.path.join(ROOT, "tests", "gatedgcn_kernel_instances.txt")


def header_functions(name):
    txt = open(os.path.join(ROOT, "include", name)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {fn: [a for a in args.split(",") if a.strip() not in ("", "void")]
            for fn, args in re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_header_and_binding_agree():
    fns = header_functions("pgcn_gatedgcn.h")
    assert sorted(fns) == sorted(cabi.GATEDGCN_SYMBOLS)
    lib = cabi.load_gatedgcn()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS, cabi.TRANSFORMER_SYMBOLS):
        assert not set(fns) & set(other)
    # the walk struct is the gated library's, not a second definition
    txt = open(os.path.join(ROOT, "include", "pgcn_gatedgcn.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_gatedgcn()
    for name in cabi.GATEDGCN_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_gatedgcn.so does not export " + name
    assert b"sm_90a" in lib.pgcn_gatedgcn_version()
    assert os.path.basename(cabi.gatedgcn_lib_path()) == "libpgcn_gatedgcn.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_gatedgcn()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.gatedgcn_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifests():
    lk = _tools()
    cabi.load_gatedgcn()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.gatedgcn_lib_path()) == want
    for load, path, manifest in ((cabi.load_gated, cabi.gated_lib_path, "gated_kernel_instances.txt"),
                                 (cabi.load_transformer, cabi.transformer_lib_path, "transformer_kernel_instances.txt"),
                                 (cabi.load_dropout, cabi.dropout_lib_path, "dropout_kernel_instances.txt"),
                                 (cabi.load, cabi.lib_path, "kernel_instances.txt")):
        load()
        with open(os.path.join(ROOT, "tests", manifest)) as fh:
            assert lk.list_kernels(lib=path()) == [ln.strip() for ln in fh if ln.strip()], manifest


def test_each_library_has_its_own_dependencies():
    shared = {os.path.abspath(build.__file__), os.path.join(ROOT, "include", "pgcn_gated.h"),
              os.path.join(build.CSRC, "gated_math.cuh")}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS, build.TRANSFORMER_DEPS):
        assert not set(build.GATEDGCN_DEPS) & set(other) - shared
    for name in (os.path.join(build.CSRC, "gatedgcn.cu"), os.path.join(build.CSRC, "gated_math.cuh"),
                 os.path.join(ROOT, "include", "pgcn_gatedgcn.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.GATEDGCN_DEPS
    assert build.GATEDGCN_SOURCES == [os.path.join(build.CSRC, "gatedgcn.cu")]
    # the gate has one definition, which the gated library depends on as well
    assert os.path.join(build.CSRC, "gated_math.cuh") in build.GATED_DEPS
    for src in ("gated.cu", "gatedgcn.cu"):
        txt = open(os.path.join(build.CSRC, src)).read()
        assert '#include "gated_math.cuh"' in txt and "float gate(" not in txt, src


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_gatedgcn()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)

    def fwd(walk=C.byref(w), m=4, h=0, Dx=p, EB=p, EBh=None, Ce=p, eps=1e-6, Z=p, den=p, E=p, work=None, f=8):
        return lib.pgcn_gatedgcn_forward(walk, m, h, Dx, EB, EBh, Ce, eps, Z, den, E, work, f, None)

    def rows(walk=C.byref(w), m=4, h=0, EB=p, EBh=None, E=p, gE=None, Z=p, den=p, gZ=p, eps=1e-6, U=p, dCe=p, dDx=p,
             work=None, f=8):
        return lib.pgcn_gatedgcn_backward_rows(walk, m, h, EB, EBh, E, gE, Z, den, gZ, eps, U, dCe, dDx, work, f, None)

    def cols(walk=C.byref(_walk(6)), perm=p, m=4, h=2, E=p, dCe=p, U=p, dEB=p, work=None, f=8):
        return lib.pgcn_gatedgcn_backward_cols(walk, perm, m, h, E, dCe, U, dEB, work, f, None)

    def err():
        return lib.pgcn_gatedgcn_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=(1 << 24) + 1) == -1 and b"f=" in err()
    for eps in (-1e-6, float("inf"), float("nan")):
        assert fwd(eps=eps) == -1 and b"eps" in err(), eps
        assert rows(eps=eps) == -1 and b"eps" in err(), eps
    assert fwd(Dx=None) == -1 and b"Dx_own" in err()
    assert fwd(Ce=None) == -1 and b"Ce" in err()
    assert fwd(h=2) == -1 and b"EB_halo" in err()
    assert fwd(E=None) == -1 and b"output" in err()
    assert fwd(walk=C.byref(_walk(4, nitems=3))) == -1 and b"work table" in err()
    assert fwd(walk=C.byref(_walk(4, nslots=2))) == -1 and b"work" in err()
    assert rows(gZ=None) == -1 and b"gZ" in err()
    assert rows(den=None) == -1 and b"den" in err()
    assert rows(U=None) == -1 and b"output" in err()
    assert rows(h=2) == -1 and b"EB_halo" in err()
    assert cols(walk=C.byref(w)) == -1 and b"rows" in err()                 # rows != m + h
    assert cols(perm=None) == -1 and b"perm" in err()
    assert cols(U=None) == -1 and b"U" in err()
    assert cols(dEB=None) == -1 and b"dEB" in err()
    assert cols(walk=C.byref(_walk(6, nslots=1))) == -1 and b"work" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_gatedgcn(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_gatedgcn_load(),\n"
            "      lib.pgcn_gatedgcn_forward(C.byref(w), 2, 0, p, p, None, p, 1e-6, p, p, p, None, 4, None),\n"
            "      lib.pgcn_gatedgcn_backward_rows(C.byref(w), 2, 0, p, None, p, None, p, p, p, 1e-6, p, p, p, None, 4,"
            " None),\n"
            "      lib.pgcn_gatedgcn_backward_cols(C.byref(w), p, 2, 0, p, p, p, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_gatedgcn_last_error().decode())\n" % ROOT)
    cabi.load_gatedgcn()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 4)
    assert [int(x) for x in parts[:4]] == [-4, -4, -4, -4] and "no CUDA device" in parts[4]


class _HostPlan(planmod.PgcnPlan):
    """A PgcnPlan's host side only (no device handle): transposed_entries on the CPU."""

    def __init__(self, lp):
        self.lp = lp
        self.device = torch.device("cpu")
        self._transposed_entries = None

    def close(self):
        pass


def _hub_lp():
    A = sp.coo_matrix(graphio.synthetic_graph(2000, 30000, seed=31))
    row = np.concatenate([A.row, np.zeros(1500, np.int64)])
    col = np.concatenate([A.col, np.arange(1500)])
    B = sp.csr_matrix((np.ones(len(row), np.float32), (row, col)), shape=A.shape)
    B.sum_duplicates()
    return planmod.build_local_plan(B, graphio.random_partvec(2000, 2, seed=3), 1, 2)


def _dup_lp():
    from test_max_aggregation import with_duplicates
    from harness import karate
    A = karate()
    return with_duplicates(planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1))


@pytest.mark.parametrize("case", ["karate", "hub", "dup"])
def test_transposed_entries_is_the_stable_column_sort(case, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    if case == "karate":
        from harness import karate
        A = karate()
        lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    else:
        lp = _hub_lp() if case == "hub" else _dup_lp()
    perm = _HostPlan(lp).transposed_entries().numpy()
    nnz = lp.nnz()
    assert perm.dtype == np.int32 and perm.shape == (nnz,)
    assert np.array_equal(np.sort(perm), np.arange(nnz))                 # a bijection of the entries
    rows = np.repeat(np.arange(lp.m), np.diff(lp.rowptr.astype(np.int64)))
    assert np.array_equal(rows[perm], lp.t_colidx)
    tcols = np.repeat(np.arange(lp.m + lp.h), np.diff(lp.t_rowptr.astype(np.int64)))
    assert np.array_equal(lp.colidx[perm], tcols)                         # each transposed row's column id
    if case == "dup":
        # duplicated (row, column) entries keep their forward order in the transpose
        key = rows.astype(np.int64) * (lp.m + lp.h) + lp.colidx
        assert len(np.unique(key)) < nnz
        for t in range(1, nnz):
            if key[perm[t]] == key[perm[t - 1]]:
                assert perm[t] > perm[t - 1]


def test_transposed_entries_refuses_a_capture(monkeypatch):
    from harness import karate
    A = karate()
    plan = _HostPlan(planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="transposed_entries"):
        plan.transposed_entries()
    assert plan._transposed_entries is None


@pytest.mark.parametrize("with_ge", [True, False])
def test_oracle_gradients_equal_torch_autograd_in_fp64(with_ge):
    rs = np.random.RandomState(5)
    A = sp.random(40, 50, density=0.15, random_state=rs, format="csr")
    A.indices[::7] = A.indices[1::7][:len(A.indices[::7])]          # some repeated columns in a row
    A.indptr[5:8] = A.indptr[5]                                      # empty rows
    A.indptr[8:] = np.maximum(A.indptr[8:], A.indptr[5])
    nnz = int(A.indptr[-1])
    idx = A.indices[:nnz]
    r, c = gco.entries(A.indptr, idx)
    rows, cols = torch.from_numpy(r), torch.from_numpy(c)
    f = 6
    Dx, gZ = rs.standard_normal((40, f)) * 2, rs.standard_normal((40, f))
    Ex, Bx = rs.standard_normal((50, f)) * 2, rs.standard_normal((50, f))
    Ce = rs.standard_normal((nnz, f))
    gE = rs.standard_normal((nnz, f)) if with_ge else None
    eps = 1e-3
    got = gco.terms(A.indptr, idx, 50, Dx, Ex, Bx, Ce, gZ, gE, eps=eps, round_e=False)
    Dt, Et, Bt, Ct = (torch.tensor(x, requires_grad=True) for x in (Dx, Ex, Bx, Ce))
    Z, Eh = gco.torch_gatedgcn(rows, cols, 40, Dt, Et, Bt, Ct, eps)
    loss = (Z * torch.from_numpy(gZ)).sum() + ((Eh * torch.from_numpy(gE)).sum() if with_ge else 0)
    loss.backward()
    for name, want in (("Z", Z.detach()), ("Ehat", Eh.detach()), ("dDx", Dt.grad), ("dEx", Et.grad),
                       ("dBx", Bt.grad), ("dCe", Ct.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-11, atol=1e-11, err_msg=name)
        if name != "Ehat":
            assert (got[name][1] >= 0).all(), name
    assert np.all(got["Z"][0][5:7] == 0.0) and np.all(got["den"][0][5:7] == 0.0)     # empty rows


def test_oracle_fp32_reference_propagates_special_values():
    rowptr, colidx = np.array([0, 2, 3, 3]), np.array([0, 1, 1])
    f32 = lambda a: np.array(a, np.float32)
    Dx = f32([[np.inf], [0.0], [0.0]])
    Ex = f32([[-np.inf], [0.0]])
    Bx = f32([[1.0], [2.0]])
    Ce = f32([[0.0], [0.0], [0.0]])
    out = gco.fp32_reference(rowptr, colidx, 2, Dx, Ex, Bx, Ce, f32([[1.0], [1.0], [1.0]]))
    assert np.isnan(out["Ehat"][0, 0]) and np.isnan(out["Z"][0, 0])   # inf - inf
    assert out["Z"][1, 0] == np.float32(np.float32(0.5) * 2) / np.float32(np.float32(0.5) + np.float32(1e-6))
    assert out["Z"][2, 0] == 0.0 and out["den"][2, 0] == 0.0          # an empty row
    assert np.isnan(out["dEx"][0, 0]) and np.isnan(out["dDx"][0, 0])


def test_oracle_bound_covers_an_fp32_evaluation():
    """The fp32 restatement (another summation and rounding order than the kernels') lies within the bound."""
    rs = np.random.RandomState(9)
    A = sp.random(60, 60, density=0.2, random_state=rs, format="csr")
    nnz = int(A.indptr[-1])
    f = 5
    Dx, Ex, Bx, gZ = ((rs.standard_normal((60, f)) * 2).astype(np.float32) for _ in range(4))
    Ce, gE = ((rs.standard_normal((nnz, f))).astype(np.float32) for _ in range(2))
    ref = gco.terms(A.indptr, A.indices, 60, Dx, Ex, Bx, Ce, gZ, gE)
    got = gco.fp32_reference(A.indptr, A.indices, 60, Dx, Ex, Bx, Ce, gZ, gE)
    assert np.array_equal(got["Ehat"].astype(np.float64), ref["Ehat"][0])
    for name in ("Z", "den", "dCe", "dDx", "dEx", "dBx"):
        val, tol = ref[name]
        assert (np.abs(got[name].astype(np.float64) - val) <= tol + 1e-30).all(), name


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "0", "-l", "2", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import gatedgcn
    with pytest.raises(SystemExit) as e:
        gatedgcn.main(argv)
    assert e.value.code == 2
    assert "usage: PGATEDGCN.py" in capsys.readouterr().out


def test_cli_run_refuses_gloo():
    from pgcn_b200 import gatedgcn
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gatedgcn.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")


class _FakePlan:
    m, n, f_max, _bound, layout, device = 4, 4, 8, True, "local", torch.device("cpu")

    def gated_walks(self):
        return None, None

    def transposed_entries(self):
        return None


def test_aggregate_gatedgcn_refusals():
    from pgcn_b200 import op
    x = torch.zeros((4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_gatedgcn(_FakePlan(), x, x, x, None)
    with pytest.raises(ValueError, match="f_max >= 2f"):
        op.aggregate_gatedgcn(_FakePlan(), torch.zeros((4, 5)), x, x, None)
    for eps in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="eps"):
            op.aggregate_gatedgcn(_FakePlan(), x, x, x, None, eps)
