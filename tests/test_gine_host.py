"""CPU-side checks of GINE: include/pgcn_gine.h against its binding, libpgcn_gine.so's exports, architecture and kernel
manifest, the libraries' separate dependency lists, the refusals of the C entry points (bad arguments, no GPU) and of
op.aggregate_gine, the oracle's analytic gradients against torch autograd in fp64, its fp32 evaluation against torch's
special values, and PGINE.py's usage errors."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import gine_oracle as gio
from conftest import ROOT
from pgcn_b200 import build, cabi

MANIFEST = os.path.join(ROOT, "tests", "gine_kernel_instances.txt")


def header_functions(name):
    txt = open(os.path.join(ROOT, "include", name)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {fn: [a for a in args.split(",") if a.strip() not in ("", "void")]
            for fn, args in re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_header_and_binding_agree():
    fns = header_functions("pgcn_gine.h")
    assert sorted(fns) == sorted(cabi.GINE_SYMBOLS)
    lib = cabi.load_gine()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS, cabi.TRANSFORMER_SYMBOLS,
                  cabi.GATEDGCN_SYMBOLS, cabi.TRANSFORMER_EDGE_SYMBOLS):
        assert not set(fns) & set(other)
    # the walk struct is the gated library's, not a second definition
    txt = open(os.path.join(ROOT, "include", "pgcn_gine.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_gine()
    for name in cabi.GINE_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_gine.so does not export " + name
    assert b"sm_90a" in lib.pgcn_gine_version()
    assert os.path.basename(cabi.gine_lib_path()) == "libpgcn_gine.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_gine()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.gine_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifest():
    lk = _tools()
    cabi.load_gine()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.gine_lib_path()) == want


def test_each_library_has_its_own_dependencies(tmp_path):
    shared = {os.path.abspath(build.__file__), os.path.join(ROOT, "include", "pgcn_gated.h"),
              os.path.join(build.CSRC, "gated_math.cuh")}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS, build.TRANSFORMER_DEPS, build.GATEDGCN_DEPS,
                  build.TRANSFORMER_EDGE_DEPS):
        assert not set(build.GINE_DEPS) & set(other) - shared
    for name in (os.path.join(build.CSRC, "gine.cu"), os.path.join(build.CSRC, "gated_math.cuh"),
                 os.path.join(ROOT, "include", "pgcn_gine.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.GINE_DEPS
    assert build.GINE_SOURCES == [os.path.join(build.CSRC, "gine.cu")]
    # touching gine.cu makes only libpgcn_gine.so stale, and touching another library's source leaves it fresh: a
    # library is stale when one of its dependencies is newer (build._stale), checked here on a library made in tmp_path
    deps = {"b200": build.DEPS, "dropout": build.DROPOUT_DEPS, "gated": build.GATED_DEPS,
            "transformer": build.TRANSFORMER_DEPS, "gatedgcn": build.GATEDGCN_DEPS,
            "transformer_edge": build.TRANSFORMER_EDGE_DEPS, "gine": build.GINE_DEPS}
    lib, newer = str(tmp_path / "lib.so"), str(tmp_path / "touched")
    for f in (lib, newer):
        open(f, "w").close()
    os.utime(lib, (1e9, 1e9))
    os.utime(newer, (2e9, 2e9))

    def stale_after_touching(src):
        return {name: build._stale(lib, [newer if d == src else lib for d in ds]) for name, ds in deps.items()}

    assert stale_after_touching(os.path.join(build.CSRC, "gine.cu")) == {n: n == "gine" for n in deps}
    for src in (os.path.join(build.CSRC, "gatedgcn.cu"), os.path.join(build.CSRC, "gated.cu"),
                os.path.join(build.CSRC, "transformer_edge.cu"), os.path.join(build.CSRC, "pgcn_b200.cu"),
                os.path.join(build.CSRC, "edge_dropout.cu"), os.path.join(build.CSRC, "transformer.cu")):
        assert not stale_after_touching(src)["gine"], src


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_gine()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)

    def fwd(walk=C.byref(w), m=4, h=0, X=p, Xh=None, E=p, Z=p, work=None, f=8):
        return lib.pgcn_gine_forward(walk, m, h, X, Xh, E, Z, work, f, None)

    def bwd(walk=C.byref(_walk(6)), perm=p, m=4, h=2, X=p, Xh=p, E=p, gZ=p, dE=None, dX=p, work=None, f=8):
        return lib.pgcn_gine_backward(walk, perm, m, h, X, Xh, E, gZ, dE, dX, work, f, None)

    def err():
        return lib.pgcn_gine_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(m=-1) == -1 and b"rows" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=(1 << 24) + 1) == -1 and b"f=" in err()
    assert fwd(X=None) == -1 and b"X_own" in err()
    assert fwd(h=2) == -1 and b"X_halo" in err()
    assert fwd(E=None) == -1 and b"null E" in err()
    assert fwd(Z=None) == -1 and b"output" in err()
    assert fwd(walk=C.byref(_walk(4, nitems=3))) == -1 and b"work table" in err()
    assert fwd(walk=C.byref(_walk(4, nslots=2))) == -1 and b"work" in err()
    assert fwd(walk=C.byref(cabi.PgcnGatedWalk(None, None, None, 4, 4, 0, 0))) == -1 and b"null idx" in err()
    assert bwd(walk=C.byref(w)) == -1 and b"rows" in err()                 # rows != m + h
    assert bwd(f=-3) == -1 and b"f=-3" in err()
    assert bwd(perm=None) == -1 and b"perm" in err()
    assert bwd(Xh=None) == -1 and b"X_halo" in err()
    assert bwd(E=None) == -1 and b"E/gZ" in err()
    assert bwd(gZ=None) == -1 and b"E/gZ" in err()
    assert bwd(dX=None) == -1 and b"dX" in err()
    assert bwd(walk=C.byref(_walk(6, nslots=1))) == -1 and b"work" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_gine(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_gine_load(),\n"
            "      lib.pgcn_gine_forward(C.byref(w), 2, 0, p, None, p, p, None, 4, None),\n"
            "      lib.pgcn_gine_backward(C.byref(w), p, 2, 0, p, None, p, p, None, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_gine_last_error().decode())\n" % ROOT)
    cabi.load_gine()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 3)
    assert [int(x) for x in parts[:3]] == [-4, -4, -4] and "no CUDA device" in parts[3]


class _Cuda(torch.Tensor):
    """A CPU tensor that passes op's is_cuda check, so that the checks after it can be reached without a GPU."""

    @property
    def is_cuda(self):
        return True


def _cuda(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype).as_subclass(_Cuda)


class _FakeLocal:
    def nnz(self):
        return 6


class _FakePlan:
    m, n, f_max, layout, device, lp = 4, 4, 8, "local", torch.device("cpu"), _FakeLocal()

    def __init__(self, bound=True):
        self._bound = bound

    def gated_walks(self):
        return None, None

    def transposed_entries(self):
        return None


def test_aggregate_gine_refusals():
    from pgcn_b200 import op
    x, e = _cuda(4, 8), _cuda(6, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_gine(_FakePlan(), torch.zeros((4, 8)), e)
    with pytest.raises(TypeError, match="float32"):
        op.aggregate_gine(_FakePlan(), _cuda(4, 8, dtype=torch.float64), e)
    with pytest.raises(TypeError, match="float32"):
        op.aggregate_gine(_FakePlan(), x, _cuda(6, 8, dtype=torch.float16))
    with pytest.raises(ValueError, match=r"X must be \[4, f\]"):
        op.aggregate_gine(_FakePlan(), _cuda(5, 8), e)
    with pytest.raises(ValueError, match="f_max"):
        op.aggregate_gine(_FakePlan(), _cuda(4, 12), _cuda(6, 12))
    for bad in ((6, 4), (5, 8), (6,)):
        with pytest.raises(ValueError, match=r"E must be \[6, 8\]"):
            op.aggregate_gine(_FakePlan(), x, _cuda(*bad))
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_gine(_FakePlan(bound=False), x, e)
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_gine_backward(_FakePlan(bound=False), x, _cuda(0, 8), e, x)


@pytest.mark.parametrize("kinks", [False, True])
def test_oracle_gradients_equal_torch_autograd_in_fp64(kinks):
    rs = np.random.RandomState(5)
    A = sp.random(40, 50, density=0.15, random_state=rs, format="csr")
    A.indices[::7] = A.indices[1::7][:len(A.indices[::7])]          # some repeated columns in a row
    A.indptr[5:8] = A.indptr[5]                                      # empty rows
    A.indptr[8:] = np.maximum(A.indptr[8:], A.indptr[5])
    nnz = int(A.indptr[-1])
    idx = A.indices[:nnz]
    r, c = gio.entries(A.indptr, idx)
    f = 6
    X, E = rs.standard_normal((50, f)), rs.standard_normal((nnz, f))
    gZ = rs.standard_normal((40, f))
    if kinks:
        X, E = np.round(X * 4) / 4, np.round(E * 4) / 4
        sel = rs.uniform(size=(nnz, f)) < 0.33
        E[sel] = -X[c][sel]                                          # pre-activations exactly 0
        X[rs.uniform(size=X.shape) < 0.1] = -0.0
        assert ((X[c] + E) == 0).mean() > 0.25
    got = gio.terms(A.indptr, idx, 50, X, E, gZ)
    Xt, Et = torch.tensor(X, requires_grad=True), torch.tensor(E, requires_grad=True)
    Z = gio.torch_gine(torch.from_numpy(r), torch.from_numpy(c), 40, Xt, Et)
    (Z * torch.from_numpy(gZ)).sum().backward()
    for name, want in (("Z", Z.detach()), ("dE", Et.grad), ("dX", Xt.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)
        assert (got[name][1] >= 0).all(), name
    assert np.array_equal(got["dE"][0], Et.grad.numpy())                 # the mask is exact
    assert np.all(got["Z"][0][5:7] == 0.0)                               # empty rows


def test_oracle_fp32_reference_propagates_special_values_as_torch():
    vals = np.array([np.nan, 0.0, -0.0, 1.0, -1.0, np.inf, -np.inf], np.float32)
    X = np.array(np.meshgrid(vals, vals)[0].reshape(-1), np.float32)     # every pair of specials
    E = np.array(np.meshgrid(vals, vals)[1].reshape(-1), np.float32)
    nnz = len(X)
    rowptr = np.arange(nnz + 1)                                         # row e holds entry e = (e, e)
    colidx = np.arange(nnz)
    gZ = np.random.RandomState(1).standard_normal((nnz, 1)).astype(np.float32)
    gZ[:7, 0] = vals                                                    # specials in the gradient too
    ref = gio.fp32_reference(rowptr, colidx, nnz, X[:, None], E[:, None], gZ)
    Xt, Et = torch.tensor(X[:, None], requires_grad=True), torch.tensor(E[:, None], requires_grad=True)
    idx = torch.from_numpy(colidx.astype(np.int64))
    Z = gio.torch_gine(idx, idx, nnz, Xt, Et)
    Z.backward(torch.from_numpy(gZ))
    b = lambda a: np.asarray(a, np.float32).view(np.uint32)
    assert np.array_equal(b(ref["Z"]), b(Z.detach().numpy()))
    assert np.array_equal(b(ref["dE"]), b(Et.grad.numpy()))
    assert np.array_equal(b(ref["dX"]), b(Xt.grad.numpy()))
    # torch.relu's rule: relu(nan) = nan, relu(-0) = -0, relu(-1) = 0; the gradient passes at nan, 1 and inf only
    with np.errstate(invalid="ignore"):
        pre = X + E
    one = np.ones((nnz, 1), np.float32)
    r = gio.fp32_reference(rowptr, colidx, nnz, X[:, None], E[:, None], one)
    assert np.array_equal(np.isnan(r["Z"][:, 0]), np.isnan(pre))
    assert np.array_equal(r["dE"][:, 0] == 1, (pre > 0) | np.isnan(pre))
    assert not np.signbit(r["Z"][pre == 0, 0]).any()                     # sums start at +0: +0 + -0 = +0


def test_oracle_bound_covers_an_fp32_evaluation():
    """The fp32 restatement (another summation order than the kernels' for dX) lies within the bound; dE is exact."""
    rs = np.random.RandomState(9)
    A = sp.random(60, 60, density=0.2, random_state=rs, format="csr")
    nnz = int(A.indptr[-1])
    f = 5
    X, gZ = ((rs.standard_normal((60, f)) * 2).astype(np.float32) for _ in range(2))
    E = rs.standard_normal((nnz, f)).astype(np.float32)
    ref = gio.terms(A.indptr, A.indices, 60, X, E, gZ)
    got = gio.fp32_reference(A.indptr, A.indices, 60, X, E, gZ)
    assert np.array_equal(got["dE"].astype(np.float64), ref["dE"][0])
    for name in ("Z", "dX"):
        val, tol = ref[name]
        assert (np.abs(got[name].astype(np.float64) - val) <= tol + 1e-30).all(), name


def test_layer_draws_its_parameters_in_the_documented_order():
    from pgcn_b200 import gine

    class _Plan:
        class lp:
            vals = np.ones(3, np.float32)
    torch.manual_seed(3)
    model = gine.PGINE(_Plan(), 4, 2)
    want = gio.init_params(2, 4, 3)
    names = [n for n, _ in model.named_parameters()]
    assert names == ["layers.%d.%s" % (l, p) for l in range(2) for p in (
        "lin_edge.weight", "lin_edge.bias", "mlp.0.weight", "mlp.0.bias", "mlp.2.weight", "mlp.2.bias")]
    got = [p.detach().numpy().astype(np.float64) for p in model.parameters()]
    for g, w in zip(got, [x for layer in want for x in layer]):
        assert np.array_equal(g, w)
    assert tuple(model.edge_input.shape) == (3, 1)
    # eps: a fixed buffer by default, a parameter (not drawn: it starts at the given eps) with train_eps
    assert not any("eps" in n for n in names)
    trained = gine.GINELayer(_Plan(), 4, eps=0.25, train_eps=True)
    assert "eps" in dict(trained.named_parameters()) and float(trained.eps) == 0.25


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "0", "-l", "2", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import gine
    with pytest.raises(SystemExit) as e:
        gine.main(argv)
    assert e.value.code == 2
    assert "usage: PGINE.py" in capsys.readouterr().out


def test_cli_run_refuses_gloo():
    from pgcn_b200 import gine
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gine.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")
