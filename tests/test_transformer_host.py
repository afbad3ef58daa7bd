"""CPU-side checks of the graph transformer attention: include/pgcn_transformer.h against its binding,
libpgcn_transformer.so's exports, architecture and kernel manifest, the other libraries' unchanged manifests, the
libraries' separate dependency lists, the refusals of the C entry points (bad arguments, no GPU), the oracle's analytic
gradients against torch autograd in fp64 with and without a mask, and PTRANSFORMER.py's usage errors."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import dropout_oracle as do
import transformer_oracle as tro
from conftest import ROOT
from pgcn_b200 import build, cabi

MANIFEST = os.path.join(ROOT, "tests", "transformer_kernel_instances.txt")


def header_functions(name):
    txt = open(os.path.join(ROOT, "include", name)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {fn: [a for a in args.split(",") if a.strip() not in ("", "void")]
            for fn, args in re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_header_and_binding_agree():
    fns = header_functions("pgcn_transformer.h")
    assert sorted(fns) == sorted(cabi.TRANSFORMER_SYMBOLS)
    lib = cabi.load_transformer()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS):
        assert not set(fns) & set(other)
    # the walk struct is the gated library's, not a second definition
    txt = open(os.path.join(ROOT, "include", "pgcn_transformer.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_transformer()
    for name in cabi.TRANSFORMER_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_transformer.so does not export " + name
    assert b"sm_90a" in lib.pgcn_transformer_version()
    assert os.path.basename(cabi.transformer_lib_path()) == "libpgcn_transformer.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_transformer()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.transformer_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifests():
    lk = _tools()
    cabi.load_transformer()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.transformer_lib_path()) == want
    cabi.load_gated()
    with open(os.path.join(ROOT, "tests", "gated_kernel_instances.txt")) as fh:
        assert lk.list_kernels(lib=cabi.gated_lib_path()) == [ln.strip() for ln in fh if ln.strip()]
    cabi.load()
    with open(os.path.join(ROOT, "tests", "kernel_instances.txt")) as fh:
        assert lk.list_kernels() == [ln.strip() for ln in fh if ln.strip()]


def test_each_library_has_its_own_dependencies():
    here = {os.path.abspath(build.__file__)}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS):
        assert not set(build.TRANSFORMER_DEPS) & set(other) - here - {os.path.join(build.CSRC, "philox.cuh"),
                                                                      os.path.join(ROOT, "include", "pgcn_gated.h")}
    assert not set(build.TRANSFORMER_DEPS) & set(build.DEPS) - here
    for name in (os.path.join(build.CSRC, "transformer.cu"), os.path.join(build.CSRC, "philox.cuh"),
                 os.path.join(ROOT, "include", "pgcn_transformer.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.TRANSFORMER_DEPS
    assert build.TRANSFORMER_SOURCES == [os.path.join(build.CSRC, "transformer.cu")]


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_transformer()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)

    def fwd(walk=w, m=4, h=0, heads=1, Q=p, KV=p, KVh=None, scale=0.5, gid=None, drop=None, ks=1.0, Z=p, L=p,
            work=None, f=8):
        return lib.pgcn_transformer_forward(walk, m, h, heads, Q, KV, KVh, scale, gid, drop, 0, ks, Z, L, work, f, None)

    def err():
        return lib.pgcn_transformer_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(heads=3) == -1 and b"heads=3" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=260, heads=4) == -1 and b"f=260" in err()
    assert fwd(f=6, heads=4) == -1 and b"multiple" in err()
    assert fwd(scale=float("inf")) == -1 and b"scale" in err()
    assert fwd(Q=None) == -1 and b"Q_own" in err()
    assert fwd(h=2) == -1 and b"KV_halo" in err()
    assert fwd(drop=p) == -1 and b"gid" in err()
    assert fwd(drop=p, gid=p, ks=float("nan")) == -1 and b"keep_scale" in err()
    assert fwd(walk=C.byref(_walk(4, nitems=3))) == -1
    assert fwd(walk=C.byref(_walk(4, nslots=2))) == -1 and b"work" in err()
    assert fwd(L=None) == -1 and b"output" in err()
    rows = lib.pgcn_transformer_backward_rows
    assert rows(C.byref(w), 4, 0, 1, p, p, None, 0.5, None, None, 0, 1.0, None, p, p, p, p, None, 8, None) == -1
    assert b"gZ" in err()
    assert rows(C.byref(w), 4, 0, 1, p, p, None, 0.5, None, None, 0, 1.0, p, p, p, p, None, None, 8, None) == -1
    assert b"dQ/D" in err()
    cols = lib.pgcn_transformer_backward_cols
    assert cols(C.byref(w), 4, 2, 1, p, p, p, 0.5, None, None, 0, 1.0, p, p, p, p, None, 8, None) == -1
    assert b"rows" in err()                                                          # rows != m + h
    assert cols(C.byref(_walk(6)), 4, 2, 1, p, p, p, 0.5, None, None, 0, 1.0, p, p, None, p, None, 8, None) == -1
    assert b"gZ/L/D" in err()
    assert cols(C.byref(_walk(6)), 4, 2, 1, p, p, p, 0.5, None, None, 0, 1.0, p, p, p, None, None, 8, None) == -1
    assert b"dKV" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_transformer(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_transformer_forward(C.byref(w), 2, 0, 2, p, p, None, 0.5, p, p, 7, 2.0, p, p, None, 4,"
            " None),\n"
            "      lib.pgcn_transformer_backward_rows(C.byref(w), 2, 0, 2, p, p, None, 0.5, None, None, 0, 1.0, p, p,"
            " p, p, p, None, 4, None),\n"
            "      lib.pgcn_transformer_backward_cols(C.byref(w), 2, 0, 2, p, p, None, 0.5, None, None, 0, 1.0, p, p,"
            " p, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_transformer_last_error().decode())\n" % ROOT)
    cabi.load_transformer()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 3)
    assert [int(x) for x in parts[:3]] == [-4, -4, -4] and "no CUDA device" in parts[3]


@pytest.mark.parametrize("heads,p", [(1, 0.0), (2, 0.0), (4, 0.3), (8, 0.3)])
def test_oracle_gradients_equal_torch_autograd_in_fp64(heads, p):
    rs = np.random.RandomState(3 + heads)
    A = sp.random(40, 50, density=0.15, random_state=rs, format="csr")
    A.indices[::7] = A.indices[1::7][:len(A.indices[::7])]          # some repeated columns in a row
    A.indptr[5:8] = A.indptr[5]                                      # empty rows
    A.indptr[8:] = np.maximum(A.indptr[8:], A.indptr[5])
    r, c = tro.entries(A.indptr, A.indices[:A.indptr[-1]])
    rows, cols = torch.from_numpy(r), torch.from_numpy(c)
    f = 2 * heads
    Q, gZ = rs.standard_normal((40, f)), rs.standard_normal((40, f))
    K, V = rs.standard_normal((50, f)), rs.standard_normal((50, f))
    scale = 0.7
    M = do.weights(r, c, heads, p, 12345, 3).numpy() if p > 0 else None
    if M is not None:
        assert (M == 0).any() and (M > 1).any()
    got = tro.attention(A.indptr, A.indices[:A.indptr[-1]], 50, Q, K, V, gZ, heads, scale, 16, M)
    Qt, Kt, Vt = (torch.tensor(x, requires_grad=True) for x in (Q, K, V))
    Z = tro.torch_transformer(rows, cols, 40, Qt, Kt, Vt, heads, scale, None if M is None else torch.from_numpy(M))
    Z.backward(torch.from_numpy(gZ))
    for name, want in (("Z", Z.detach()), ("dQ", Qt.grad), ("dK", Kt.grad), ("dV", Vt.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)
        assert (got[name][1] > 0).all(), name
    # L is the rows' log-sum-exp of the scores
    s = (Q[r].reshape(-1, heads, 2) * K[c].reshape(-1, heads, 2)).sum(2) * scale
    for i in (0, 12, 39):
        sel = r == i
        if sel.any():
            np.testing.assert_allclose(got["L"][0][i], np.log(np.exp(s[sel]).sum(0)), rtol=1e-12)
    assert np.isneginf(got["L"][0][6]).all()


def test_oracle_fp32_reference_propagates_special_values():
    rowptr, colidx = np.array([0, 2, 3, 3]), np.array([0, 1, 1])
    f32 = lambda a: np.array(a, np.float32)
    Q = f32([[np.inf], [1.0], [1.0]])
    K = f32([[1.0], [-1.0]])
    V = f32([[1.0], [2.0]])
    items = np.array([[0, 0, 2, -1], [1, 2, 3, -1], [2, 3, 3, -1]], np.int32)
    out = tro.fp32_reference(rowptr, colidx, 2, Q, K, V, f32([[1.0], [1.0], [1.0]]), 1, 1.0, items,
                             np.zeros((0, 3), np.int32))
    assert np.isnan(out["Z"][0, 0])                # scores +inf and -inf: exp(inf - inf)
    assert out["Z"][1, 0] == 2.0 and out["Z"][2, 0] == 0.0
    assert np.isneginf(out["L"][2, 0])


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--heads", "3"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--heads", "16"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "12", "--heads", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--heads", "two"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--attn-dropout", "1.0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--attn-dropout", "-0.1"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import transformer
    with pytest.raises(SystemExit) as e:
        transformer.main(argv)
    assert e.value.code == 2
    assert "usage: PTRANSFORMER.py" in capsys.readouterr().out


def test_cli_run_refuses_gloo():
    from pgcn_b200 import transformer
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        transformer.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")


class _FakePlan:
    m, n, f_max, _bound, layout, device = 4, 4, 8, True, "local", torch.device("cpu")

    def gated_walks(self):
        return None, None

    def global_ids(self):
        return None


def test_aggregate_transformer_refusals():
    from pgcn_b200 import op
    x = torch.zeros((4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_transformer(_FakePlan(), x, x, x, 2)
    with pytest.raises(ValueError, match="f_max >= 2f"):
        op.aggregate_transformer(_FakePlan(), torch.zeros((4, 5)), x, x, 1)
    with pytest.raises(ValueError, match="heads=3"):
        op.aggregate_transformer(_FakePlan(), x, x, x, 3)
    with pytest.raises(ValueError, match="multiple"):
        op.aggregate_transformer(_FakePlan(), torch.zeros((4, 6)), x, x, 4)
    big = _FakePlan()
    big.f_max = 1024
    with pytest.raises(ValueError, match="f <= 256"):
        op.aggregate_transformer(big, torch.zeros((4, 264)), x, x, 1)


def test_default_scale_is_the_float32_inverse_root_of_the_head_width():
    from pgcn_b200 import op
    for f, heads in ((128, 4), (136, 8), (3, 1)):
        assert op.transformer_scale(f, heads) == float(np.float32(1.0 / np.sqrt(f / heads)))
