"""CPU-side checks of the graph transformer attention with edge features: include/pgcn_transformer_edge.h against its
binding, libpgcn_transformer_edge.so's exports, architecture and kernel manifest, the other libraries' unchanged
manifests, the libraries' separate dependency lists and the shared transformer math, the refusals of the C entry
points (bad arguments, no GPU) and of op.aggregate_transformer_edge, the oracle's analytic gradients against torch
autograd in fp64 with and without a mask, and PTRANSFORMER.py's usage errors for --edge-values."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import dropout_oracle as do
import transformer_edge_oracle as teo
import transformer_oracle as tro
from conftest import ROOT
from pgcn_b200 import build, cabi
from test_transformer_host import header_functions

MANIFEST = os.path.join(ROOT, "tests", "transformer_edge_kernel_instances.txt")


def test_header_and_binding_agree():
    fns = header_functions("pgcn_transformer_edge.h")
    assert sorted(fns) == sorted(cabi.TRANSFORMER_EDGE_SYMBOLS)
    lib = cabi.load_transformer_edge()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS, cabi.TRANSFORMER_SYMBOLS,
                  cabi.GATEDGCN_SYMBOLS):
        assert not set(fns) & set(other)
    txt = open(os.path.join(ROOT, "include", "pgcn_transformer_edge.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_transformer_edge()
    for name in cabi.TRANSFORMER_EDGE_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_transformer_edge.so does not export " + name
    assert b"sm_90a" in lib.pgcn_transformer_edge_version()
    assert os.path.basename(cabi.transformer_edge_lib_path()) == "libpgcn_transformer_edge.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_transformer_edge()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.transformer_edge_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifests():
    lk = _tools()
    cabi.load_transformer_edge()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.transformer_edge_lib_path()) == want
    for load, path, manifest in ((cabi.load_transformer, cabi.transformer_lib_path, "transformer_kernel_instances.txt"),
                                 (cabi.load_gatedgcn, cabi.gatedgcn_lib_path, "gatedgcn_kernel_instances.txt"),
                                 (cabi.load_gated, cabi.gated_lib_path, "gated_kernel_instances.txt"),
                                 (cabi.load_dropout, cabi.dropout_lib_path, "dropout_kernel_instances.txt"),
                                 (cabi.load, cabi.lib_path, "kernel_instances.txt")):
        load()
        with open(os.path.join(ROOT, "tests", manifest)) as fh:
            assert lk.list_kernels(lib=path()) == [ln.strip() for ln in fh if ln.strip()], manifest


def test_each_library_has_its_own_dependencies():
    math = os.path.join(build.CSRC, "transformer_math.cuh")
    shared = {os.path.abspath(build.__file__), os.path.join(ROOT, "include", "pgcn_gated.h"),
              os.path.join(build.CSRC, "philox.cuh")}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS, build.GATEDGCN_DEPS):
        assert not set(build.TRANSFORMER_EDGE_DEPS) & set(other) - shared
    assert not set(build.TRANSFORMER_EDGE_DEPS) & set(build.TRANSFORMER_DEPS) - shared - {math}
    for name in (os.path.join(build.CSRC, "transformer_edge.cu"), math, os.path.join(build.CSRC, "philox.cuh"),
                 os.path.join(ROOT, "include", "pgcn_transformer_edge.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.TRANSFORMER_EDGE_DEPS
    assert build.TRANSFORMER_EDGE_SOURCES == [os.path.join(build.CSRC, "transformer_edge.cu")]
    # the lane math has one definition, which both transformer libraries depend on
    assert math in build.TRANSFORMER_DEPS
    for src in ("transformer.cu", "transformer_edge.cu"):
        txt = open(os.path.join(build.CSRC, src)).read()
        assert '#include "transformer_math.cuh"' in txt and "float head_dot(" not in txt and "struct TrArgs" not in txt


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_transformer_edge()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)

    def fwd(walk=C.byref(w), m=4, h=0, heads=1, Q=p, KV=p, KVh=None, E=p, scale=0.5, gid=None, drop=None, ks=1.0,
            Z=p, L=p, work=None, f=8):
        return lib.pgcn_transformer_edge_forward(walk, m, h, heads, Q, KV, KVh, E, scale, gid, drop, 0, ks, Z, L,
                                                 work, f, None)

    def rows(walk=C.byref(w), m=4, h=0, heads=1, E=p, gZ=p, Z=p, L=p, dQ=p, D=p, PS=p, dE=None, work=None, f=8):
        return lib.pgcn_transformer_edge_backward_rows(walk, m, h, heads, p, p, None, E, 0.5, None, None, 0, 1.0, gZ,
                                                       Z, L, dQ, D, PS, dE, work, f, None)

    def cols(walk=C.byref(_walk(6)), perm=p, m=4, h=2, heads=1, Q=p, gZ=p, PS=p, scale=0.5, dKV=p, work=None, f=8):
        return lib.pgcn_transformer_edge_backward_cols(walk, perm, m, h, heads, Q, gZ, PS, scale, dKV, work, f, None)

    def err():
        return lib.pgcn_transformer_edge_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(heads=3) == -1 and b"heads=3" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=260, heads=4) == -1 and b"f=260" in err()
    assert fwd(f=6, heads=4) == -1 and b"multiple" in err()
    assert fwd(scale=float("nan")) == -1 and b"scale" in err()
    assert fwd(Q=None) == -1 and b"Q_own" in err()
    assert fwd(h=2) == -1 and b"KV_halo" in err()
    assert fwd(E=None) == -1 and b"null E" in err()
    assert fwd(drop=p) == -1 and b"gid" in err()
    assert fwd(drop=p, gid=p, ks=float("inf")) == -1 and b"keep_scale" in err()
    assert fwd(walk=C.byref(_walk(4, nitems=3))) == -1 and b"work table" in err()
    assert fwd(walk=C.byref(_walk(4, nslots=2))) == -1 and b"work" in err()
    assert fwd(Z=None) == -1 and b"output" in err()
    assert rows(E=None) == -1 and b"null E" in err()
    assert rows(gZ=None) == -1 and b"gZ" in err()
    assert rows(D=None) == -1 and b"dQ/D" in err()
    assert rows(PS=None) == -1 and b"PS" in err()
    assert cols(walk=C.byref(w)) == -1 and b"rows" in err()                # rows != m + h
    assert cols(perm=None) == -1 and b"perm" in err()
    assert cols(PS=None) == -1 and b"Q_own/gZ/PS" in err()
    assert cols(dKV=None) == -1 and b"dKV" in err()
    assert cols(heads=16) == -1 and b"heads=16" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_transformer_edge(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_transformer_edge_load(),\n"
            "      lib.pgcn_transformer_edge_forward(C.byref(w), 2, 0, 2, p, p, None, p, 0.5, p, p, 7, 2.0, p, p, None,"
            " 4, None),\n"
            "      lib.pgcn_transformer_edge_backward_rows(C.byref(w), 2, 0, 2, p, p, None, p, 0.5, None, None, 0, 1.0,"
            " p, p, p, p, p, p, None, None, 4, None),\n"
            "      lib.pgcn_transformer_edge_backward_cols(C.byref(w), p, 2, 0, 2, p, p, p, 0.5, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_transformer_edge_last_error().decode())\n" % ROOT)
    cabi.load_transformer_edge()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 4)
    assert [int(x) for x in parts[:4]] == [-4, -4, -4, -4] and "no CUDA device" in parts[4]


def _graph(rs):
    A = sp.random(40, 50, density=0.15, random_state=rs, format="csr")
    A.indices[::7] = A.indices[1::7][:len(A.indices[::7])]          # some repeated columns in a row
    A.indptr[5:8] = A.indptr[5]                                      # empty rows
    A.indptr[8:] = np.maximum(A.indptr[8:], A.indptr[5])
    return A.indptr, A.indices[:A.indptr[-1]]


@pytest.mark.parametrize("heads,p", [(1, 0.0), (2, 0.0), (4, 0.3), (8, 0.3)])
def test_oracle_gradients_equal_torch_autograd_in_fp64(heads, p):
    rs = np.random.RandomState(5 + heads)
    rowptr, idx = _graph(rs)
    r, c = tro.entries(rowptr, idx)
    rows, cols = torch.from_numpy(r), torch.from_numpy(c)
    f = 2 * heads
    Q, gZ = rs.standard_normal((40, f)), rs.standard_normal((40, f))
    K, V = rs.standard_normal((50, f)), rs.standard_normal((50, f))
    E = rs.standard_normal((len(r), f))
    scale = 0.7
    M = do.weights(r, c, heads, p, 12345, 3).numpy() if p > 0 else None
    if M is not None:
        assert (M == 0).any() and (M > 1).any()
    got = teo.attention(rowptr, idx, 50, Q, K, V, E, gZ, heads, scale, 16, M)
    Qt, Kt, Vt, Et = (torch.tensor(x, requires_grad=True) for x in (Q, K, V, E))
    Z = teo.torch_transformer_edge(rows, cols, 40, Qt, Kt, Vt, Et, heads, scale,
                                   None if M is None else torch.from_numpy(M))
    Z.backward(torch.from_numpy(gZ))
    for name, want in (("Z", Z.detach()), ("dQ", Qt.grad), ("dK", Kt.grad), ("dV", Vt.grad), ("dE", Et.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)
        assert (got[name][1] > 0).all(), name
    # with E = 0 the values and the bounds' magnitudes are the attention's without edges
    zero = teo.attention(rowptr, idx, 50, Q, K, V, np.zeros_like(E), gZ, heads, scale, 16, M)
    plain = tro.attention(rowptr, idx, 50, Q, K, V, gZ, heads, scale, 16, M)
    for name in ("Z", "L", "dQ", "dK", "dV"):
        np.testing.assert_allclose(zero[name][0], plain[name][0], rtol=1e-13, atol=1e-13, err_msg=name)
        assert (zero[name][1] >= plain[name][1]).all(), name


def test_oracle_bound_covers_an_fp32_restatement():
    """The kernels' formulas evaluated in fp32 with numpy (kk and vv rounded first, a plain softmax) lie within the
    oracle's bound of fp64."""
    rs = np.random.RandomState(11)
    rowptr, idx = _graph(rs)
    r, c = tro.entries(rowptr, idx)
    heads, f = 2, 8
    f32 = np.float32
    Q, gZ = (rs.standard_normal((40, f)).astype(f32) for _ in range(2))
    K, V = (rs.standard_normal((50, f)).astype(f32) for _ in range(2))
    E = rs.standard_normal((len(r), f)).astype(f32)
    sc = f32(0.5)
    ref = teo.attention(rowptr, idx, 50, Q, K, V, E, gZ, heads, float(sc), 16)
    KK, VV = K[c] + E, V[c] + E
    s = (Q[r] * KK).reshape(-1, heads, f // heads).sum(2, dtype=f32) * sc
    m = np.full((40, heads), -np.inf, f32)
    np.maximum.at(m, r, s)
    e = np.exp(s - m[r])
    l = np.zeros((40, heads), f32)
    np.add.at(l, r, e)
    P = e / l[r]
    Z = np.zeros((40, f), f32)
    np.add.at(Z, r, np.repeat(P, f // heads, 1) * VV)
    has = np.diff(rowptr) > 0
    val, tol = ref["Z"]
    assert (np.abs(Z[has].astype(np.float64) - val[has]) <= tol[has]).all()


class _FakePlan:
    m, n, f_max, _bound, layout, device = 4, 4, 8, True, "local", torch.device("cpu")

    class lp:
        m, h = 4, 0

        @staticmethod
        def nnz():
            return 6

    def gated_walks(self):
        return None, None

    def global_ids(self):
        return None

    def transposed_entries(self):
        return None


def test_aggregate_transformer_edge_refusals(monkeypatch):
    from pgcn_b200 import op
    x, E = torch.zeros((4, 4)), torch.zeros((6, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_transformer_edge(_FakePlan(), x, x, x, E, 2)
    with pytest.raises(ValueError, match="f_max >= 2f"):
        op.aggregate_transformer_edge(_FakePlan(), torch.zeros((4, 5)), x, x, E, 1)
    with pytest.raises(ValueError, match="heads=3"):
        op.aggregate_transformer_edge(_FakePlan(), x, x, x, E, 3)
    with pytest.raises(ValueError, match="multiple"):
        op.aggregate_transformer_edge(_FakePlan(), torch.zeros((4, 6)), x, x, E, 4)
    big = _FakePlan()
    big.f_max = 1024
    with pytest.raises(ValueError, match="f <= 256"):
        op.aggregate_transformer_edge(big, torch.zeros((4, 264)), x, x, E, 1)
    drop = op.EdgeDropout(0.1, 1, torch.device("meta"))
    with pytest.raises(ValueError, match="EdgeDropout state lives on meta"):
        op.aggregate_transformer_edge(_FakePlan(), x, x, x, E, 2, drop=drop)

    # past the device check (this machine has no GPU): the operands' shapes, dtypes and the plan's binding
    def f32_only(t, what):
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32, got %s" % (what, t.dtype))
    monkeypatch.setattr(op, "_check_f32", f32_only)
    for bad, match in ((torch.zeros((5, 4)), r"E must be \[6, 4\]"), (torch.zeros((6, 2)), r"E must be \[6, 4\]"),
                       (torch.zeros(24), r"E must be \[6, 4\]")):
        with pytest.raises(ValueError, match=match):
            op.aggregate_transformer_edge(_FakePlan(), x, x, x, bad, 2)
    with pytest.raises(TypeError, match="E must be float32"):
        op.aggregate_transformer_edge(_FakePlan(), x, x, x, E.double(), 2)
    with pytest.raises(TypeError, match="Q must be float32"):
        op.aggregate_transformer_edge(_FakePlan(), x.half(), x, x, E, 2)
    unbound = _FakePlan()
    unbound._bound = False
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_transformer_edge(unbound, x, x, x, E, 2)
    with pytest.raises(ValueError, match="snapshot"):
        op.aggregate_transformer_edge_backward(_FakePlan(), x, x, x, E, x, x, x, 2, drop=op.EdgeDropout(0.1, 1, "meta"))


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--edge-values=1"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--edge-values-on"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "12", "--heads", "8", "--edge-values"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--edge-values", "--attn-dropout",
     "1.0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8", "--edge-values"],
    ["-a", "x.mtx", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--edge-values"],   # -p missing
])
def test_cli_prints_usage_on_bad_edge_values_flags(argv, capsys):
    from pgcn_b200 import transformer
    with pytest.raises(SystemExit) as e:
        transformer.main(argv)
    assert e.value.code == 2
    out = capsys.readouterr().out
    assert "usage: PTRANSFORMER.py" in out and "[--edge-values]" in out


def test_edge_values_layer_draws_lin_edge_between_value_and_skip():
    """The layer's parameters are PyG's TransformerConv(edge_dim=1) order, and the flag changes no draw of a layer
    without it."""
    from pgcn_b200.transformer import PTRANSFORMER

    class Plan:
        class lp:
            vals = np.arange(6, dtype=np.float64)

    torch.manual_seed(3)
    plain = PTRANSFORMER(Plan(), 4, 4)
    torch.manual_seed(3)
    edge = PTRANSFORMER(Plan(), 4, 4, edge_values=True)
    assert [n for n, _ in plain.named_parameters()] == ["lin_key.weight", "lin_key.bias", "lin_query.weight",
                                                        "lin_query.bias", "lin_value.weight", "lin_value.bias",
                                                        "lin_skip.weight", "lin_skip.bias"]
    assert [n for n, _ in edge.named_parameters()] == ["lin_key.weight", "lin_key.bias", "lin_query.weight",
                                                       "lin_query.bias", "lin_value.weight", "lin_value.bias",
                                                       "lin_edge.weight", "lin_skip.weight", "lin_skip.bias"]
    assert tuple(edge.lin_edge.weight.shape) == (4, 1) and "edge_input" not in edge.state_dict()
    assert torch.equal(edge.edge_input, torch.arange(6, dtype=torch.float32).reshape(-1, 1))
    want = teo.init_params(1, 4, 3)[0]
    got = [t.detach().numpy() for t in edge.parameters()]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert all(torch.equal(a, b) for a, b in zip(plain.lin_key.parameters(), edge.lin_key.parameters()))
