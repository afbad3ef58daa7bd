"""CPU-side checks of GATv2 attention with edge features: include/pgcn_gatv2_edge.h against its binding,
libpgcn_gatv2_edge.so's exports, architecture and kernel manifest, the libraries' separate dependency lists and the
shared transformer math, the refusals of the C entry points (bad arguments, no GPU) and of op.aggregate_gatv2_edge /
op.PGATv2EdgeAttention, the oracle's analytic gradients against torch autograd of a dense masked GATv2 in fp64 (inputs
at the LeakyReLU kink, with and without a dropout mask), pgat.PGATv2's parameter draws with and without edge_values,
and PGAT.py's usage errors for --edge-values."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_oracle as do
import gatv2_edge_oracle as geo
import gatv2_oracle as go
import transformer_oracle as tro
from conftest import ROOT
from pgcn_b200 import build, cabi
from test_transformer_host import header_functions

MANIFEST = os.path.join(ROOT, "tests", "gatv2_edge_kernel_instances.txt")


def test_header_and_binding_agree():
    fns = header_functions("pgcn_gatv2_edge.h")
    assert sorted(fns) == sorted(cabi.GATV2_EDGE_SYMBOLS)
    lib = cabi.load_gatv2_edge()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS, cabi.TRANSFORMER_SYMBOLS,
                  cabi.GATEDGCN_SYMBOLS, cabi.TRANSFORMER_EDGE_SYMBOLS, cabi.GINE_SYMBOLS, cabi.RGCN_SYMBOLS):
        assert not set(fns) & set(other)
    txt = open(os.path.join(ROOT, "include", "pgcn_gatv2_edge.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_gatv2_edge()
    for name in cabi.GATV2_EDGE_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_gatv2_edge.so does not export " + name
    assert b"sm_90a" in lib.pgcn_gatv2_edge_version()
    assert os.path.basename(cabi.gatv2_edge_lib_path()) == "libpgcn_gatv2_edge.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_gatv2_edge()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.gatv2_edge_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifest():
    lk = _tools()
    cabi.load_gatv2_edge()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.gatv2_edge_lib_path()) == want


def test_each_library_has_its_own_dependencies():
    math = os.path.join(build.CSRC, "transformer_math.cuh")
    shared = {os.path.abspath(build.__file__), os.path.join(ROOT, "include", "pgcn_gated.h"),
              os.path.join(build.CSRC, "philox.cuh")}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS, build.GATEDGCN_DEPS, build.GINE_DEPS,
                  build.RGCN_DEPS):
        assert not set(build.GATV2_EDGE_DEPS) & set(other) - shared
    for other in (build.TRANSFORMER_DEPS, build.TRANSFORMER_EDGE_DEPS):
        assert not set(build.GATV2_EDGE_DEPS) & set(other) - shared - {math}
    for name in (os.path.join(build.CSRC, "gatv2_edge.cu"), math, os.path.join(build.CSRC, "philox.cuh"),
                 os.path.join(ROOT, "include", "pgcn_gatv2_edge.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.GATV2_EDGE_DEPS
    assert build.GATV2_EDGE_SOURCES == [os.path.join(build.CSRC, "gatv2_edge.cu")]
    # the lane math is the transformer's one definition
    txt = open(os.path.join(build.CSRC, "gatv2_edge.cu")).read()
    assert '#include "transformer_math.cuh"' in txt and "float head_dot(" not in txt and "struct TrArgs" not in txt


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_work_rows_counts_the_slots_and_one_datt_partial_per_cta():
    lib = cabi.load_gatv2_edge()
    assert lib.pgcn_gatv2_edge_work_rows(None) == -1
    for nitems, nslots, want in ((4, 0, 1), (8, 0, 1), (9, 2, 4), (0, 0, 0), (1000, 7, 7 + 125)):
        assert lib.pgcn_gatv2_edge_work_rows(C.byref(_walk(0, nitems, nslots))) == want


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_gatv2_edge()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(4)

    def fwd(walk=C.byref(w), m=4, h=0, heads=1, XL=p, XLh=None, XR=p, att=p, E=p, slope=0.2, gid=None, drop=None,
            ks=1.0, Z=p, L=p, work=None, f=8):
        return lib.pgcn_gatv2_edge_forward(walk, m, h, heads, XL, XLh, XR, att, E, slope, gid, drop, 0, ks, Z, L, work,
                                           f, None)

    def rows(walk=C.byref(w), m=4, heads=1, att=p, E=p, gZ=p, Z=p, L=p, dXR=p, D=p, PS=p, G=p, datt=p, work=p, f=8):
        return lib.pgcn_gatv2_edge_backward_rows(walk, m, 0, heads, p, None, p, att, E, 0.2, None, None, 0, 1.0, gZ, Z,
                                                 L, dXR, D, PS, G, datt, work, f, None)

    def cols(walk=C.byref(_walk(6)), perm=p, m=4, h=2, heads=1, gZ=p, PS=p, G=p, dXL=p, work=None, f=8):
        return lib.pgcn_gatv2_edge_backward_cols(walk, perm, m, h, heads, gZ, PS, G, dXL, work, f, None)

    def err():
        return lib.pgcn_gatv2_edge_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(heads=3) == -1 and b"heads=3" in err()
    assert fwd(heads=16) == -1 and b"heads=16" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=260, heads=4) == -1 and b"f=260" in err()
    assert fwd(f=6, heads=4) == -1 and b"multiple" in err()
    assert fwd(XL=None) == -1 and b"XL_own" in err()
    assert fwd(XR=None) == -1 and b"XR" in err()
    assert fwd(h=2) == -1 and b"XL_halo" in err()
    assert fwd(att=None) == -1 and b"null att" in err()
    assert fwd(slope=float("nan")) == -1 and b"negative_slope" in err()
    assert fwd(slope=float("inf")) == -1 and b"negative_slope" in err()
    assert fwd(E=None) == -1 and b"null E" in err()
    assert fwd(drop=p) == -1 and b"gid" in err()
    assert fwd(drop=p, gid=p, ks=float("inf")) == -1 and b"keep_scale" in err()
    assert fwd(walk=C.byref(_walk(4, nitems=3))) == -1 and b"work table" in err()
    assert fwd(walk=C.byref(_walk(4, nslots=2))) == -1 and b"work" in err()
    assert fwd(Z=None) == -1 and b"output" in err()
    assert rows(E=None) == -1 and b"null E" in err()
    assert rows(att=None) == -1 and b"null att" in err()
    assert rows(gZ=None) == -1 and b"gZ" in err()
    assert rows(dXR=None) == -1 and b"dXR/D" in err()
    assert rows(PS=None) == -1 and b"PS/G" in err()
    assert rows(G=None) == -1 and b"PS/G" in err()
    assert rows(datt=None) == -1 and b"datt" in err()
    assert rows(work=None) == -1 and b"work" in err()
    assert rows(f=264, heads=8) == -1 and b"f=264" in err()
    assert cols(walk=C.byref(w)) == -1 and b"rows" in err()                # rows != m + h
    assert cols(perm=None) == -1 and b"perm" in err()
    assert cols(gZ=None) == -1 and b"gZ" in err()
    assert cols(PS=None) == -1 and b"PS/G" in err()
    assert cols(G=None) == -1 and b"PS/G" in err()
    assert cols(dXL=None) == -1 and b"dXL" in err()
    assert cols(heads=16) == -1 and b"heads=16" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_gatv2_edge(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_gatv2_edge_load(),\n"
            "      lib.pgcn_gatv2_edge_forward(C.byref(w), 2, 0, 2, p, None, p, p, p, 0.2, p, p, 7, 2.0, p, p, None, 4,"
            " None),\n"
            "      lib.pgcn_gatv2_edge_backward_rows(C.byref(w), 2, 0, 2, p, None, p, p, p, 0.2, None, None, 0, 1.0,"
            " p, p, p, p, p, p, p, p, p, 4, None),\n"
            "      lib.pgcn_gatv2_edge_backward_cols(C.byref(w), p, 2, 0, 2, p, p, p, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_gatv2_edge_last_error().decode())\n" % ROOT)
    cabi.load_gatv2_edge()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 4)
    assert [int(x) for x in parts[:4]] == [-4, -4, -4, -4] and "no CUDA device" in parts[4]


# ---- the oracle ------------------------------------------------------------------------------------------------------

def _graph(rs, nr=30, nc=36):
    """A CSR without repeated columns in a row (so that a dense [nr, nc] mask states it), with empty rows."""
    dense = rs.uniform(size=(nr, nc)) < 0.2
    dense[4:7] = False
    rowptr = np.concatenate([[0], np.cumsum(dense.sum(1))]).astype(np.int64)
    return rowptr, np.nonzero(dense)[1].astype(np.int64), dense


def dense_gatv2_edge(mask, xl, xr, att, Ed, slope, Md=None):
    """GATv2 with the edge term written densely: the score of every (i, j) pair from (xr[i] + xl[j]) + Ed[i, j],
    non-edges masked with -inf, rows without entries 0; Md [nr, nc, K] the dropout factors."""
    K, d = att.shape
    T = (xr[:, None, :] + xl[None, :, :]) + Ed
    S = (F.leaky_relu(T, slope).view(T.shape[0], T.shape[1], K, d) * att).sum(3)
    S = S.masked_fill(~mask[:, :, None], -float("inf"))
    has = mask.any(1)
    alpha = torch.where(has[:, None, None], torch.softmax(torch.where(has[:, None, None], S, torch.zeros_like(S)), 1),
                        torch.zeros_like(S))
    alpha = alpha * mask[:, :, None]
    if Md is not None:
        alpha = alpha * Md
    return torch.einsum("ijh,jhd->ihd", alpha, xl.view(-1, K, d)).reshape(T.shape[0], K * d)


@pytest.mark.parametrize("heads,p,kink", [(1, 0.0, False), (2, 0.0, True), (4, 0.3, False), (8, 0.3, True),
                                          (2, 0.5, True)])
def test_oracle_gradients_equal_dense_torch_autograd_in_fp64(heads, p, kink):
    rs = np.random.RandomState(7 + heads)
    rowptr, idx, dense = _graph(rs)
    r, c = tro.entries(rowptr, idx)
    f, slope = 2 * heads, 0.2
    if kink:            # halves: many t = (xr + xl) + E are exactly 0, in fp64 and in fp32
        draw = lambda *s: rs.randint(-2, 3, size=s) * 0.5
    else:
        draw = lambda *s: rs.standard_normal(s)
    XR, gZ, XL = draw(30, f), rs.standard_normal((30, f)), draw(36, f)
    E = draw(len(r), f)
    att = rs.standard_normal((heads, f // heads))
    if kink:
        t = (XR[r] + XL[c]) + E
        assert (t == 0).mean() > 0.1
    M = do.weights(r, c, heads, p, 12345, 3).numpy() if p > 0 else None
    if M is not None:
        assert (M == 0).any() and (M > 1).any()
    got = geo.attention(rowptr, idx, 36, XL, XR, att, E, gZ, slope, 16, M)
    mask = torch.from_numpy(dense)
    Ed = np.zeros((30, 36, f))
    Ed[r, c] = E
    Md = None
    if M is not None:
        Md = np.zeros((30, 36, heads))
        Md[r, c] = M
        Md = torch.from_numpy(Md)
    tl, tr, ta, te = (torch.tensor(x, requires_grad=True) for x in (XL, XR, att, Ed))
    Z = dense_gatv2_edge(mask, tl, tr, ta, te, slope, Md)
    Z.backward(torch.from_numpy(gZ))
    for name, want in (("Z", Z.detach()), ("dXL", tl.grad), ("dXR", tr.grad), ("datt", ta.grad),
                       ("dE", te.grad[r, c])):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-11, atol=1e-11, err_msg=name)
        assert (got[name][1] > 0).all(), name
    # the gather form of the same model, used by the loss curves, agrees too
    rows, cols = torch.from_numpy(r), torch.from_numpy(c)
    Zg = geo.torch_gatv2_edge(rows, cols, 30, tl.detach(), tr.detach(), ta.detach(), torch.from_numpy(E), slope,
                              None if M is None else torch.from_numpy(M))
    np.testing.assert_allclose(Zg.numpy(), Z.detach().numpy(), rtol=1e-12, atol=1e-12)


def test_zero_edge_term_gives_the_gatv2_oracle():
    rs = np.random.RandomState(3)
    rowptr, idx, _ = _graph(rs, 36, 36)
    r, c = tro.entries(rowptr, idx)
    heads, f, slope = 4, 16, 0.2
    XL, XR, gZ = (rs.standard_normal((36, f)) for _ in range(3))
    att = rs.standard_normal((heads, f // heads))
    got = geo.attention(rowptr, idx, 36, XL, XR, att, np.zeros((len(r), f)), gZ, slope, 16)
    Z, alpha, _ = go.forward(r, c, 36, XL, XR, att, slope)
    dxl, dxr, datt, _, dscore = go.backward(r, c, 36, XL, XR, att, slope, alpha, gZ)
    for name, want in (("Z", Z), ("dXL", dxl), ("dXR", dxr), ("datt", datt), ("P", alpha), ("ds", dscore)):
        np.testing.assert_allclose(got[name][0], want, rtol=1e-12, atol=1e-12, err_msg=name)


def test_oracle_bound_covers_an_fp32_restatement():
    """The formulas evaluated in fp32 with numpy (t rounded twice, a plain softmax and plain sums) lie within the
    oracle's bound of fp64, for every output."""
    rs = np.random.RandomState(11)
    rowptr, idx, _ = _graph(rs, 36, 36)
    r, c = tro.entries(rowptr, idx)
    heads, f, slope = 2, 8, 0.2
    f32 = np.float32
    XL, XR, gZ = (rs.standard_normal((36, f)).astype(f32) for _ in range(3))
    E = rs.standard_normal((len(r), f)).astype(f32)
    att = rs.standard_normal((heads, f // heads)).astype(f32)
    ref = geo.attention(rowptr, idx, 36, XL, XR, att, E, gZ, slope, 16)
    items = np.stack([np.arange(36), rowptr[:-1], rowptr[1:], -np.ones(36, np.int64)], 1)
    got = geo.fp32_reference(rowptr, idx, XL, XR, att, E, gZ, slope, items, np.zeros((0, 3), np.int64))
    has = np.diff(rowptr) > 0
    for name in ("Z", "L", "dXR", "dXL", "datt", "dE"):
        val, tol = ref[name]
        g = got[name]
        if name == "L":
            g, val, tol = g[has], val[has], tol[has]
        assert (np.abs(g.astype(np.float64) - val) <= tol).all(), name


# ---- the operator ----------------------------------------------------------------------------------------------------

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


def test_aggregate_gatv2_edge_refusals(monkeypatch):
    from pgcn_b200 import op
    x, E, att = torch.zeros((4, 4)), torch.zeros((6, 4)), torch.zeros((2, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, att, E)
    drop = op.EdgeDropout(0.1, 1, torch.device("meta"))
    with pytest.raises(ValueError, match="EdgeDropout state lives on meta"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, att, E, drop=drop)

    # past the device check (this machine has no GPU): the operands' shapes, dtypes and the plan's binding
    def f32_only(t, what):
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32, got %s" % (what, t.dtype))
    monkeypatch.setattr(op, "_check_f32", f32_only)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(ValueError, match="f_max"):
        op.aggregate_gatv2_edge(_FakePlan(), torch.zeros((4, 12)), torch.zeros((4, 12)), att, E)
    big = _FakePlan()
    big.f_max = 1024
    with pytest.raises(ValueError, match="f <= 256"):
        op.aggregate_gatv2_edge(big, torch.zeros((4, 264)), torch.zeros((4, 264)), torch.zeros((1, 264)), E)
    with pytest.raises(ValueError, match="same width"):
        op.aggregate_gatv2_edge(_FakePlan(), x, torch.zeros((4, 8)), att, E)
    with pytest.raises(ValueError, match=r"att must be \[heads, f / heads\]"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, torch.zeros(4), E)
    with pytest.raises(ValueError, match="heads=3"):
        op.aggregate_gatv2_edge(_FakePlan(), torch.zeros((4, 6)), torch.zeros((4, 6)), torch.zeros((3, 2)), E)
    with pytest.raises(ValueError, match="multiple"):
        op.aggregate_gatv2_edge(_FakePlan(), torch.zeros((4, 6)), torch.zeros((4, 6)), torch.zeros((4, 1)), E)
    with pytest.raises(ValueError, match=r"att must be \[2, 2\]"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, torch.zeros((2, 3)), E)
    with pytest.raises(TypeError, match="att must be a float32"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, att.double(), E)
    for bad in (torch.zeros((5, 4)), torch.zeros((6, 2)), torch.zeros(24)):
        with pytest.raises(ValueError, match=r"E must be \[6, 4\]"):
            op.aggregate_gatv2_edge(_FakePlan(), x, x, att, bad)
    with pytest.raises(TypeError, match="E must be float32"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x, att, E.double())
    with pytest.raises(TypeError, match="XL must be float32"):
        op.aggregate_gatv2_edge(_FakePlan(), x.half(), x, att, E)
    with pytest.raises(TypeError, match="XR must be float32"):
        op.aggregate_gatv2_edge(_FakePlan(), x, x.half(), att, E)
    unbound = _FakePlan()
    unbound._bound = False
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_gatv2_edge(unbound, x, x, att, E)
    with pytest.raises(ValueError, match="snapshot"):
        op.aggregate_gatv2_edge_backward(_FakePlan(), x, x, x, att, E, x, x, x, drop=op.EdgeDropout(0.1, 1, "meta"))


# ---- the layer and the command line ----------------------------------------------------------------------------------

class _Plan:
    class lp:
        vals = np.arange(6, dtype=np.float64)


def test_v2_layer_draws_lin_edge_after_the_other_parameters():
    """pgat.PGATv2's parameters: lin_l, lin_r and att as before, lin_edge drawn after them with edge_values, so the
    flag changes no draw of a layer without it."""
    from pgcn_b200.pgat import PGATv2
    torch.manual_seed(3)
    plain = PGATv2(_Plan(), 4, 4, 0.2, 2)
    torch.manual_seed(3)
    edge = PGATv2(_Plan(), 4, 4, 0.2, 2, edge_values=True)
    assert [n for n, _ in plain.named_parameters()] == ["att", "lin_l.weight", "lin_r.weight"]
    assert [n for n, _ in edge.named_parameters()] == ["att", "lin_l.weight", "lin_r.weight", "lin_edge.weight"]
    for a, b in zip(plain.parameters(), edge.parameters()):
        assert torch.equal(a, b)
    assert tuple(edge.lin_edge.weight.shape) == (4, 1) and edge.lin_edge.bias is None
    assert "edge_input" not in edge.state_dict()
    assert torch.equal(edge.edge_input, torch.arange(6, dtype=torch.float32).reshape(-1, 1))
    want = geo.init_params(1, 4, 3, 2)[0]
    got = {n: x.detach().numpy() for n, x in edge.named_parameters()}
    for name, w in zip(("lin_l.weight", "lin_r.weight", "att", "lin_edge.weight"), want):
        assert np.array_equal(got[name], w), name
    # the oracle of the layer without edges draws the same first three
    for a, b in zip(go.init_params(1, 4, 3, 2)[0], want[:3]):
        assert np.array_equal(a, b)


def test_v2_layer_refuses_dropout_without_edge_values():
    from pgcn_b200.op import EdgeDropout
    from pgcn_b200.pgat import PGATv2
    drop = EdgeDropout(0.5, 1, torch.device("meta"))
    with pytest.raises(ValueError, match="edge_values"):
        PGATv2(_Plan(), 4, 4, 0.2, 1, attn_dropout=drop)
    assert PGATv2(_Plan(), 4, 4, 0.2, 1, edge_values=True, attn_dropout=drop).attn_dropout is drop


BASE = ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8"]


@pytest.mark.parametrize("argv", [
    ["--edge-values"],                                         # without --v2
    ["--edge-values", "--attn-dropout", "0.5"],
    ["--v2", "--edge-values", "--heads", "3"],
    ["--v2", "--edge-values", "--heads", "16"],
    ["--v2", "--edge-values", "-f", "12", "--heads", "8"],
    ["--v2", "--edge-values", "--attn-dropout", "1.0"],
    ["--v2", "--edge-values", "--attn-dropout", "-0.1"],
    ["--v2", "--attn-dropout", "0.5"],                         # dropout without edges stays refused
])
def test_cli_prints_usage_on_bad_edge_values_flags(argv, capsys):
    from pgcn_b200 import pgat
    with pytest.raises(SystemExit) as e:
        pgat.main((BASE + argv) if "-f" not in argv else (BASE[:-2] + argv))
    assert e.value.code == 2
    out = capsys.readouterr().out
    assert "usage: PGAT.py" in out and "--edge-values" in out


@pytest.mark.parametrize("argv", [["--v2", "--edge-values=1"], ["--v2", "--edge-values-on"]])
def test_cli_refuses_a_malformed_edge_values_switch(argv, capsys):
    from pgcn_b200 import pgat
    with pytest.raises(SystemExit) as e:
        pgat.main(BASE + argv)
    assert e.value.code == 2


def test_cli_passes_edge_values_and_dropout_to_the_v2_run(monkeypatch):
    from pgcn_b200 import pgat
    seen = {}
    monkeypatch.setattr(pgat, "launch", lambda fn, rank, size, args, kw: seen.update(fn=fn, kw=kw))
    pgat.main(BASE + ["--v2", "--edge-values", "--attn-dropout", "0.25", "--heads", "2"])
    assert seen["fn"] is pgat.run
    assert seen["kw"]["v2"] and seen["kw"]["edge_values"] and seen["kw"]["attn_dropout"] == 0.25
    assert seen["kw"]["heads"] == 2
