"""CPU-side checks of R-GCN's relational aggregation: include/pgcn_rgcn.h against its binding, libpgcn_rgcn.so's
exports, architecture and kernel manifest, the libraries' separate dependency lists, the refusals of the C entry points
(bad arguments, no GPU) and of the operator, PgcnPlan.relation_walks' tables and refusals, the oracle against torch
autograd of a dense per-relation product in fp64, the synthetic relation hash's independence of the partition, and
PRGCN.py's parameter order and usage errors."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import rgcn_oracle as ro
from conftest import ROOT
from pgcn_b200 import build, cabi, graphio, plan as planmod
from test_gatedgcn_host import _dup_lp, _hub_lp
from test_gine_host import _cuda, _tools, header_functions

MANIFEST = os.path.join(ROOT, "tests", "rgcn_kernel_instances.txt")


def test_header_and_binding_agree():
    fns = header_functions("pgcn_rgcn.h")
    assert sorted(fns) == sorted(cabi.RGCN_SYMBOLS)
    lib = cabi.load_rgcn()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    for other in (cabi.SYMBOLS, cabi.HALO_SYMBOLS, cabi.DROPOUT_SYMBOLS, cabi.GATED_SYMBOLS, cabi.TRANSFORMER_SYMBOLS,
                  cabi.GATEDGCN_SYMBOLS, cabi.TRANSFORMER_EDGE_SYMBOLS, cabi.GINE_SYMBOLS):
        assert not set(fns) & set(other)
    # the walk struct is the gated library's, not a second definition
    txt = open(os.path.join(ROOT, "include", "pgcn_rgcn.h")).read()
    assert '#include "pgcn_gated.h"' in txt and "typedef struct" not in txt


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_rgcn()
    for name in cabi.RGCN_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_rgcn.so does not export " + name
    assert b"sm_90a" in lib.pgcn_rgcn_version()
    assert os.path.basename(cabi.rgcn_lib_path()) == "libpgcn_rgcn.so"


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_rgcn()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.rgcn_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifest():
    lk = _tools()
    cabi.load_rgcn()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.rgcn_lib_path()) == want


def test_each_library_has_its_own_dependencies(tmp_path):
    shared = {os.path.abspath(build.__file__), os.path.join(ROOT, "include", "pgcn_gated.h"),
              os.path.join(build.CSRC, "gated_math.cuh")}
    for other in (build.DEPS, build.DROPOUT_DEPS, build.GATED_DEPS, build.TRANSFORMER_DEPS, build.GATEDGCN_DEPS,
                  build.TRANSFORMER_EDGE_DEPS, build.GINE_DEPS):
        assert not set(build.RGCN_DEPS) & set(other) - shared
    for name in (os.path.join(build.CSRC, "rgcn.cu"), os.path.join(build.CSRC, "gated_math.cuh"),
                 os.path.join(ROOT, "include", "pgcn_rgcn.h"), os.path.join(ROOT, "include", "pgcn_gated.h")):
        assert name in build.RGCN_DEPS
    assert build.RGCN_SOURCES == [os.path.join(build.CSRC, "rgcn.cu")]
    deps = {"b200": build.DEPS, "dropout": build.DROPOUT_DEPS, "gated": build.GATED_DEPS,
            "transformer": build.TRANSFORMER_DEPS, "gatedgcn": build.GATEDGCN_DEPS,
            "transformer_edge": build.TRANSFORMER_EDGE_DEPS, "gine": build.GINE_DEPS, "rgcn": build.RGCN_DEPS}
    lib, newer = str(tmp_path / "lib.so"), str(tmp_path / "touched")
    for f in (lib, newer):
        open(f, "w").close()
    os.utime(lib, (1e9, 1e9))
    os.utime(newer, (2e9, 2e9))

    def stale_after_touching(src):
        return {name: build._stale(lib, [newer if d == src else lib for d in ds]) for name, ds in deps.items()}

    assert stale_after_touching(os.path.join(build.CSRC, "rgcn.cu")) == {n: n == "rgcn" for n in deps}
    for src in (os.path.join(build.CSRC, "gine.cu"), os.path.join(build.CSRC, "gatedgcn.cu"),
                os.path.join(build.CSRC, "gated.cu"), os.path.join(build.CSRC, "transformer_edge.cu"),
                os.path.join(build.CSRC, "pgcn_b200.cu"), os.path.join(build.CSRC, "edge_dropout.cu"),
                os.path.join(build.CSRC, "transformer.cu")):
        assert not stale_after_touching(src)["rgcn"], src


def _walk(rows, nitems=None, nslots=0):
    return cabi.PgcnGatedWalk(8, 16, 8, rows, rows if nitems is None else nitems, 0, nslots)


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_rgcn()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    w = _walk(8)                                                          # m = 4, R = 2

    def fwd(walk=C.byref(w), perm=p, m=4, h=0, R=2, X=p, Xh=None, wt=p, Z=p, work=None, f=8):
        return lib.pgcn_rgcn_forward(walk, perm, m, h, R, X, Xh, wt, Z, work, f, None)

    def bwd(walk=C.byref(_walk(6)), perm=p, m=4, h=2, R=2, gZ=p, wt=None, dX=p, work=None, f=8):
        return lib.pgcn_rgcn_backward(walk, perm, m, h, R, gZ, wt, dX, work, f, None)

    def err():
        return lib.pgcn_rgcn_last_error()

    assert fwd(walk=None) == -1 and b"null walk" in err()
    assert fwd(m=5) == -1 and b"rows" in err()
    assert fwd(R=4) == -1 and b"rows" in err()                              # rows != m R
    assert fwd(m=-1) == -1 and b"sizes" in err()
    assert fwd(R=0) == -1 and b"R=0" in err()
    assert fwd(R=-3) == -1 and b"R=-3" in err()
    assert fwd(m=1 << 30, R=2) == -1 and b"2^31" in err()
    assert fwd(f=0) == -1 and b"f=0" in err()
    assert fwd(f=(1 << 24) + 1) == -1 and b"f=" in err()
    assert fwd(X=None) == -1 and b"X_own" in err()
    assert fwd(h=2) == -1 and b"X_halo" in err()
    assert fwd(Z=None) == -1 and b"output" in err()
    assert fwd(perm=None) == -1 and b"perm" in err()                       # weights need perm
    assert fwd(walk=C.byref(_walk(8, nitems=7))) == -1 and b"work table" in err()
    assert fwd(walk=C.byref(_walk(8, nslots=2))) == -1 and b"work" in err()
    assert fwd(walk=C.byref(cabi.PgcnGatedWalk(None, None, None, 8, 8, 0, 0))) == -1 and b"null idx" in err()
    assert bwd(walk=C.byref(w)) == -1 and b"rows" in err()                 # rows != m + h
    assert bwd(f=-3) == -1 and b"f=-3" in err()
    assert bwd(R=0) == -1 and b"R=0" in err()
    assert bwd(wt=p, perm=None) == -1 and b"perm" in err()
    assert bwd(gZ=None) == -1 and b"gZ" in err()
    assert bwd(dX=None) == -1 and b"dX" in err()
    assert bwd(walk=C.byref(_walk(6, nslots=1))) == -1 and b"work" in err()


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_rgcn(build_if_missing=False)\n"
            "b = (C.c_float * 64)(); p = C.cast(b, C.c_void_p).value\n"
            "w = cabi.PgcnGatedWalk(p, p, p, 4, 4, 0, 0)\n"
            "t = cabi.PgcnGatedWalk(p, p, p, 2, 2, 0, 0)\n"
            "rc = [lib.pgcn_rgcn_load(),\n"
            "      lib.pgcn_rgcn_forward(C.byref(w), p, 2, 0, 2, p, None, p, p, None, 4, None),\n"
            "      lib.pgcn_rgcn_backward(C.byref(t), p, 2, 0, 2, p, None, p, None, 4, None)]\n"
            "print(*rc, lib.pgcn_rgcn_last_error().decode())\n" % ROOT)
    cabi.load_rgcn()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    parts = out.stdout.split(" ", 3)
    assert [int(x) for x in parts[:3]] == [-4, -4, -4] and "no CUDA device" in parts[3]


# ---- PgcnPlan.relation_walks ----------------------------------------------------------------------------------------

class _HostPlan(planmod.PgcnPlan):
    """A PgcnPlan's host side only (no device handle): relation_walks and transposed_entries on the CPU."""

    def __init__(self, lp):
        self.lp = lp
        self.device = torch.device("cpu")
        self._transposed_entries = None
        self._relation_walks = {}

    def close(self):
        pass


def _karate_lp():
    from harness import karate
    A = karate()
    return planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)


def _lp(case):
    return {"karate": _karate_lp, "hub": _hub_lp, "dup": _dup_lp}[case]()


@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("case", ["karate", "hub", "dup"])
def test_relation_walks_contents(case, R, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    lp = _lp(case)
    nnz, m = lp.nnz(), lp.m
    rel = torch.from_numpy(np.random.RandomState(R).randint(0, R, nnz))
    plan = _HostPlan(lp)
    fwd, tr, perm_f, mean, R_ = plan.relation_walks(rel, R)
    assert R_ == R and plan.relation_walks(rel, R).fwd is fwd              # cached
    r = rel.numpy()
    rows = np.repeat(np.arange(m), np.diff(lp.rowptr.astype(np.int64)))
    v = rows * R + r
    pf = perm_f.numpy()
    assert pf.dtype == np.int32 and np.array_equal(np.sort(pf), np.arange(nnz))
    # sorted by virtual row, and stable: a virtual row keeps its entries in forward order
    assert (np.diff(v[pf]) >= 0).all()
    same = np.diff(v[pf]) == 0
    assert (np.diff(pf)[same] > 0).all()
    items = fwd.items.numpy()
    assert fwd.rows == m * R and fwd.c.rows == m * R
    vptr = np.concatenate([[0], np.cumsum(np.bincount(v, minlength=m * R))])
    for row, e0, e1, slot in items[items[:, 3] < 0]:
        assert e0 == vptr[row] and e1 == vptr[row + 1]
    assert sorted(set(items[:, 0])) == list(range(m * R))                 # every virtual row, empty ones included
    assert np.array_equal(fwd.idx.numpy(), lp.colidx[pf])
    # the transposed walk: the plan's transposed CSR with virtual row indices
    pt = plan.transposed_entries().numpy()
    assert tr.rows == m + lp.h
    assert np.array_equal(tr.idx.numpy(), lp.t_colidx.astype(np.int64) * R + r[pt])
    assert np.array_equal(tr.idx.numpy() // R, lp.t_colidx) and np.array_equal(tr.idx.numpy(), v[pt])
    # mean weights: the fp32 quotient 1 / c of every entry's pair
    cnt = np.bincount(v, minlength=m * R)
    assert mean.dtype == torch.float32
    assert np.array_equal(mean.numpy(), np.float32(1) / cnt[v].astype(np.float32))
    assert np.array_equal(mean.numpy(), ro.kernel_weights(lp.rowptr, r, R, aggr="mean"))
    if R > 1:
        assert (cnt == 0).any()                                           # empty (row, relation) pairs exist


def test_relation_walks_cache_follows_the_tensor_and_its_version(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    lp = _karate_lp()
    plan = _HostPlan(lp)
    rel = torch.zeros(lp.nnz(), dtype=torch.int64)
    a = plan.relation_walks(rel, 2)
    assert plan.relation_walks(rel, 2) is a
    assert plan.relation_walks(rel, 3) is not a                           # another R
    assert plan.relation_walks(rel.clone(), 2) is not a                   # another tensor
    rel[::2] = 1                                                           # an in-place change moves the version
    b = plan.relation_walks(rel, 2)
    assert b is not a and (b.tr.idx.numpy() % 2 == 1).any()
    assert sum(1 for v in plan._relation_walks.values() if v[0] is rel) == 1


def test_relation_walks_refuses_a_capture(monkeypatch):
    lp = _karate_lp()
    plan = _HostPlan(lp)
    rel = torch.zeros(lp.nnz(), dtype=torch.int32)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(RuntimeError, match=r"relation_walks.*before the capture"):
        plan.relation_walks(rel, 2)
    assert plan._relation_walks == {}
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    walks = plan.relation_walks(rel, 2)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    assert plan.relation_walks(rel, 2) is walks                           # built before the capture: taken as is


def test_relation_walks_rejects_bad_input(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    lp = _karate_lp()
    plan = _HostPlan(lp)
    nnz = lp.nnz()
    good = torch.zeros(nnz, dtype=torch.int64)
    bad_value = good.clone()
    bad_value[5] = 3
    negative = good.clone()
    negative[-1] = -1
    with pytest.raises(ValueError, match=r"relation 3, outside \[0, R\)"):
        plan.relation_walks(bad_value, 3)
    with pytest.raises(ValueError, match="relation -1"):
        plan.relation_walks(negative, 3)
    for shape in ((nnz - 1,), (nnz, 1), (1, nnz)):
        with pytest.raises(ValueError, match=r"rel must be \[%d\]" % nnz):
            plan.relation_walks(torch.zeros(shape, dtype=torch.int64), 2)
    for dtype in (torch.float32, torch.bool):
        with pytest.raises(TypeError, match="integer"):
            plan.relation_walks(torch.zeros(nnz, dtype=dtype), 2)
    with pytest.raises(TypeError, match="integer tensor"):
        plan.relation_walks(np.zeros(nnz, np.int64), 2)
    for R in (0, -2):
        with pytest.raises(ValueError, match="R=%d" % R):
            plan.relation_walks(good, R)
    for R in (2.0, True):
        with pytest.raises(TypeError):
            plan.relation_walks(good, R)
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        plan.relation_walks(good, (2 ** 31) // lp.m + 1)
    assert plan._relation_walks == {}


# ---- the operator's refusals ----------------------------------------------------------------------------------------

class _FakeLocal:
    m, h = 4, 0

    def nnz(self):
        return 6


class _FakePlan:
    m, n, f_max, layout, device, lp = 4, 4, 8, "local", torch.device("cpu"), _FakeLocal()

    def __init__(self, bound=True):
        self._bound = bound

    def transposed_entries(self):
        return None


_WALKS = planmod.RelationWalks(None, None, None, "mean weights", 2)


def test_operator_refusals():
    from pgcn_b200 import op
    x = _cuda(4, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_rgcn(_FakePlan(), _WALKS, torch.zeros((4, 8)), None)
    with pytest.raises(TypeError, match="float32"):
        op.aggregate_rgcn(_FakePlan(), _WALKS, _cuda(4, 8, dtype=torch.float64), None)
    with pytest.raises(ValueError, match=r"X must be \[4, f\]"):
        op.aggregate_rgcn(_FakePlan(), _WALKS, _cuda(5, 8), None)
    with pytest.raises(ValueError, match="f_max"):
        op.aggregate_rgcn(_FakePlan(), _WALKS, _cuda(4, 12), None)
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_rgcn(_FakePlan(bound=False), _WALKS, x, None)
    for bad in ((4, 8), (4, 3, 8), (5, 2, 8)):
        with pytest.raises(ValueError, match=r"gZ must be \[4, 2, f\]"):
            op.aggregate_rgcn_backward(_FakePlan(), _WALKS, _cuda(*bad), None)
    with pytest.raises(ValueError, match="f_max"):
        op.aggregate_rgcn_backward(_FakePlan(), _WALKS, _cuda(4, 2, 12), None)
    with pytest.raises(RuntimeError, match="bind_values"):
        op.aggregate_rgcn_backward(_FakePlan(bound=False), _WALKS, _cuda(4, 2, 8), None)
    # the weights: an aggregation it does not know, and a w that asks for a gradient it has not
    with pytest.raises(ValueError, match="aggr='max'"):
        op.rgcn_weights(_FakePlan(), _WALKS, None, "max")
    w = torch.ones(6, requires_grad=True)
    with pytest.raises(ValueError, match="no gradient for its edge weights"):
        op.rgcn_weights(_FakePlan(), _WALKS, w, "add")
    assert op.rgcn_weights(_FakePlan(), _WALKS, None, "add") is None
    assert op.rgcn_weights(_FakePlan(), _WALKS, None, "mean") == "mean weights"
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        op.rgcn_weights(_FakePlan(), _WALKS, torch.ones(6), "add")


# ---- the oracle -----------------------------------------------------------------------------------------------------

def _typed_csr(rs, nr=40, nc=50, R=3):
    A = sp.random(nr, nc, density=0.15, random_state=rs, format="csr")
    n7 = len(A.indices[1::7])
    A.indices[:7 * n7:7] = A.indices[1::7]                           # some repeated columns in a row
    A.indptr[5:8] = A.indptr[5]                                      # empty rows
    A.indptr[8:] = np.maximum(A.indptr[8:], A.indptr[5])
    nnz = int(A.indptr[-1])
    return A.indptr, A.indices[:nnz], rs.randint(0, R, nnz)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("aggr", ["add", "mean"])
def test_oracle_equals_torch_autograd_of_dense_relations_in_fp64(aggr, weighted):
    rs = np.random.RandomState(5)
    R, f = 3, 6
    rowptr, idx, rel = _typed_csr(rs, R=R)
    nnz = len(idx)
    rel[rel == 2] = 1                                                # relation 2 never occurs
    w = rs.uniform(-2, 2, nnz).astype(np.float32) if weighted else None
    X = rs.standard_normal((50, f))
    gZ = rs.standard_normal((40, R, f))
    got = ro.terms(rowptr, idx, 50, rel, R, X, gZ, w, aggr)
    Xt = torch.tensor(X, requires_grad=True)
    Z = ro.torch_dense(rowptr, idx, 50, rel, R, Xt, w, aggr)
    (Z * torch.from_numpy(gZ)).sum().backward()
    for name, want in (("Z", Z.detach()), ("dX", Xt.grad)):
        np.testing.assert_allclose(got[name][0], want.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)
        assert (got[name][1] >= 0).all(), name
    assert np.all(got["Z"][0][5:7] == 0.0) and np.all(got["Z"][1][5:7] == 0.0)    # empty rows
    assert np.all(got["Z"][0][:, 2] == 0.0)                                         # a relation that never occurs
    if aggr == "mean" and not weighted:
        # each (row, relation) pair's mean of X over its entries
        rows, cols = ro.entries(rowptr, idx)
        i = rows[0]
        s = (rows == i) & (rel == rel[0])
        np.testing.assert_allclose(got["Z"][0][i, rel[0]], X[cols[s]].mean(0), rtol=1e-12)


@pytest.mark.parametrize("aggr,weighted", [("add", False), ("add", True), ("mean", False), ("mean", True)])
def test_oracle_bound_covers_an_fp32_evaluation(aggr, weighted):
    """The fp32 restatement (another summation order than the kernels' for dX) lies within the bound."""
    rs = np.random.RandomState(9)
    R, f = 4, 5
    rowptr, idx, rel = _typed_csr(rs, 60, 60, R)
    w = rs.uniform(-2, 2, len(idx)).astype(np.float32) if weighted else None
    X = (rs.standard_normal((60, f)) * 2).astype(np.float32)
    gZ = rs.standard_normal((60, R, f)).astype(np.float32)
    ref = ro.terms(rowptr, idx, 60, rel, R, X, gZ, w, aggr)
    got = ro.fp32_reference(rowptr, idx, 60, rel, R, X, gZ, w, aggr)
    for name in ("Z", "dX"):
        val, tol = ref[name]
        assert (np.abs(got[name].astype(np.float64) - val) <= tol + 1e-30).all(), name


def test_relation_hash_is_the_same_on_one_and_three_ranks(monkeypatch):
    """The synthetic relations, taken through edge_pairs() of a host plan, give every global entry the same type on
    1 rank and on each of 3 ranks."""
    from pgcn_b200.rgcn import relation_hash
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    A = sp.coo_matrix(graphio.synthetic_graph(3000, 40000, seed=7))
    pv = graphio.random_partvec(3000, 3, seed=1)
    R = 5

    def typed(lp):
        plan = _HostPlan(lp)
        plan._edge_pairs = None
        pairs = plan.edge_pairs().numpy().astype(np.int64)
        rel = relation_hash(plan.edge_pairs(), R).numpy()
        return {(int(a), int(b)): int(t) for (a, b), t in zip(pairs, rel)}

    one = typed(planmod.build_local_plan(A, np.zeros(3000, dtype=np.int64), 0, 1))
    parts = [typed(planmod.build_local_plan(A, pv, r, 3)) for r in range(3)]
    merged = {}
    for p in parts:
        assert not set(p) & set(merged)
        merged.update(p)
    assert merged == one
    assert set(one.values()) == set(range(R))
    rows, cols = np.array(list(one)).T
    assert np.array_equal(ro.relation_hash(rows, cols, R), np.array(list(one.values())))


def test_layer_draws_its_parameters_in_the_documented_order():
    from pgcn_b200 import rgcn

    class _Plan:
        def edge_pairs(self):
            return torch.tensor([[0, 1], [1, 0], [2, 2]], dtype=torch.int32)
    for bases, names in ((None, ("weight", "root", "bias")), (2, ("weight", "comp", "root", "bias"))):
        torch.manual_seed(3)
        model = rgcn.PRGCN(_Plan(), 4, 2, 3, bases)
        want = ro.init_params(2, 4, 3, bases, 3)
        got_names = [n for n, _ in model.named_parameters()]
        assert got_names == ["layers.%d.%s" % (l, p) for l in range(2) for p in names]
        got = [p.detach().numpy().astype(np.float64) for p in model.parameters()]
        flat = [x for layer in want for x in layer]
        assert len(got) == len(flat)
        for g, w in zip(got, flat):
            assert np.array_equal(g, w)
        assert tuple(model.layers[0].relation_weights().shape) == (3, 4, 4)
    # the layer's options: no root, no bias, add, and refused aggregations and bases
    layer = rgcn.RGCNLayer(_Plan(), None, 3, 4, 5, aggr="add", root_weight=False, bias=False)
    assert [n for n, _ in layer.named_parameters()] == ["weight"]
    with pytest.raises(ValueError, match="aggr"):
        rgcn.RGCNLayer(_Plan(), None, 3, 4, 5, aggr="max")
    with pytest.raises(ValueError, match="num_bases"):
        rgcn.RGCNLayer(_Plan(), None, 3, 4, 5, num_bases=0)


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8"],                 # no --relations
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--relations", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--relations", "two"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8", "--relations", "3",
     "--bases", "0"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8", "--relations", "3"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0", "--relations", "3"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "0", "-l", "2", "-f", "8", "--relations", "3"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "gloo", "-s", "1", "-l", "2", "-f", "8", "--relations", "3"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import rgcn
    with pytest.raises(SystemExit) as e:
        rgcn.main(argv)
    assert e.value.code == 2
    assert "usage: PRGCN.py" in capsys.readouterr().out


def test_cli_run_refuses_gloo_and_a_missing_relation_count():
    from pgcn_b200 import rgcn
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        rgcn.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo", relations=2)
    with pytest.raises(ValueError, match="relations"):
        rgcn.run(0, 1, 1, 4, "x.mtx", "x.part", "nccl")
