"""CPU-side checks of edge dropout: the NumPy Philox4x32-10 against the Random123 known answers, the threshold and scale
of the mask rule, include/pgcn_dropout.h against its binding and libpgcn_dropout.so (exports, sm_90a, kernel manifest),
the refusals of the C entry point (bad arguments, no GPU), the fp64 references at p = 0 against the attention oracles
without dropout, and PGAT.py's --attn-dropout argument errors."""
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
import pgat_heads_oracle as ho
from conftest import ROOT
from helpers import GOLDEN
from pgcn_b200 import build, cabi, op

MANIFEST = os.path.join(ROOT, "tests", "dropout_kernel_instances.txt")


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = do.philox4x32_10(np.array([ctr], dtype=np.uint64), key)
    assert tuple(int(w) for w in got[0]) == want


@pytest.mark.parametrize("p,T,scale", [
    (0.0, 0, 1.0),
    (0.5, 2 ** 31, 2.0),
    (0.6, 2576980377, float(np.float32(2.5))),
    (1 - 2.0 ** -20, 2 ** 32 - 2 ** 12, 2.0 ** 20),
])
def test_threshold_and_scale(p, T, scale):
    assert op.dropout_constants(p) == (T, scale)
    assert do.constants(p) == (T, np.float32(scale))


@pytest.mark.parametrize("p", [-0.1, 1.0, 1.5, float("nan")])
def test_probability_outside_0_1_is_refused(p):
    with pytest.raises(ValueError):
        op.dropout_constants(p)


def test_mask_keeps_one_minus_p_and_scales_exactly():
    rs = np.random.RandomState(0)
    gi, gj = rs.randint(0, 2 ** 31 - 1, 200000), rs.randint(0, 2 ** 31 - 1, 200000)
    x = rs.uniform(-1, 1, (200000, 4)).astype(np.float32)
    y = do.apply(x, gi, gj, 0.6, 12345, 1)
    kept = y != 0
    assert abs(kept.mean() - 0.4) < 5 * np.sqrt(0.24 / kept.size)
    assert np.array_equal(y[kept], x[kept] * np.float32(2.5))
    # NaN stays NaN, dropped or kept; the same (row, column) gives the same bits
    z = do.apply(np.full((4, 1), np.nan, np.float32), gi[:4], gj[:4], 0.6, 12345, 1)
    assert np.isnan(z).all()
    assert np.array_equal(do.apply(x[:1].repeat(3, 0), gi[[7] * 3], gj[[7] * 3], 0.6, 12345, 1),
                          do.apply(x[:1], gi[[7]], gj[[7]], 0.6, 12345, 1).repeat(3, 0))


def header_functions():
    txt = open(os.path.join(ROOT, "include", "pgcn_dropout.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {name: [a for a in args.split(",") if a.strip() not in ("", "void")]
            for name, args in re.findall(r"\b(pgcn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_header_and_binding_agree():
    fns = header_functions()
    assert sorted(fns) == sorted(cabi.DROPOUT_SYMBOLS)
    lib = cabi.load_dropout()
    for name, args in fns.items():
        assert len(getattr(lib, name).argtypes) == len(args), name
    assert "pgcn_edge_dropout" not in cabi.SYMBOLS


def test_library_exports_every_symbol_and_names_sm_90a():
    lib = cabi.load_dropout()
    for name in cabi.DROPOUT_SYMBOLS:
        assert hasattr(lib, name), "libpgcn_dropout.so does not export " + name
    assert b"sm_90a" in lib.pgcn_dropout_version()
    assert os.path.basename(cabi.dropout_lib_path()) == "libpgcn_dropout.so"


def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import list_kernels
    if list_kernels.cuda_tool("cuobjdump") is None or list_kernels.cuda_tool("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not available")
    return list_kernels


def test_built_for_sm_90a():
    lk = _tools()
    cabi.load_dropout()
    out = subprocess.run([lk.cuda_tool("cuobjdump"), "-lelf", cabi.dropout_lib_path()], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out


def test_kernels_equal_the_manifest():
    lk = _tools()
    cabi.load_dropout()
    with open(MANIFEST) as fh:
        want = [ln.strip() for ln in fh if ln.strip()]
    assert lk.list_kernels(lib=cabi.dropout_lib_path()) == want


def test_each_library_has_its_own_dependencies():
    assert not set(build.DEPS) & set(build.DROPOUT_DEPS) - {os.path.abspath(build.__file__)}
    assert os.path.join(build.CSRC, "philox.cuh") in build.DROPOUT_DEPS


def test_bad_arguments_are_refused_before_any_device_work():
    lib = cabi.load_dropout()
    buf = (C.c_int64 * 4)()
    p = C.cast(buf, C.c_void_p)
    assert lib.pgcn_edge_dropout(None, 4, 2, 0, 1.0, p, p, p, None) == -1
    assert b"null" in lib.pgcn_dropout_last_error()
    assert lib.pgcn_edge_dropout(p, 4, 3, 0, 1.0, p, p, p, None) == -1
    assert b"heads" in lib.pgcn_dropout_last_error()
    assert lib.pgcn_edge_dropout(p, -1, 2, 0, 1.0, p, p, p, None) == -1
    assert lib.pgcn_edge_dropout(p, 4, 2, 0, float("inf"), p, p, p, None) == -1


def test_no_gpu_returns_minus_4():
    # no device visible to the child process, whatever this machine has
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import pgcn_b200; from pgcn_b200 import cabi\n"
            "lib = cabi.load_dropout(build_if_missing=False)\n"
            "b = (C.c_int64 * 4)(); p = C.cast(b, C.c_void_p)\n"
            "rc = lib.pgcn_edge_dropout(p, 1, 1, 0, 1.0, p, p, p, None)\n"
            "print(rc, lib.pgcn_dropout_last_error().decode())\n" % ROOT)
    cabi.load_dropout()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    rc, msg = out.stdout.split(" ", 1)
    assert int(rc) == -4 and "no CUDA device" in msg


def karate():
    z = np.load(os.path.join(GOLDEN, "pgat_karate_k1.npz"))
    n = int(z["n"])
    return sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n)), z["H"].astype(np.float64)


@pytest.mark.parametrize("heads", [1, 4])
def test_oracle_at_p_0_is_the_attention_oracle(heads):
    A, H = karate()
    f = 8
    rs = np.random.RandomState(heads)
    H = rs.uniform(-1, 1, size=(A.shape[0], f))
    params = ho.init_params(2, f, 3, heads)
    got = do.intended_forward(A, H, params, 0.2, 0.0, 3, 1, heads)
    want = ho.intended_forward(A, H, params, 0.2, heads)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-13, atol=1e-13 * float(want.abs().max()))
    assert np.allclose(do.intended_training(A, 2, 4, 7, 1.0, 0.0, epochs=3, heads=heads),
                       ho.intended_training(A, 2, 4, 7, 1.0, epochs=3, heads=heads), rtol=1e-13)


def test_oracle_dropout_changes_the_curve_and_each_epoch_draws_anew():
    A, _ = karate()
    a = do.intended_training(A, 2, 4, 7, 1.0, 0.5, epochs=4)
    b = do.intended_training(A, 2, 4, 7, 1.0, 0.0, epochs=4)
    assert a[0] != b[0]
    C = sp.coo_matrix(A)
    assert not np.array_equal(do.keep(C.row, C.col, 1, 0.5, 7 * 2 ** 16, 1), do.keep(C.row, C.col, 1, 0.5, 7 * 2 ** 16, 2))
    assert not np.array_equal(do.keep(C.row, C.col, 1, 0.5, 7 * 2 ** 16, 1),
                              do.keep(C.row, C.col, 1, 0.5, 7 * 2 ** 16 + 1, 1))


def test_cli_dropout_key_depends_on_seed_and_layer_only():
    from pgcn_b200 import pgat
    assert pgat.dropout_key(None, 0) == 0 and pgat.dropout_key(7, 1) == 7 * 2 ** 16 + 1
    state = torch.get_rng_state()
    assert pgat.dropout_key(3, 2) == 3 * 2 ** 16 + 2
    assert torch.equal(state, torch.get_rng_state())


@pytest.mark.parametrize("argv", [
    ["--attn-dropout", "1"],
    ["--attn-dropout", "1.5"],
    ["--attn-dropout", "-0.1"],
    ["--attn-dropout", "nan"],
    ["--attn-dropout", "0.5", "--v2"],
    ["--v2", "--attn-dropout", "0"],
])
def test_cli_refuses_bad_attn_dropout(argv, capsys):
    from pgcn_b200 import pgat
    base = ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8"]
    with pytest.raises(SystemExit) as e:
        pgat.main(base + argv)
    assert e.value.code == 2
    assert "usage: PGAT.py" in capsys.readouterr().out
