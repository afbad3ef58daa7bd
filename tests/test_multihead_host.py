"""CPU-side checks of multi-head sparse graph attention: the fp64 multi-head reference (pgat_heads_oracle) against
oracle/pgat_oracle.py at heads=1 and against a dense, -inf-masked per-head formulation; the binding of the five new
entry points and their refusal of null plans; PGAT.py's --heads argument errors."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

import pgat_heads_oracle as ho
from helpers import GOLDEN
from oracle import pgat_oracle as po
from pgcn_b200 import cabi

NEW = ["pgcn_edge_softmax_heads", "pgcn_edge_softmax_backward_heads", "pgcn_forward_heads", "pgcn_backward_heads",
       "pgcn_sddmm_heads"]


def karate():
    z = np.load(os.path.join(GOLDEN, "pgat_karate_k1.npz"))
    n = int(z["n"])
    return sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n)), z["H"].astype(np.float64)


def gemat11():
    z = np.load(os.path.join(GOLDEN, "pgat_gemat11_k1.npz"))
    n = int(z["n"])
    return sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n)), z["H"].astype(np.float64)


def test_heads_one_is_the_single_head_oracle():
    A, H = karate()
    f = H.shape[1]
    for a, b in zip(ho.init_params(2, f, 7), po.init_params(2, f, 7)):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    params = po.init_params(2, f, 7)
    assert torch.equal(ho.intended_forward(A, H, params, 0.2), po.intended_forward(A, H, params, 0.2))
    assert ho.intended_training(A, 2, 4, 7, 1.0, epochs=3) == po.intended_training(A, 2, 4, 7, 1.0, epochs=3)


def dense_heads(A, H, params, slope, heads):
    """Every head written densely: non-edges masked with -inf, rows without entries set to 0, heads concatenated."""
    P = sp.csr_matrix(A, copy=True)
    P.data[:] = 1.0
    mask = torch.from_numpy(P.toarray() != 0)
    X = torch.as_tensor(H, dtype=torch.float64)
    for W, a in params:
        W, a = torch.as_tensor(W), torch.as_tensor(a)
        f = W.shape[0]
        d = f // heads
        Z = X @ W.T
        outs = []
        for h in range(heads):
            Zh = Z[:, h * d:(h + 1) * d]
            S = F.leaky_relu(Zh @ a[:d, h:h + 1] + (Zh @ a[d:, h:h + 1]).T, slope)
            S = torch.where(mask, S, torch.full_like(S, -float("inf")))
            outs.append(torch.nan_to_num(torch.softmax(S, 1), nan=0.0) @ Zh)
        X = torch.cat(outs, 1)
    return X


@pytest.mark.parametrize("heads", [2, 4, 8])
@pytest.mark.parametrize("slope", [0.2, 1.0])
def test_multi_head_oracle_matches_a_dense_masked_softmax(heads, slope):
    A, _ = gemat11()
    A = sp.coo_matrix(A)
    keep = A.row != 3                                       # an empty row
    A = sp.csr_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)
    f = 16
    rs = np.random.RandomState(heads)
    H = rs.uniform(-1, 1, size=(A.shape[0], f))
    params = ho.init_params(2, f, 5, heads)
    assert params[0][1].shape == (2 * f // heads, heads)
    got = ho.intended_forward(A, H, params, slope, heads).numpy()
    want = dense_heads(A, H, params, slope, heads).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    assert np.all(got[3] == 0)


def test_binding_declares_the_new_symbols():
    lib = cabi.load()
    for name in NEW:
        assert name in cabi.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None, name


def test_null_plan_is_invalid_not_a_crash():
    lib = cabi.load()
    assert lib.pgcn_edge_softmax_heads(None, 2, None, None, None, 0.2, None, None) == -1
    assert b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_edge_softmax_backward_heads(None, 2, None, None, None, None, None, 0.2, None, None, None) == -1
    assert lib.pgcn_forward_heads(None, 2, None, None, None, None, 8, None) == -1
    assert lib.pgcn_backward_heads(None, 2, None, None, None, 8, None) == -1
    assert lib.pgcn_sddmm_heads(None, 2, None, None, None, None, 8, None) == -1


@pytest.mark.parametrize("argv", [
    ["--heads", "3"],                                      # not 1, 2, 4 or 8
    ["--heads", "16"],
    ["--heads", "x"],
    ["-f", "6", "--heads", "4"],                           # f % heads != 0
])
def test_cli_refuses_bad_heads(argv, capsys):
    from pgcn_b200 import pgat
    base = ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8"]
    with pytest.raises(SystemExit) as e:
        pgat.main(base + argv)
    assert e.value.code == 2
    assert "usage: PGAT.py" in capsys.readouterr().out
