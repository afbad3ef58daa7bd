"""CPU-side checks of GATv2 attention: the fp64 reference (gatv2_oracle) against a dense, masked torch float64 GATv2
with autograd, forward and all three gradients; the binding of the two entry points against the header and their
refusal of null plans; PGAT.py --v2's argument errors."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

import gatv2_oracle as go
from conftest import ROOT
from helpers import GOLDEN
from pgcn_b200 import cabi

NEW = ["pgcn_forward_gatv2", "pgcn_backward_gatv2"]


def graph(name):
    z = np.load(os.path.join(GOLDEN, "pgat_%s_k1.npz" % name))
    n = int(z["n"])
    A = sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n))
    if name == "gemat11":                                   # an empty row
        keep = A.row != 3
        A = sp.coo_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)
    A = sp.csr_matrix(A)
    A.sum_duplicates()
    return A.tocoo()


def dense_gatv2(A, xl, xr, att, slope):
    """GATv2 written densely: the score of every (i, j) pair, non-edges masked with -inf, rows without entries 0."""
    n = A.shape[0]
    K, d = att.shape
    mask = torch.from_numpy(A.toarray() != 0)
    outs = []
    for h in range(K):
        sl = slice(h * d, (h + 1) * d)
        T = xl[None, :, sl] + xr[:, None, sl]                               # [i, j, d]
        S = (F.leaky_relu(T, slope) * att[h]).sum(2)
        S = torch.where(mask, S, torch.full_like(S, -float("inf")))
        outs.append(torch.nan_to_num(torch.softmax(S, 1), nan=0.0) @ xl[:, sl])
    return torch.cat(outs, 1)


@pytest.mark.parametrize("name", ["karate", "gemat11"])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("slope", [0.2, 1.0])
def test_oracle_matches_a_dense_masked_gatv2(name, K, slope):
    A = graph(name)
    n, f = A.shape[0], 16
    if name == "gemat11":
        keep = np.unique(np.concatenate([np.arange(300), A.row[:2000]]))   # dense [n, n, d] stays small
        A = sp.coo_matrix(sp.csr_matrix(A)[keep][:, keep])
        n = A.shape[0]
    rs = np.random.RandomState(K + int(10 * slope))
    xl, xr, gZ = (rs.uniform(-1, 1, (n, f)) for _ in range(3))
    att = rs.standard_normal((K, f // K))
    rows, cols = A.row.astype(np.int64), A.col.astype(np.int64)
    Z, alpha, _ = go.forward(rows, cols, n, xl, xr, att, slope)
    dxl, dxr, datt, _, _ = go.backward(rows, cols, n, xl, xr, att, slope, alpha, gZ)
    tl, tr, ta = (torch.tensor(x, requires_grad=True) for x in (xl, xr, att))
    want = dense_gatv2(A, tl, tr, ta, slope)
    (want * torch.from_numpy(gZ)).sum().backward()
    for got, ref, what in ((Z, want.detach(), "Z"), (dxl, tl.grad, "dxl"), (dxr, tr.grad, "dxr"),
                           (datt, ta.grad, "datt")):
        ref = ref.numpy()
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * (np.abs(ref).max() + 1), err_msg=what)
    deg = np.bincount(rows, minlength=n)
    assert np.all(Z[deg == 0] == 0)
    tw = go.forward_torch(torch.from_numpy(rows), torch.from_numpy(cols), n, torch.tensor(xl), torch.tensor(xr),
                          torch.tensor(att), slope)
    np.testing.assert_allclose(tw.numpy(), Z, rtol=1e-12, atol=1e-14)


def test_binding_declares_the_new_symbols_with_the_header_argument_counts():
    header = open(os.path.join(ROOT, "include", "pgcn_b200.h")).read()
    lib = cabi.load()
    for name in NEW:
        assert name in cabi.SYMBOLS
        m = re.search(r"int %s\(([^;]*)\);" % name, header)
        assert m, name
        nargs = len(m.group(1).split(","))
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == nargs, name


def test_null_plan_is_invalid_not_a_crash():
    lib = cabi.load()
    assert lib.pgcn_forward_gatv2(None, 2, None, None, None, 0.2, None, None, None, 8, None) == -1
    assert b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_backward_gatv2(None, 2, None, None, None, None, None, None, 0.2, None, None, None, None, 8,
                                   None) == -1


@pytest.mark.parametrize("argv", [
    ["--v2", "--heads", "3"],                              # not 1, 2, 4 or 8
    ["--v2", "--heads", "16"],
    ["--v2", "--heads", "x"],
    ["--v2", "-f", "6", "--heads", "4"],                   # f % heads != 0
])
def test_cli_v2_refuses_bad_heads(argv, capsys):
    from pgcn_b200 import pgat
    base = ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "8"]
    with pytest.raises(SystemExit) as e:
        pgat.main(base + argv)
    assert e.value.code == 2
    assert "usage: PGAT.py" in capsys.readouterr().out
