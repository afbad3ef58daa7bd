"""CPU-side checks of the max aggregation: the NumPy oracle (sage_oracle) against torch.scatter_reduce("amax") and
numpy.argmax on crafted rows (ties, NaN, +-inf, all -inf, signed zeros, empty rows); the binding of pgcn_forward_max /
pgcn_backward_max and their refusal of null plans; no CPU fallback in op.aggregate_max; PSAGE.py's usage errors and its
refusal of gloo."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import sage_oracle as so
from pgcn_b200 import cabi

NEW = ["pgcn_forward_max", "pgcn_backward_max"]


def random_csr(n, nnz, seed):
    rs = np.random.RandomState(seed)
    A = sp.csr_matrix((np.ones(nnz, np.float32), (rs.randint(0, n, nnz), rs.randint(0, n, nnz))), shape=(n, n))
    A.sum_duplicates()
    A.sort_indices()
    return A


def test_oracle_values_equal_scatter_reduce_amax():
    A = random_csr(300, 3000, 1)
    rs = np.random.RandomState(2)
    X = rs.permutation(300 * 7).reshape(300, 7).astype(np.float32) / 7.0      # distinct values: no ties
    Z, arg = so.max_aggregate(A.indptr, A.indices, X)
    rows = np.repeat(np.arange(300), np.diff(A.indptr))
    idx = torch.from_numpy(rows)[:, None].expand(-1, 7)
    want = torch.zeros((300, 7)).scatter_reduce(0, idx, torch.from_numpy(X[A.indices]), "amax", include_self=False)
    assert np.array_equal(Z, want.numpy())
    deg = np.diff(A.indptr)
    assert np.all(arg[deg == 0] == -1) and np.all(arg[deg > 0] >= 0)
    assert np.array_equal(X[A.indices[arg[deg > 0]], np.arange(7)], Z[deg > 0])


def crafted():
    """One row per case, its entries over consecutive columns of a one-feature X."""
    inf, nan = np.inf, np.nan
    cases = [
        [1.0, 3.0, 3.0, 2.0],                  # tie: the first 3.0
        [2.0, nan, 5.0, nan],                  # NaN above every number: the first NaN
        [nan, nan],
        [-inf, -inf, -inf],                    # all -inf: the first
        [-inf, 1.0, inf, inf],
        [-0.0, 0.0],                           # equal: the first, with its sign
        [0.0, -0.0],
        [-1.0],
        [-2.0, -0.5, -0.5],
    ]
    return cases


def test_oracle_index_is_numpy_argmax_on_crafted_rows():
    for vals in crafted():
        x = np.array(vals, dtype=np.float32)
        rowptr = np.array([0, len(x)])
        colidx = np.arange(len(x))
        Z, arg = so.max_aggregate(rowptr, colidx, x[:, None])
        assert arg[0, 0] == np.argmax(x), vals
        assert Z.view(np.uint32)[0, 0] == x.view(np.uint32)[np.argmax(x)], vals


def test_oracle_signed_zero_and_nan_bits_are_kept():
    x = np.array([-0.0, 0.0], dtype=np.float32)[:, None]
    Z, _ = so.max_aggregate(np.array([0, 2]), np.array([0, 1]), x)
    assert np.signbit(Z[0, 0])
    payload = np.array([0x7fc01234], dtype=np.uint32).view(np.float32)
    x = np.concatenate([np.array([1.0], np.float32), payload, np.array([np.nan], np.float32)])[:, None]
    Z, arg = so.max_aggregate(np.array([0, 3]), np.array([0, 1, 2]), x)
    assert arg[0, 0] == 1 and Z.view(np.uint32)[0, 0] == 0x7fc01234


def test_oracle_empty_rows_give_zero_and_minus_one():
    rowptr = np.array([0, 0, 2, 2, 3])
    colidx = np.array([1, 0, 2])
    X = np.array([[5.0, -1.0], [4.0, 7.0], [-3.0, -3.0]], dtype=np.float32)
    Z, arg = so.max_aggregate(rowptr, colidx, X)
    for i in (0, 2):
        assert np.all(Z[i] == 0) and np.all(arg[i] == -1)
    assert arg[1].tolist() == [1, 0] and Z[1].tolist() == [5.0, 7.0]
    G = so.max_backward(colidx, arg, np.ones((4, 2)), 3)
    assert G.tolist() == [[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]]


def test_oracle_gather_gradient_goes_to_the_first_winner():
    rowptr, colidx = np.array([0, 3]), np.array([0, 1, 2])
    P = torch.tensor([[2.0], [2.0], [1.0]], dtype=torch.float64, requires_grad=True)
    so.max_gather(rowptr, colidx, P).sum().backward()
    assert P.grad[:, 0].tolist() == [1.0, 0.0, 0.0]


def test_binding_declares_the_new_symbols():
    lib = cabi.load()
    for name in NEW:
        assert name in cabi.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None, name


def test_null_plan_is_invalid_not_a_crash():
    lib = cabi.load()
    assert lib.pgcn_forward_max(None, None, None, None, 8, None) == -1
    assert b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_backward_max(None, None, None, None, 8, None) == -1


class _FakePlan:
    m, n, f_max, _bound, layout = 4, 4, 8, True, "local"


def test_aggregate_max_has_no_cpu_fallback():
    from pgcn_b200 import op
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_max(_FakePlan(), torch.zeros((4, 8)))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op.aggregate_max_backward(_FakePlan(), torch.zeros((4, 8), dtype=torch.int32), torch.zeros((4, 8)))


@pytest.mark.parametrize("argv", [
    ["-a", "x.mtx"],                                       # -p/-l/-f missing
    ["--no-such-flag"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "two", "-f", "8"],
    ["-a", "x.mtx", "-p", "x.part", "-b", "nccl", "-s", "1", "-l", "2", "-f", "0"],
])
def test_cli_prints_usage_on_missing_or_bad_flags(argv, capsys):
    from pgcn_b200 import sage
    with pytest.raises(SystemExit) as e:
        sage.main(argv)
    assert e.value.code == 2
    assert "usage: PSAGE.py" in capsys.readouterr().out


def test_cli_refuses_gloo():
    from pgcn_b200 import sage
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sage.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")
