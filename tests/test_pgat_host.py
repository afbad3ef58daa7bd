"""CPU-side checks of sparse graph attention: the fp64 oracle against the unmodified reference (tests/golden/pgat_*.npz,
make_pgat_golden.py) in its `literal` mode and against a dense -inf-masked formulation in its `intended` mode; the
binding of the new entry points (pgcn_edge_softmax, pgcn_edge_softmax_backward, pgcn_halo_rows) and their refusal of
null plans; the PGAT command line's usage errors and its refusal of gloo."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from helpers import GOLDEN
from oracle import pgat_oracle as po
from pgcn_b200 import cabi

NEW = ["pgcn_edge_softmax", "pgcn_edge_softmax_backward", "pgcn_halo_rows"]


def golden(case):
    z = np.load(os.path.join(GOLDEN, "pgat_%s.npz" % case))
    n = int(z["n"])
    A = sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n))
    return z, A, z["partvec"].astype(np.int64), int(z["k"]), int(z["f"]), int(z["seed"])


@pytest.mark.parametrize("case", ["karate_k1", "karate_k3", "gemat11_k1"])
@pytest.mark.parametrize("nlayers", [1, 2])
def test_literal_oracle_matches_the_reference(case, nlayers):
    z, A, pv, k, f, seed = golden(case)
    params = po.init_params(nlayers, f, seed + nlayers)
    H = z["H"].astype(np.float64)
    labels = np.arange(A.shape[0]) % f
    for r in range(k):
        logits, loss, grads = po.literal_rank_grads(A, pv, r, H, params, labels)
        ref = z["r%d_L%d_logits" % (r, nlayers)]
        np.testing.assert_allclose(logits, ref, rtol=2e-5, atol=2e-5 * np.abs(ref).max(),
                                   err_msg="%s L=%d rank %d logits" % (case, nlayers, r))
        assert abs(loss - float(z["r%d_L%d_loss" % (r, nlayers)])) <= 1e-5 * max(1.0, abs(loss))
        for i, (dW, da) in enumerate(grads):
            for got, key in ((dW, "dW"), (da, "da")):
                want = z["r%d_L%d_%s%d" % (r, nlayers, key, i)]
                np.testing.assert_allclose(got, want, rtol=1e-3, atol=1e-4 * (np.abs(want).max() + 1e-30),
                                           err_msg="%s L=%d rank %d layer %d %s" % (case, nlayers, r, i, key))


def dense_intended(A, H, params, slope):
    """The intended layer written densely: non-edges masked with -inf, rows without entries set to 0. The mask is the
    stored pattern (gemat11 stores entries whose value is 0)."""
    P = sp.csr_matrix(A, copy=True)
    P.data[:] = 1.0
    mask = torch.from_numpy(P.toarray() != 0)
    X = torch.as_tensor(H, dtype=torch.float64)
    for W, a in params:
        W, a = torch.as_tensor(W), torch.as_tensor(a)
        f = W.shape[0]
        Z = X @ W.T
        S = F.leaky_relu(Z @ a[:f] + (Z @ a[f:]).T, slope)
        S = torch.where(mask, S, torch.full_like(S, -float("inf")))
        P = torch.nan_to_num(torch.softmax(S, 1), nan=0.0)
        X = P @ Z
    return X


@pytest.mark.parametrize("case", ["karate_k1", "gemat11_k1"])
@pytest.mark.parametrize("slope", [0.2, 1.0])
def test_intended_oracle_matches_a_dense_masked_softmax(case, slope):
    z, A, pv, k, f, seed = golden(case)
    A = sp.coo_matrix(A)
    keep = A.row != 3                                       # an empty row
    A = sp.csr_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)
    params = po.init_params(2, f, seed)
    H = z["H"].astype(np.float64)
    got = po.intended_forward(A, H, params, slope).numpy()
    want = dense_intended(A, H, params, slope).numpy()
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
    assert lib.pgcn_edge_softmax(None, None, None, None, 0.2, None, None) == -1
    assert b"null" in lib.pgcn_last_error(None)
    assert lib.pgcn_edge_softmax_backward(None, None, None, None, None, None, 0.2, None, None, None) == -1
    assert lib.pgcn_halo_rows(None, None, None, 4, None) == -1


def test_cli_usage_and_backend_errors():
    from pgcn_b200 import pgat
    with pytest.raises(SystemExit):
        pgat.main(["-a", "x.mtx"])                         # -p/-l/-f missing
    with pytest.raises(SystemExit):
        pgat.main(["--no-such-flag"])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pgat.run(0, 1, 1, 4, "x.mtx", "x.part", "gloo")    # gloo/CPU is refused, loudly
