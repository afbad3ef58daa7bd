"""Reader of the CPU path's on-disk formats (SURVEY.md §8f rank 4) against files written by the reference's
own partitioner binary (tests/golden/cpu_path, make_cpu_path_fixtures.py): A.k / H.k / conn.k / buff.k /
config of GCN-HP/main.cpp -> the (A, partvec) inputs of the plan builder."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.io import mmread

from helpers import GOLDEN
from pgcn_b200 import graphio, plan as planmod

CPU = os.path.join(GOLDEN, "cpu_path")


def test_karate_partition_roundtrip_and_connectivity():
    d = os.path.join(CPU, "karate_k3")
    P = graphio.read_cpu_partition(d, 3)
    A0 = sp.csr_matrix(mmread(os.path.join(d, "input.A.mtx")))
    assert P["config"] == {"nlayers": 3, "n": 34, "widths": [4, 4, 2]}
    assert P["A"].shape == (34, 34) and P["A"].nnz == A0.nnz
    # A.k values are printed with %.2f (GCN-HP/main.cpp:242): equal to the input within 0.005
    assert abs(sp.csr_matrix(P["A"]) - A0).max() <= 0.005 + 1e-9
    pv = P["partvec"]
    assert set(pv) == {0, 1, 2}
    for r in range(3):
        lp = planmod.build_local_plan(P["A"], pv, r, 3)
        # symmetric pattern: the reference's conn lists == the send lists the plan builder derives
        send = lp.send_map()
        conn = P["conn"][r]
        assert sorted(t for t in conn) == sorted(t for t in send if len(send[t]))
        for tgt, ids in conn.items():
            assert np.array_equal(np.sort(ids), send[tgt])
        bs, br = P["buff"][r]
        assert bs == {t: len(v) for t, v in send.items() if len(v)}
        assert br == {s: len(v) for s, v in lp.recv_map().items() if len(v)}
        # the local block of the plan is exactly what A.r holds
        n, i, j, v = graphio.read_cpu_matrix_part(os.path.join(d, "A.%d" % r))
        assert lp.nnz() == len(i) and np.array_equal(np.unique(i), lp.owned[np.diff(lp.rowptr) > 0])


def test_unsymmetric_input_exposes_transposed_connectivity():
    """GCN-HP/main.cpp:154-170 lists, for part k, its vertices that have an OUT-entry into another part; row-wise
    aggregation needs the vertices other parts' rows REFERENCE. They differ on an unsymmetric pattern: the reader
    reports the reference's lists, the plan is built from A itself."""
    d = os.path.join(CPU, "unsym_k4_rp")
    P = graphio.read_cpu_partition(d, 4)
    A, pv = P["A"].tocoo(), P["partvec"]
    differs = False
    for r in range(4):
        lp = planmod.build_local_plan(A, pv, r, 4)
        for tgt in range(4):
            if tgt == r:
                continue
            out_entries = np.unique(A.row[(pv[A.row] == r) & (pv[A.col] == tgt)])      # the reference's rule
            ref_ids = np.sort(P["conn"][r].get(tgt, np.zeros(0, dtype=np.int64)))
            assert np.array_equal(ref_ids, out_entries)
            if not np.array_equal(ref_ids, lp.send_map()[tgt]):
                differs = True
        # the plan built from A is right: product check against the dense truth
        H = np.arange(A.shape[0] * 2, dtype=np.float64).reshape(-1, 2)
        Aloc = sp.csr_matrix((lp.vals.astype(np.float64), lp.colidx, lp.rowptr), shape=(lp.m, lp.m + lp.h))
        np.testing.assert_allclose(Aloc @ H[np.concatenate([lp.owned, lp.halo])], (sp.csr_matrix(A) @ H)[lp.owned], rtol=1e-6)
    assert differs


def test_malformed_files_are_rejected(tmp_path):
    (tmp_path / "H.0").write_text("3\n0\n1\n")
    with pytest.raises(ValueError):
        graphio.read_cpu_rows_part(str(tmp_path / "H.0"))
    (tmp_path / "A.0").write_text("4 2\n0 1 0.5\n")
    with pytest.raises(ValueError):
        graphio.read_cpu_matrix_part(str(tmp_path / "A.0"))
