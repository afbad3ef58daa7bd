"""CLI-level parity (SURVEY.md §4 (3)): the PGCN.py clone prints the reference's stdout fields, the
same exchange statistics, and — with seeded weights — the same loss curve as the unmodified
reference run under gloo (tests/golden/gemat11_e2e.json written by make_golden.py)."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from harness import TIMEOUT, spawn_ranks
from helpers import GOLDEN, Golden


def _write_inputs(tmp_path, case):
    from scipy.io import mmwrite
    from pgcn_b200 import graphio
    g = Golden(case)
    a = str(tmp_path / "gemat11.mtx")
    mmwrite(a, g.A, precision=17)
    p = str(tmp_path / ("gemat11.mtx.%d.hp" % g.k))
    graphio.write_partvec(p, g.partvec)
    return a, p, g


def test_cli_usage_and_backend_errors():
    from pgcn_b200 import pgcn
    with pytest.raises(SystemExit):
        pgcn.main(["-a", "x.mtx"])                         # -p/-l/-f missing
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pgcn.run(0, 1, 2, 16, "x.mtx", "x.part", "gloo")   # gloo/CPU is refused, loudly


@pytest.mark.gpu
def test_cli_single_rank_matches_reference_losses(tmp_path):
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    a, p, g = _write_inputs(tmp_path, "gemat11_k1")
    env = dict(os.environ, SLURM_NPROCS="1", SLURM_PROCID="0", MASTER_ADDR="127.0.0.1", MASTER_PORT="29650")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "PGCN.py"), "-a", a, "-p", p, "-b", "nccl", "-s", "1",
                          "-l", "2", "-f", "16", "--seed", "1000"], env=env, capture_output=True, text=True,
                         timeout=TIMEOUT)
    assert out.returncode == 0, out.stderr[-2000:]
    ref = json.load(open(os.path.join(GOLDEN, "gemat11_e2e.json")))["k1"]
    losses = [float(l.split("Loss")[1]) for l in out.stdout.splitlines() if l.startswith("Epoch")]
    assert [l[:11] for l in out.stdout.splitlines() if l.startswith("Epoch")] == ["Epoch %05d" % i for i in range(4)]
    np.testing.assert_allclose(losses, ref["losses"], rtol=2e-4)
    assert "Elapsed time" in out.stdout
    assert "total_vol: %d total_nmsg: %d" % (ref["total_vol"], ref["total_nmsg"]) in out.stdout
    assert "'send_volume': 0" in out.stdout


def _mg_worker(rank, k, port, a, p):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(k))
    from pgcn_b200 import pgcn
    buf = io.StringIO()
    res = pgcn.init_process(rank, k, pgcn.run, 2, 16, a, p, "nccl", ref_quirks=True, seed=1000 + rank, out=buf)
    return res, buf.getvalue()


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("k", [2, 3])
def test_cli_multi_rank_matches_reference(tmp_path, k):
    """k = 2: Q3 cannot bite, Q1 is emulated by --ref-quirks, Q2 (stale scratch) perturbs the reference's
    own curve by ~1e-4 relative -> losses agree to 1e-3; volumes and message counts agree exactly.
    k = 3: statistics exact; the loss is compared loosely (Q3 makes the reference's gradients wrong)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < k:
        pytest.skip("needs %d GPUs" % k)
    a, p, g = _write_inputs(tmp_path, "gemat11_k2" if k == 2 else "gemat11_k3_hp")
    res = spawn_ranks(_mg_worker, k, (29660 + k, a, p))
    ref = json.load(open(os.path.join(GOLDEN, "gemat11_e2e.json")))["k%d" % k]
    out0, text0 = res[0]
    assert out0["total_vol"] == ref["total_vol"] and out0["total_nmsg"] == ref["total_nmsg"]
    assert "total_vol: %d total_nmsg: %d" % (ref["total_vol"], ref["total_nmsg"]) in text0
    np.testing.assert_allclose(out0["losses"], ref["losses"], rtol=1e-3 if k == 2 else 5e-2)


@pytest.mark.gpu
def test_minibatch_driver_matches_reference_losses(tmp_path):
    """SURVEY.md §8f rank 3: the mini-batch trainer (one plan per pre-sampled batch, swapped per step) against the
    loss curve of the UNMODIFIED GPU/PGCN-Mini-batch.py run() on karate (tests/golden/make_minibatch_e2e_golden.py:
    one rank, 3 layers, f = 4, batch_size = 12, seeded weights) — same sampling sequence, same per-batch
    sub-matrices, same loss bookkeeping (epoch sums start at 1)."""
    import io
    import pickle
    import shutil
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device")
    from pgcn_b200 import minibatch
    ref = json.load(open(os.path.join(GOLDEN, "karate_minibatch_e2e.json")))
    z = np.load(os.path.join(GOLDEN, "karate_minibatch.npz"))
    import scipy.sparse as sp
    from scipy.io import mmwrite
    n = int(z["n"])
    A = sp.coo_matrix((z["val"], (z["row"], z["col"])), shape=(n, n))
    a = str(tmp_path / "karate.mtx")
    mmwrite(a, A)
    pv = str(tmp_path / "pv1.pkl")
    pickle.dump([0] * n, open(pv, "wb"))
    buf = io.StringIO()
    res = minibatch.run(0, 1, ref["layers"], ref["f"], a, pv, "nccl", ref["batch_size"], out=buf, seed=ref["seed"])
    assert res["nbatches"] == (n // ref["batch_size"] + 1) * 3
    np.testing.assert_allclose(res["losses"], ref["losses"], rtol=5e-4)
    text = buf.getvalue()
    assert "Epoch 00003 | Loss" in text and "total_vol: 0 total_nmsg: 0" in text
    with pytest.raises(RuntimeError):
        minibatch.run(0, 1, 3, 4, a, pv, "gloo", 12)
