"""harness.spawn_ranks on the CPU, with workers that only return, raise or sleep: results come back by rank, a rank's
error and a missed deadline fail the test, and no worker outlives the call on any of these paths."""
import multiprocessing
import os
import time

import pytest

from harness import spawn_ranks


def _work(rank, k, d, what):
    with open(os.path.join(d, "pid.%d" % rank), "w") as fh:
        fh.write(str(os.getpid()))
    if what == "raise" and rank == 1:
        t0 = time.monotonic()
        while not os.path.exists(os.path.join(d, "pid.0")) and time.monotonic() - t0 < 60:
            time.sleep(0.05)
        raise ValueError("rank one gives up")
    if (what == "raise" and rank == 0) or (what == "sleep" and rank == 1):
        time.sleep(3600)
    return 10 * rank


def assert_no_worker_left(d, k):
    assert multiprocessing.active_children() == []
    for r in range(k):
        with open(os.path.join(d, "pid.%d" % r)) as fh:
            pid = int(fh.read())
        with pytest.raises(ProcessLookupError):
            os.kill(pid, 0)


def test_results_come_back_by_rank(tmp_path):
    assert spawn_ranks(_work, 3, (str(tmp_path), "return"), timeout=120) == {0: 0, 1: 10, 2: 20}
    assert_no_worker_left(str(tmp_path), 3)


def test_a_failing_rank_fails_the_test_and_its_sleeping_peer_is_killed(tmp_path):
    with pytest.raises(pytest.fail.Exception, match="(?s)rank 1 failed.*rank one gives up"):
        spawn_ranks(_work, 2, (str(tmp_path), "raise"), timeout=120)
    assert_no_worker_left(str(tmp_path), 2)


def test_a_rank_past_its_deadline_fails_the_test_and_is_killed(tmp_path):
    t0 = time.monotonic()
    with pytest.raises(pytest.fail.Exception, match=r"ranks \[1\] gave no result within 20 s"):
        spawn_ranks(_work, 2, (str(tmp_path), "sleep"), timeout=20)
    assert time.monotonic() - t0 < 60
    assert_no_worker_left(str(tmp_path), 2)
