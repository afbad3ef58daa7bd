"""world_size = 2 and 3 gloo processes on CPU: the host-side logic of the N > 1 path.

Each rank builds ITS plan independently from the same (A, partvec) — as the reference does
(GPU/PGCN.py:171-176) — and the test checks, with real inter-process messages, the one invariant the
wire format relies on: what rank r packs for p in send order is exactly what p expects at its halo
positions (GPU/PGCN.py:47-48), in both directions, plus count symmetry and the stat counters."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

from harness import spawn_ranks
from helpers import Golden


def _worker(rank, k, port, case):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=k)
    from pgcn_b200 import plan as planmod
    g = Golden(case)
    lp = planmod.build_local_plan(g.A, g.partvec, rank, k)
    # counts: my send count to p == p's recv count from me
    mine = torch.tensor([lp.send_off[p + 1] - lp.send_off[p] for p in range(k)] +
                        [lp.recv_off[p + 1] - lp.recv_off[p] for p in range(k)])
    allc = [torch.zeros_like(mine) for _ in range(k)]
    dist.all_gather(allc, mine)
    for p in range(k):
        assert int(allc[p][k + rank]) == int(mine[p]), "recv count of peer != my send count"
        assert int(allc[p][rank]) == int(mine[k + p])
    # forward wire: pack rows of a tagged H (row i carries its global id) and ship them
    H_own = torch.from_numpy(lp.owned.astype(np.float32)).reshape(-1, 1).repeat(1, 3)
    slab = H_own[torch.from_numpy(lp.send_idx.astype(np.int64))]
    halo = torch.zeros((lp.h, 3))
    reqs = []
    for p in range(k):
        if p == rank:
            continue
        s = slab[lp.send_off[p]:lp.send_off[p + 1]].contiguous()
        r = halo[lp.recv_off[p]:lp.recv_off[p + 1]]
        if s.shape[0]:
            reqs.append(dist.isend(s, p))
        if r.shape[0]:
            buf = torch.zeros_like(r)
            dist.recv(buf, p)
            halo[lp.recv_off[p]:lp.recv_off[p + 1]] = buf
    for r_ in reqs:
        r_.wait()
    assert np.array_equal(halo[:, 0].numpy().astype(np.int64), lp.halo), "halo rows arrive in receiver order"
    # reverse wire: halo partials go home and land on send_idx positions
    back = torch.from_numpy(lp.halo.astype(np.float32)).reshape(-1, 1)
    got = torch.zeros((lp.S, 1))
    reqs = []
    for p in range(k):
        if p == rank:
            continue
        s = back[lp.recv_off[p]:lp.recv_off[p + 1]].contiguous()
        if s.shape[0]:
            reqs.append(dist.isend(s, p))
        if lp.send_off[p + 1] > lp.send_off[p]:
            buf = torch.zeros((lp.send_off[p + 1] - lp.send_off[p], 1))
            dist.recv(buf, p)
            got[lp.send_off[p]:lp.send_off[p + 1]] = buf
    for r_ in reqs:
        r_.wait()
    assert np.array_equal(got[:, 0].numpy().astype(np.int64), lp.send_gid)
    send_ref, recv_ref = g.maps(rank)
    for p in send_ref:
        assert np.array_equal(lp.send_map()[p], send_ref[p]) and np.array_equal(lp.recv_map()[p], recv_ref[p])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("k,case,port", [(2, "gemat11_k2", 29901), (3, "gemat11_k3_hp", 29902), (3, "karate_k3_stchp", 29903)])
def test_wire_order_invariant_over_gloo(k, case, port):
    spawn_ranks(_worker, k, (port, case))
