"""The real transports of the halo exchange on >= 2 GPUs of one box: NCCL grouped send/recv
(all-to-all-v) and the peer-memory path (rows stored straight into the neighbour's slab over
NVLink). One process per GPU, as in the reference (GPU/PGCN.py:280-283).

Checks, per rank: PSpMM forward/backward == fp64 truth within the fp32 bound, == the golden
reference outputs (gemat11, k = 2), both transports give identical bits, overlap on/off agree,
and the host stats equal the reference's counters."""
import os

import numpy as np
import pytest
import torch

from harness import spawn_ranks
from helpers import Golden, fp32_tol
from oracle import pgcn_oracle as orc

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _worker(rank, k, port, case, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    from pgcn_b200 import graphio, plan as planmod
    from pgcn_b200.op import PSpMM
    if case == "rmat":
        n, f = 20000, 128
        A = graphio.synthetic_graph(n, 400000, seed=4)
        pv = graphio.random_partvec(n, k, seed=9)
        rs = np.random.RandomState(3)
        H = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
        G = rs.uniform(-1, 1, size=(n, f)).astype(np.float32)
        gold = None
    else:
        gold = Golden(case)
        A, pv, H, G, f, n = gold.A, gold.partvec, gold.H, gold.G, gold.f, gold.n
    p = planmod.build_plan(A, pv, rank, k, f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    own = p.lp.owned
    res = {}
    for overlap in (1, 0):
        p.set_option("overlap", overlap)
        Hd = torch.from_numpy(H[own]).cuda().requires_grad_(True)
        Z = PSpMM.apply(p, Hd)
        Z.backward(torch.from_numpy(G[own]).cuda())
        torch.cuda.synchronize()
        res[overlap] = (Z.detach().cpu().numpy(), Hd.grad.cpu().numpy())
    # repeated calls (epoch parity of the peer-memory slabs, stale-data hazards)
    for _ in range(5):
        Z = PSpMM.apply(p, Hd.detach())
    torch.cuda.synchronize()
    assert np.array_equal(Z.cpu().numpy(), res[0][0])
    Z64 = orc.truth_forward(A, H)[own]; G64 = orc.truth_backward(A, G)[own]
    tz = fp32_tol(A, H, int(orc.row_degree(A).max()))[own]
    tg = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))[own]
    for overlap in (1, 0):
        z, g = res[overlap]
        assert (np.abs(z - Z64) <= tz).all(), "forward beyond fp32 bound (overlap=%d)" % overlap
        assert (np.abs(g - G64) <= tg).all(), "backward beyond fp32 bound (overlap=%d)" % overlap
    if gold is not None:
        np.testing.assert_allclose(res[1][0], gold.get(rank, "Z1_own"), rtol=2e-5, atol=2e-6 * max(1.0, np.abs(Z64).max()))
        if k <= 2:     # Q3 cannot bite with two ranks: the reference gradient is right
            np.testing.assert_allclose(res[1][1], gold.get(rank, "Hgrad_own"), rtol=2e-5, atol=2e-6 * max(1.0, np.abs(G64).max()))
    # a width the peer-store kernels do not take (f % 4 != 0) goes through the NCCL fallback
    st0 = dict(p.stats)
    Hodd = torch.from_numpy(np.ascontiguousarray(H[own][:, :6])).cuda().requires_grad_(True)
    Zodd = PSpMM.apply(p, Hodd)
    Zodd.backward(torch.from_numpy(np.ascontiguousarray(G[own][:, :6])).cuda())
    torch.cuda.synchronize()
    Z64o = orc.truth_forward(A, H[:, :6])[own]; G64o = orc.truth_backward(A, G[:, :6])[own]
    assert (np.abs(Zodd.detach().cpu().numpy() - Z64o) <= fp32_tol(A, H[:, :6], int(orc.row_degree(A).max()))[own]).all()
    assert (np.abs(Hodd.grad.cpu().numpy() - G64o) <= fp32_tol(A.T, G[:, :6], int(orc.row_degree(A.T).max()))[own]).all()
    p.stats.update(st0)
    # stats as the reference counts them: rows, messages incl. empty ones; 2 fwd+bwd pairs + 5 fwd
    st = p.stats
    assert st["send_nmsg"] == (2 * 2 + 5) * (k - 1)
    assert st["send_volume"] == (2 + 5) * p.lp.S + 2 * p.lp.h
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, res[1][0], res[1][1]


def _need(k):
    if not torch.cuda.is_available() or torch.cuda.device_count() < k:
        pytest.skip("needs %d GPUs" % k)


@pytest.mark.parametrize("case", ["gemat11_k2", "rmat"])
def test_two_gpus_nccl_and_p2p_agree(case):
    _need(2)
    a = spawn_ranks(_worker, 2, (29801, case, "nccl"))
    b = spawn_ranks(_worker, 2, (29802, case, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        assert np.array_equal(a[r][1], b[r][1]) and np.array_equal(a[r][2], b[r][2])


@pytest.mark.parametrize("k", [3, 4, 8])
def test_more_gpus(k):
    _need(k)
    case = "gemat11_k3_hp" if k == 3 else "rmat"
    a = spawn_ranks(_worker, k, (29810 + k, case, "nccl"))
    b = spawn_ranks(_worker, k, (29830 + k, case, "auto"))
    for r in range(k):
        assert np.array_equal(a[r][1], b[r][1]) and np.array_equal(a[r][2], b[r][2])
