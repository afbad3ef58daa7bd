"""The ring SpMM walked in 64-float slices (ring_tile_floats = 64: 256-byte row slots, the slices gathered one after
the other) against the full-width ring: the same products summed in the same order, so forward and backward
outputs are bit-identical at equal block size, and within the fp32 bound of the fp64 truth."""
import numpy as np
import pytest
import torch

from helpers import assert_close_fp32, fp32_tol
from oracle import pgcn_oracle as orc
from pgcn_b200 import graphio
from test_gpu_parity import backward_all, build_plans, forward_all, skewed_graph

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("f", [128, 256, 384, 512])
@pytest.mark.parametrize("opts", [
    dict(kernel=7), dict(kernel=7, ring_slots=16, ring_edges_per_block=90, persistent=0),
    dict(kernel=7, ring_slots=32, ring_edges_per_block=200), dict(kernel=7, ring_slots=64, ring_edges_per_block=300),
    dict(kernel=7, ring_slots=64, ring_groups=4, ring_edges_per_block=64, ring_long_row=100),
    dict(kernel=5, ring_slots=32, ring_edges_per_block=100, ring_long_row=150), dict(kernel=5, persistent=0),
    dict(kernel=6),
])
def test_sliced_ring_matches_truth_and_full_width(f, opts):
    """Head and tail blocks inside a piece, hub rows split into segments (small blocks), persistent and one-shot
    CTAs, 1-D and 2-D TMA fills, 2-rank plans with a halo slab, forward and transposed."""
    n = 4000
    A = skewed_graph(n, 120000, seed=11)
    rng = np.random.RandomState(f)
    H = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    Z64 = orc.truth_forward(A, H); G64 = orc.truth_backward(A, G)
    tolZ = fp32_tol(A, H, int(orc.row_degree(A).max())); tolG = fp32_tol(A.T, G, int(orc.row_degree(A.T).max()))
    for k in (1, 2):
        pv = np.zeros(n, dtype=np.int64) if k == 1 else graphio.random_partvec(n, 2, seed=5)
        plans = build_plans(A, pv, k, f)
        zs = forward_all(plans, H, ring_tile_floats=64, **opts)
        gs = backward_all(plans, G)
        zs2 = forward_all(plans, H)
        zf = forward_all(plans, H, ring_tile_floats=0)
        gf = backward_all(plans, G)
        for r, p in enumerate(plans):
            own = p.lp.owned
            assert torch.equal(zs[r], zs2[r])
            assert_close_fp32(zs[r].cpu().numpy(), Z64[own], tolZ[own], "sliced fwd %s f=%d k=%d r%d" % (opts, f, k, r))
            assert_close_fp32(gs[r].cpu().numpy(), G64[own], tolG[own], "sliced bwd %s f=%d k=%d r%d" % (opts, f, k, r))
            assert torch.equal(zs[r], zf[r]), "sliced != full-width fwd %s f=%d k=%d r%d" % (opts, f, k, r)
            assert torch.equal(gs[r], gf[r]), "sliced != full-width bwd %s f=%d k=%d r%d" % (opts, f, k, r)
            if k == 1 and opts.get("ring_edges_per_block", 1024) <= 100:
                assert p.get_option("ring_long_rows_fwd") > 0
            p.close()


def test_tile_option_and_autotune():
    n, f = 6000, 256
    A = skewed_graph(n, 150000, seed=13)
    H = np.random.RandomState(4).uniform(-1, 1, size=(n, f)).astype(np.float32)
    p = build_plans(A, np.zeros(n, dtype=np.int64), 1, f)[0]
    assert p.get_option("ring_tile_floats") == 0
    with pytest.raises(RuntimeError):
        p.set_option("ring_tile_floats", 96)
    p.set_option("ring_tile_floats", 64)
    assert p.get_option("ring_tile_floats") == 64
    p.set_option("ring_tile_floats", 0)
    p.autotune(f)                                # picks full width (0) or 64-float slices per matrix
    assert p.get_option("ring_tile_floats") in (0, 64)
    z = forward_all([p], H)[0]
    assert_close_fp32(z.cpu().numpy(), orc.truth_forward(A, H), fp32_tol(A, H, int(orc.row_degree(A).max())), "autotuned")
    p.close()
