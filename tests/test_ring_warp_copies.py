"""The tensor-map ring issues each group's row copies once per warp, from warp-uniform operands. Only how a copy is
issued changed, not which rows land where or the order of the sums, so every row tile width and ring depth must give
the same bits as the per-lane 1-D bulk copies (kernel 5, unchanged) and as the full-width ring, forward and
transposed, on one rank and on two (halo slab)."""
import numpy as np
import pytest
import torch

from pgcn_b200 import graphio
from test_gpu_parity import backward_all, build_plans, forward_all, skewed_graph

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("f", [128, 256])
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("sched", [
    dict(ring_edges_per_block=512),
    # blocks that start and end mid-piece and mid-group, long rows split into segments
    dict(ring_edges_per_block=90, ring_long_row=100),
    dict(ring_edges_per_block=200, persistent=0),
])
def test_warp_copies_match_lane_copies_and_full_width(f, k, sched):
    n = 4000
    A = skewed_graph(n, 120000, seed=23)
    rng = np.random.RandomState(f + k)
    H = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    G = rng.uniform(-1, 1, size=(n, f)).astype(np.float32)
    pv = np.zeros(n, dtype=np.int64) if k == 1 else graphio.random_partvec(n, 2, seed=7)
    plans = build_plans(A, pv, k, f)
    # kernel 5 (1-D bulk, one copy per lane) has the 16- and 32-slot rings; kernel 7 also has the two 64-slot rings
    ref = {}
    for tile in (64, 128):
        for slots in (16, 32):
            zl = forward_all(plans, H, kernel=5, ring_tile_floats=tile, ring_slots=slots, **sched)
            gl = backward_all(plans, G)
            ref[tile, slots] = (zl, gl)
    zfull = forward_all(plans, H, kernel=7, ring_tile_floats=0, ring_slots=16, **sched)
    gfull = backward_all(plans, G)
    if k == 1 and sched["ring_edges_per_block"] <= 100:
        assert plans[0].get_option("ring_long_rows_fwd") > 0
    for tile in (64, 128) + ((256,) if f == 256 else ()):
        for slots, groups in ((16, 2), (32, 2), (64, 2), (64, 4)):
            zw = forward_all(plans, H, kernel=7, ring_tile_floats=tile, ring_slots=slots, ring_groups=groups, **sched)
            gw = backward_all(plans, G)
            what = "tile=%d slots=%dx%d f=%d k=%d %s" % (tile, slots, groups, f, k, sched)
            for r in range(k):
                assert torch.equal(zw[r], zfull[r]), "fwd != full width: " + what
                assert torch.equal(gw[r], gfull[r]), "bwd != full width: " + what
                if (tile, slots) in ref:
                    assert torch.equal(zw[r], ref[tile, slots][0][r]), "fwd != per-lane copies: " + what
                    assert torch.equal(gw[r], ref[tile, slots][1][r]), "bwd != per-lane copies: " + what
    for p in plans:
        p.close()
