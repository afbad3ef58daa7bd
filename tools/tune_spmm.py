#!/usr/bin/env python
"""Sweep the SpMM scheduling options on a benchmark config and print one JSON line per point
(development tool; results are summarised under profiles/).

    python tools/tune_spmm.py --config C2 --sweep default
    python tools/tune_spmm.py --config C2 --single edges_per_block=256,tile_floats=0 --iters 5   (for ncu)
    python tools/tune_spmm.py --gather-sweep        (L2 capacity / bandwidth probe with windowed columns)
    python tools/tune_spmm.py --gather-sweep --mixed   (0-40 % of the columns from a 512 MB window, the rest from 16 MB)
    python tools/tune_spmm.py --gather-sweep --all-hit --iters 20   (the ring's own cost per copy; see the option's help)
    python tools/tune_spmm.py --config C2 --sweep slices   (ring row tile: full width vs 64-float slices)
"""
import argparse
import itertools
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, iters, warm=3):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--f", type=int, default=0)
    ap.add_argument("--sweep", default="")
    ap.add_argument("--single", default="")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--baselines", action="store_true")
    ap.add_argument("--gather-sweep", action="store_true")
    ap.add_argument("--mixed", action="store_true", help="with --gather-sweep: mix a 512 MB and a 16 MB window of columns")
    ap.add_argument("--all-hit", action="store_true", help="with --gather-sweep: only the 16 MB window, full width and 64-float "
                    "slices at 16 and 32 slots")
    ap.add_argument("--transpose", action="store_true")
    ap.add_argument("--cache", default="/tmp/pgcn_b200_cache")
    ap.add_argument("--out", default="")
    ap.add_argument("--hot-sweep", default="", help="comma list of hot-set sizes in MB (rebuilds the plan each time)")
    args = ap.parse_args()

    import torch
    import scipy.sparse as sp
    from pgcn_b200 import cabi, graphio, plan as planmod
    dev = torch.device("cuda", 0)
    lib = cabi.load()
    stream = torch.cuda.current_stream().cuda_stream
    peak = 6567.4
    try:
        peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    outf = open(args.out, "a") if args.out else None

    def emit(rec):
        s = json.dumps(rec)
        print(s, flush=True)
        if outf:
            outf.write(s + "\n"); outf.flush()

    if args.gather_sweep and args.mixed:
        # a fraction of the columns uniform over a 512 MB window (1 M rows: they miss L2), the rest over a 16 MB window
        # (32 K rows: they hit); the plan marks the wide-window columns cold. Shows what a given share of L2-missing
        # gathers costs the ring at each row tile and ring depth (DESIGN §6, cold look-ahead).
        n, d, f, hot_rows = 1_000_000, 16, 128, 32_000
        rng = np.random.default_rng(0)
        for frac in (0.0, 0.1, 0.2, 0.4):
            wide = rng.random(n * d) < frac
            col = np.where(wide, rng.integers(0, n, size=n * d), rng.integers(0, hot_rows, size=n * d))
            row = np.repeat(np.arange(n, dtype=np.int64), d)
            A = sp.coo_matrix((np.ones(n * d, dtype=np.float32), (row, col)), shape=(n, n))
            p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev)
            H = torch.rand((n, f), device=dev); Z = torch.empty((n, f), device=dev)
            for tile, slots in itertools.product((0, 64), (16, 32)):
                p.set_option("ring_tile_floats", tile)
                p.set_option("ring_slots", slots)
                med, mn = timed(lambda: cabi.check(lib.pgcn_spmm(p.handle, 0, H.data_ptr(), None, Z.data_ptr(), None, f, stream), p.handle), args.iters, warm=20)
                emit({"probe": "gather-mixed", "wide_frac": frac, "ring_tile_floats": tile, "ring_slots": slots, "ms": med,
                      "gather_GBs": p.lp.nnz() * f * 4 / med / 1e6})
            p.close()
        return

    if args.gather_sweep and args.all_hit:
        # every gathered row hits L2 (16 MB window), so the time is what the ring itself pays per copied byte. Run it
        # on the probe builds as well (PGCN_B200_VARIANT=<name> PGCN_B200_DEFS=-DPGCN_RING_DIAG=1 / 2 / 3: no slot
        # reads or FFMA / no row copies or waits / neither) to split copy rate, shared-memory reads and bookkeeping.
        n, d, f, W = 1_000_000, 16, 128, 32_000
        rng = np.random.default_rng(0)
        col = rng.integers(0, W, size=n * d, dtype=np.int64)
        row = np.repeat(np.arange(n, dtype=np.int64), d)
        A = sp.coo_matrix((np.ones(n * d, dtype=np.float32), (row, col)), shape=(n, n))
        p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev)
        H = torch.rand((n, f), device=dev); Z = torch.empty((n, f), device=dev)
        nnz = p.lp.nnz()
        for tile, slots in itertools.product((128, 64), (16, 32)):
            p.set_option("ring_tile_floats", tile)
            p.set_option("ring_slots", slots)
            med, mn = timed(lambda: cabi.check(lib.pgcn_spmm(p.handle, 0, H.data_ptr(), None, Z.data_ptr(), None, f, stream), p.handle),
                            args.iters, warm=20)
            emit({"probe": "gather-all-hit", "lib": os.path.basename(cabi.lib_path()), "window_MB": W * f * 4 / 1e6,
                  "ring_tile_floats": tile, "ring_slots": slots, "ms": med, "gather_GBs": nnz * f * 4 / med / 1e6,
                  "copies_per_us": nnz * (f // tile) / med / 1e3})
        p.close()
        return

    if args.gather_sweep:
        # n rows, degree d, columns uniform in a window of W rows: working set W*f*4 bytes
        n, d, f = 1_000_000, 16, 128
        rng = np.random.default_rng(0)
        windows = (32_000, 1_000_000) if args.iters <= 3 else (32_000, 64_000, 96_000, 128_000, 192_000, 256_000, 384_000, 512_000, 1_000_000)
        for W in windows:
            col = rng.integers(0, W, size=n * d, dtype=np.int64)
            row = np.repeat(np.arange(n, dtype=np.int64), d)
            A = sp.coo_matrix((np.ones(n * d, dtype=np.float32), (row, col)), shape=(n, n))
            p = planmod.build_plan(A, np.zeros(n, dtype=np.int64), 0, 1, f, device=dev)
            H = torch.rand((n, f), device=dev); Z = torch.empty((n, f), device=dev)
            for tile in (0, 64):                 # ring row tile: full width, 64-float slices
                p.set_option("ring_tile_floats", tile)
                med, mn = timed(lambda: cabi.check(lib.pgcn_spmm(p.handle, 0, H.data_ptr(), None, Z.data_ptr(), None, f, stream), p.handle), args.iters)
                nnz = p.lp.nnz()
                emit({"probe": "gather", "window_rows": W, "window_MB": W * f * 4 / 1e6, "ring_tile_floats": tile, "ms": med,
                      "gather_GBs": nnz * f * 4 / med / 1e6, "edges_per_s": nnz / med * 1e3})
            p.close()
        return

    n, nnz, f, _, _ = graphio.CONFIGS[args.config]
    if args.f:
        f = args.f
    t0 = time.time()
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    p = planmod.PgcnPlan(lp, f, device=dev)
    emit({"info": "plan", "config": args.config, "n": n, "nnz": lp.nnz(), "f": f, "build_s": time.time() - t0,
          "max_degree": int(np.diff(lp.rowptr).max())})
    gen = torch.Generator(device=dev).manual_seed(1)
    H = torch.rand((n, f), device=dev, generator=gen) * 2 - 1
    Z = torch.empty((n, f), device=dev)
    ab = p.algorithmic_bytes(f)
    alg = ab["spmm_bwd"] if args.transpose else ab["spmm_fwd"]

    def run():
        nonlocal p
        if args.transpose:
            cabi.check(lib.pgcn_spmm(p.handle, 1, H.data_ptr(), None, Z.data_ptr(), None, f, stream), p.handle)
        else:
            cabi.check(lib.pgcn_spmm(p.handle, 0, H.data_ptr(), None, Z.data_ptr(), None, f, stream), p.handle)

    def point(opts):
        nonlocal p
        for k_, v in opts.items():
            p.set_option(k_, v)
        med, mn = timed(run, args.iters)
        emit(dict(opts, ms=med, ms_min=mn, edges_per_s=lp.nnz() / med * 1e3, alg_GBs=alg / med / 1e6,
                  frac=alg / med / 1e6 / peak, gather_GBs=ab["gather_fwd"] / med / 1e6))

    if args.hot_sweep:
        for hot in [int(x) for x in args.hot_sweep.split(",")]:
            os.environ["PGCN_HOT_MB"] = str(hot)
            p.close()
            p = planmod.PgcnPlan(lp, f, device=dev)
            for epb in (128, 192):
                point({"edges_per_block": epb, "hot_mb_env": hot} if False else {"edges_per_block": epb})
                print(json.dumps({"hot_mb": hot}), flush=True)
    elif args.single:
        opts = {kv.split("=")[0]: int(kv.split("=")[1]) for kv in args.single.split(",") if kv}
        point(opts)
    elif args.sweep == "default":
        for epb, tile in itertools.product((64, 128, 256, 512), (0, 64, 32, 16)):
            point({"edges_per_block": epb, "tile_floats": tile})
    elif args.sweep == "depth":
        for epb in (96, 112, 120, 128, 136, 144, 152, 160, 192):
            point({"edges_per_block": epb})
    elif args.sweep == "epb":
        for epb, lr in itertools.product((64, 96, 128, 160, 192, 256, 384), (0, 100000)):
            point({"edges_per_block": epb, "tile_floats": 0, "long_row": lr})
    elif args.sweep == "ring":
        # register pipeline (kernel 4) vs the shared-memory ring filled by 1-D TMA bulk copies (5) / cp.async (6) /
        # 2-D tensor-map TMA (7); ring shapes: 16 slots (2 groups of 8), 32 (2 x 16), 64 (2 x 32 or 4 x 16)
        point({"kernel": 4})
        for kern, (slots, groups), epb in itertools.product((7, 5), ((16, 2), (32, 2), (64, 2), (64, 4)), (256, 512, 1024)):
            if kern == 5 and slots == 64:
                continue
            point({"kernel": kern, "ring_slots": slots, "ring_groups": groups, "ring_edges_per_block": epb, "persistent": 1})
        point({"kernel": 7, "ring_slots": 32, "ring_groups": 2, "ring_edges_per_block": 512, "persistent": 0})
        point({"kernel": 6, "ring_slots": 16, "ring_groups": 2, "ring_edges_per_block": 512, "persistent": 1})
    elif args.sweep == "slices":
        for tile, slots, epb in itertools.product((0, 64), (16, 32, 64), (256, 512, 1024)):
            point({"ring_tile_floats": tile, "ring_slots": slots, "ring_edges_per_block": epb})
    elif args.sweep == "ring-small":
        point({"kernel": 4})
        for kern, slots, epb, pers in ((5, 32, 1024, 0), (5, 16, 1024, 0), (5, 32, 2048, 1), (6, 32, 1024, 0), (6, 16, 1024, 0)):
            point({"kernel": kern, "ring_slots": slots, "ring_edges_per_block": epb, "persistent": pers})
    elif args.sweep == "mini":
        for epb in (128, 160):
            point({"edges_per_block": epb, "tile_floats": 0})
    elif args.sweep == "small":
        for epb in (96, 128, 192, 256):
            point({"edges_per_block": epb, "tile_floats": 0})
    elif args.sweep == "fine":
        for epb, tile, lr in itertools.product((96, 128, 192, 256, 384), (0, 64, 32), (0, 256, 1024, 4096)):
            point({"edges_per_block": epb, "tile_floats": tile, "long_row": lr})

    if args.baselines:
        # the library path the reference would take on this box (GPU/PGCN.py:127): uncoalesced COO, and CSR
        idx = torch.from_numpy(np.vstack([A.row, A.col]).astype(np.int64)).to(dev)
        val = torch.from_numpy(A.data.astype(np.float32)).to(dev)
        coo = torch.sparse_coo_tensor(idx, val, (n, n))
        med, _ = timed(lambda: torch.sparse.mm(coo, H), max(3, args.iters // 2), warm=1)
        emit({"baseline": "torch.sparse.mm COO uncoalesced (reference's call)", "ms": med, "edges_per_s": lp.nnz() / med * 1e3})
        csr = coo.coalesce().to_sparse_csr()
        med, _ = timed(lambda: torch.sparse.mm(csr, H), args.iters, warm=2)
        emit({"baseline": "torch.sparse.mm CSR prebuilt (cuSPARSE)", "ms": med, "edges_per_s": lp.nnz() / med * 1e3})
        med, _ = timed(lambda: Z.copy_(H), args.iters)
        emit({"baseline": "copy H->Z (2 x %d MB)" % (n * f * 4 // 1000000), "ms": med, "GBs": 2 * n * f * 4 / med / 1e6})
    p.close()


if __name__ == "__main__":
    main()
