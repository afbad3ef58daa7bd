#!/usr/bin/env python
"""Offline (CPU) comparison of part vectors for a benchmark config: what the 1-D row partition of GPU/PGCN.py:37-64 would
exchange and how the SpMM work is balanced, per method (hp / gp shipped under bench_data/, rp = uniform random seed 1,
block = contiguous ranges). One markdown row per (method, k): halo rows in (max / mean per rank), stored entries (max /
mean per rank), total halo rows, and the two bounds they imply per layer at f floats per row:
   t_xchg >= 4 f max_in / 450 GB/s (H100 NVLink 4 per direction, data sheet)     t_spmm ~ max entries / single-GPU rate.

    python tools/partition_table.py --config C5 --k 8 [--methods hp gp rp block]
"""
import argparse, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def metrics(A, pv, k):
    prow, pcol = pv[A.row], pv[A.col]
    ent = np.bincount(prow, minlength=k)
    cross = prow != pcol
    keys = np.unique(prow[cross].astype(np.int64) * A.shape[0] + A.col[cross])          # (receiver, column) pairs
    halo_in = np.bincount(keys // A.shape[0], minlength=k)
    return ent, halo_in


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--k", type=int, nargs="+", default=[8])
    ap.add_argument("--methods", nargs="+", default=["hp", "gp", "rp", "block"])
    ap.add_argument("--cache", default="/tmp/pgcn_b200_cache")
    args = ap.parse_args()
    from pgcn_b200 import graphio
    n, nnz, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache).tocoo()
    print("| config | k | method | halo rows in: max / mean per rank | entries: max / mean per rank | total halo rows | exchange bound (ms) |")
    print("|---|---|---|---|---|---|---|")
    for k in args.k:
        for m in args.methods:
            if m in ("hp", "gp"):
                path = os.path.join(ROOT, "bench_data", "%s.%d.%s.npz" % (args.config, k, m))
                if not os.path.exists(path):
                    continue
                pv = np.load(path)["partvec"].astype(np.int64)
            elif m == "rp":
                pv = graphio.random_partvec(n, k, seed=1)
            else:
                pv = graphio.block_partvec(n, k)
            ent, hin = metrics(A, pv, k)
            print("| %s | %d | %s | %d / %d | %d / %d | %d | %.2f |" % (
                args.config, k, m, hin.max(), hin.mean(), ent.max(), ent.mean(), hin.sum(), 4 * f * hin.max() / 770e9 * 1e3), flush=True)


if __name__ == "__main__":
    main()
