"""R-GCN's relational aggregation on C2 (R-MAT 1 M vertices / 16 M edges + self loops), one GPU: what the two
relational walks cost at f = 64 and 128 and R = 2, 4 and 8, and the aggregation step against the two ways of getting
there without them.

    python tools/bench_rgcn.py [--iters 20] [--warmup 5] [--config C2] [--widths 64,128] [--relations 2,4,8]

The relations are rgcn.relation_hash of every entry's global (row, column); the weights are aggr="mean"'s 1 / c.
Reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward       pgcn_rgcn_forward, pgcn_rgcn_backward
  step_rgcn                op.aggregate_rgcn + op.aggregate_rgcn_backward (allocations included)
  step_spmm_weighted       R x op.PSpMMWeighted on the one plan, values w * (rel == r), forward and autograd backward
  step_torch_native        w * X[col] index_add_ into [m R, f] at i R + rel, autograd backward to X
and the achieved rates of the byte models (model bytes over time):
  forward   per entry 4f + 12 B (X[j] gathered; its column, its forward entry and its weight); per virtual row 4f B
            (Z written)
  backward  per transposed entry 4f + 12 B (gZ[i R + rel] gathered; the index, the permutation, the weight); per
            column 4f B (dX written)
The native step and the masked-SpMM step give Z and dX too; their largest differences from the kernels' are reported.
Prints the card's name and power limit read in the same run, then one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_edge_values import card, median_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--widths", default="64,128")
    ap.add_argument("--relations", default="2,4,8")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    from pgcn_b200.rgcn import relation_hash
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgcn.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = graphio.CONFIGS[args.config][0]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    widths = [int(x) for x in args.widths.split(",")]
    rels = [int(x) for x in args.relations.split(",")]
    plan = planmod.PgcnPlan(lp, max(widths), device=dev)
    plan.bind_values()
    perm_t = plan.transposed_entries()
    pairs = plan.edge_pairs()
    lib = cabi.load_rgcn()
    st = lambda: torch.cuda.current_stream().cuda_stream
    chk = cabi.check_rgcn
    out = {"config": args.config, "n": n, "nnz": nnz, "iters": args.iters, "warmup": args.warmup, "card": card(),
           "runs": []}
    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), np.diff(lp.rowptr.astype(np.int64)))).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)

    for R in rels:
        rel = relation_hash(pairs, R)
        walks = plan.relation_walks(rel, R)
        w = op.rgcn_weights(plan, walks, None, "mean")
        masked = [w * (rel == r) for r in range(R)]
        for f in widths:
            gen = torch.Generator(device=dev).manual_seed(f + R)
            X = torch.randn((n, f), device=dev, generator=gen)
            gZ = torch.randn((n, R, f), device=dev, generator=gen)
            Z, dX = torch.empty((n, R, f), device=dev), torch.empty((n, f), device=dev)
            w1 = torch.empty((walks.fwd.nslots, f), device=dev)
            w2 = torch.empty((walks.tr.nslots, f), device=dev)
            run = {"R": R, "f": f, "virtual_rows": n * R,
                   "empty_virtual_rows": int((torch.bincount(rows * R + rel, minlength=n * R) == 0).sum()),
                   "split_virtual_rows": int(walks.fwd.c.nsplits), "split_cols": int(walks.tr.c.nsplits)}
            calls = {"forward": lambda: chk(lib.pgcn_rgcn_forward(
                         C.byref(walks.fwd.c), walks.perm_f.data_ptr(), n, 0, R, X.data_ptr(), None, w.data_ptr(),
                         Z.data_ptr(), w1.data_ptr(), f, st())),
                     "backward": lambda: chk(lib.pgcn_rgcn_backward(
                         C.byref(walks.tr.c), perm_t.data_ptr(), n, 0, R, gZ.data_ptr(), w.data_ptr(), dX.data_ptr(),
                         w2.data_ptr(), f, st()))}
            ms = {name: median_ms(fn, args.iters, args.warmup) for name, fn in calls.items()}
            for fn in calls.values():
                fn()
            torch.cuda.synchronize()

            def step_rgcn():
                Zo, _ = op.aggregate_rgcn(plan, walks, X, w)
                return Zo, op.aggregate_rgcn_backward(plan, walks, gZ, w)
            ms["step_rgcn"] = median_ms(step_rgcn, args.iters, args.warmup)

            Xl = X.clone().requires_grad_(True)

            def step_spmm_weighted():
                Xl.grad = None
                Zs = torch.stack([op.PSpMMWeighted.apply(plan, masked[r], Xl) for r in range(R)], 1)
                Zs.backward(gZ)
                return Zs
            ms["step_spmm_weighted"] = median_ms(step_spmm_weighted, args.iters, args.warmup)
            Zs = step_spmm_weighted().detach()
            diff = {"spmm_weighted_Z_max_abs_diff": float((Zs - Z).abs().max()),
                    "spmm_weighted_dX_max_abs_diff": float((Xl.grad - dX).abs().max())}
            del Zs
            Xl.grad = None
            plan.use_values(None)

            v = rows * R + rel
            try:
                def step_torch_native():
                    Xl.grad = None
                    Zn = torch.zeros((n * R, f), device=dev).index_add_(0, v, w[:, None] * Xl[cols])
                    Zn.backward(gZ.reshape(n * R, f))
                    return Zn
                ms["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
                Zn = step_torch_native().detach().reshape(n, R, f)
                diff.update({"torch_native_Z_max_abs_diff": float((Zn - Z).abs().max()),
                             "torch_native_dX_max_abs_diff": float((Xl.grad - dX).abs().max())})
                del Zn
            except RuntimeError as err:                    # report, do not hide
                run["torch_native_error"] = str(err)[:200]
            del Xl, v
            bytes_ = {"forward": nnz * (4 * f + 12) + n * R * 4 * f, "backward": nnz * (4 * f + 12) + n * 4 * f}
            run.update({"ms": ms, "bytes": bytes_, "check": diff,
                        "tbps": {k + "_tbps": b / ms[k] / 1e9 for k, b in bytes_.items()},
                        "spmm_weighted_over_rgcn": ms["step_spmm_weighted"] / ms["step_rgcn"]})
            if "step_torch_native" in ms:
                run["torch_native_over_rgcn"] = ms["step_torch_native"] / ms["step_rgcn"]
            out["runs"].append(run)
            del X, gZ, Z, dX, w1, w2
            torch.cuda.empty_cache()
        del masked

    for run in out["runs"]:
        head = "R=%d f=%-4d" % (run["R"], run["f"])
        for k_, v_ in list(run["ms"].items()) + list(run["tbps"].items()):
            print("%s %-24s %.4g" % (head, k_, v_))
        for k_ in ("spmm_weighted_over_rgcn", "torch_native_over_rgcn"):
            if k_ in run:
                print("%s %-24s %.3g" % (head, k_, run[k_]))
        print("%s %s" % (head, run["check"]))
    print("card: %s, power limit %s W" % (out["card"]["name"], out["card"]["power_limit_w"]))
    print(json.dumps(out))
    plan.close()


if __name__ == "__main__":
    main()
