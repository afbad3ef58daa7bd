"""Attention dropout on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU, for K = 1, 4 and 8 heads:
the edge-dropout launch against torch.nn.functional.dropout on the same [nnz, K] tensor, and the GAT step (forward +
backward; PGATAttention at K = 1, PGATMultiHeadAttention otherwise) at p = 0 and p = 0.6.

    python tools/bench_attention_dropout.py [--iters 30] [--warmup 10] [--config C2] [--heads 1,4,8]

Reports, per K, the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  edge_dropout        pgcn_edge_dropout on alpha [nnz, K], out of place, with its model bytes (8 + 8K per entry:
                      the pair, K values read, K written) per second
  torch_dropout       F.dropout(alpha, 0.6) on the same tensor
  step_p0 / step_p06  the GAT step without dropout and with EdgeDropout(0.6), then step_p0 once more for its spread
and the ratios edge_dropout / torch_dropout and step_p06 / (the smaller step_p0), with the card's name and power limit read in the same
run. Prints one JSON line last.
"""
import argparse
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
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--heads", default="1,4,8")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from pgcn_b200 import graphio, plan as planmod
    from pgcn_b200.op import EdgeDropout, PGATAttention, PGATMultiHeadAttention, _mask
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_dropout.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, _, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    plan = planmod.PgcnPlan(lp, f, device=dev)
    plan.autotune(f)
    plan.bind_values()
    pairs = plan.edge_pairs()
    gen = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *s: torch.rand(s, device=dev, generator=gen) * 2 - 1
    Z, g = rnd(n, f), rnd(n, f)
    res = {}
    for K in [int(x) for x in args.heads.split(",")]:
        r = {}
        alpha = torch.rand((nnz, K), device=dev, generator=gen)
        out = torch.empty_like(alpha)
        drop = EdgeDropout(0.6, 1, dev)
        snap = drop.draw()
        r["edge_dropout"] = median_ms(lambda: _mask(pairs, snap, drop, alpha, out), args.iters, args.warmup)
        r["edge_dropout_GBps"] = (8 + 8 * K) * nnz / (r["edge_dropout"] * 1e-3) / 1e9
        r["torch_dropout"] = median_ms(lambda: F.dropout(alpha, 0.6, training=True), args.iters, args.warmup)
        r["dropout_over_torch"] = r["edge_dropout"] / r["torch_dropout"]
        del alpha, out

        el, er = (rnd(n) if K == 1 else rnd(n, K)), (rnd(n) if K == 1 else rnd(n, K))
        Zp, elp, erp = (x.clone().requires_grad_(True) for x in (Z, el, er))
        fn = PGATAttention if K == 1 else PGATMultiHeadAttention

        def step(d):
            for x in (Zp, elp, erp):
                x.grad = None
            o = fn.apply(plan, Zp, elp, erp, 0.2, d)
            o.backward(g)

        r["step_p0"] = median_ms(lambda: step(None), args.iters, args.warmup)
        d06 = EdgeDropout(0.6, 2, dev)
        r["step_p06"] = median_ms(lambda: step(d06), args.iters, args.warmup)
        r["step_p0_again"] = median_ms(lambda: step(None), args.iters, args.warmup)       # the spread of step_p0
        r["step_p06_over_p0"] = r["step_p06"] / min(r["step_p0"], r["step_p0_again"])
        res["K%d" % K] = r
        del Zp, elp, erp
        torch.cuda.empty_cache()

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "iters": args.iters, "warmup": args.warmup,
              "card": card(), "ms": res}
    for K, r in res.items():
        for k_, v_ in r.items():
            print("%-4s %-22s %.4g" % (K, k_, v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
