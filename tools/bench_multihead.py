"""Multi-head sparse graph attention on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU, for
K = 1, 4 and 8 heads: what each multi-head entry point costs, the PGATMultiHeadAttention step, the same heads run as K
single-head PGATAttention layers on d = f / K slices (the per-head loop), and a PyTorch-native multi-head step.

    python tools/bench_multihead.py [--iters 30] [--warmup 10] [--config C2] [--heads 1,4,8]

Reports, per K, the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  edge_softmax_heads / edge_softmax_backward_heads / forward_heads / backward_heads / sddmm_heads   one entry point
  step_multihead      PGATMultiHeadAttention forward + backward (gradients of Z, el and er)
  step_loop           K PGATAttention forward + backward steps on the d-wide slices with their own el / er
  step_torch_native   the multi-head step in PyTorch ops (gather, scatter_reduce amax, index_add_) on the same CSR
plus spmm_ring_fwd (pgcn_spmm at f, the ring kernel) next to forward_heads (the register kernel), whether the multi-head
and loop outputs and gradients agree within the fp32 bound, and the card's name and power limit read in the same run.
Prints one JSON line last.
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
    ap.add_argument("--no-torch", action="store_true", help="skip the PyTorch-native step")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from pgcn_b200 import cabi, graphio, plan as planmod
    from pgcn_b200.op import PGATAttention, PGATMultiHeadAttention
    if not torch.cuda.is_available():
        raise SystemExit("bench_multihead.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, _, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    plan = planmod.PgcnPlan(lp, f, device=dev)
    plan.autotune(f)
    plan.bind_values()
    lib = cabi.load()
    st = lambda: torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *s: torch.rand(s, device=dev, generator=gen) * 2 - 1
    Z, g = rnd(n, f), rnd(n, f)
    out = torch.empty((n, f), device=dev)
    G = torch.empty((n, f), device=dev)
    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    res = {}
    res["spmm_ring_fwd"] = median_ms(lambda: cabi.check(lib.pgcn_spmm(plan.handle, 0, Z.data_ptr(), None, out.data_ptr(),
                                                                      None, f, st()), plan.handle),
                                     args.iters, args.warmup)
    for K in [int(x) for x in args.heads.split(",")]:
        d = f // K
        r = {}
        el, er = rnd(n, K), rnd(n, K)
        alpha, dalpha, dpre = torch.empty((nnz, K), device=dev), rnd(nnz, K), torch.empty((nnz, K), device=dev)
        d_el = torch.empty((n, K), device=dev)
        call = lambda rc: cabi.check(rc, plan.handle)
        r["edge_softmax_heads"] = median_ms(lambda: call(lib.pgcn_edge_softmax_heads(
            plan.handle, K, el.data_ptr(), er.data_ptr(), None, 0.2, alpha.data_ptr(), st())), args.iters, args.warmup)
        r["edge_softmax_backward_heads"] = median_ms(lambda: call(lib.pgcn_edge_softmax_backward_heads(
            plan.handle, K, el.data_ptr(), er.data_ptr(), None, alpha.data_ptr(), dalpha.data_ptr(), 0.2,
            dpre.data_ptr(), d_el.data_ptr(), st())), args.iters, args.warmup)
        r["forward_heads"] = median_ms(lambda: call(lib.pgcn_forward_heads(
            plan.handle, K, alpha.data_ptr(), Z.data_ptr(), out.data_ptr(), None, f, st())), args.iters, args.warmup)
        r["backward_heads"] = median_ms(lambda: call(lib.pgcn_backward_heads(
            plan.handle, K, alpha.data_ptr(), g.data_ptr(), G.data_ptr(), f, st())), args.iters, args.warmup)
        r["sddmm_heads"] = median_ms(lambda: call(lib.pgcn_sddmm_heads(
            plan.handle, K, g.data_ptr(), Z.data_ptr(), None, dalpha.data_ptr(), f, st())), args.iters, args.warmup)

        Zp, elp, erp = (x.clone().requires_grad_(True) for x in (Z, el, er))

        def step_multihead():
            for x in (Zp, elp, erp):
                x.grad = None
            o = PGATMultiHeadAttention.apply(plan, Zp, elp, erp, 0.2)
            o.backward(g)
            return o

        Zs = [Z[:, h * d:(h + 1) * d].contiguous().requires_grad_(True) for h in range(K)]
        els = [el[:, h].contiguous().requires_grad_(True) for h in range(K)]
        ers = [er[:, h].contiguous().requires_grad_(True) for h in range(K)]
        gs = [g[:, h * d:(h + 1) * d].contiguous() for h in range(K)]

        def step_loop():
            outs = []
            for h in range(K):
                for x in (Zs[h], els[h], ers[h]):
                    x.grad = None
                o = PGATAttention.apply(plan, Zs[h], els[h], ers[h], 0.2)
                o.backward(gs[h])
                outs.append(o)
            return outs

        def step_torch_native():
            for x in (Zp, elp, erp):
                x.grad = None
            s = F.leaky_relu(elp[rows] + erp[cols], 0.2)                                   # [nnz, K]
            mx = torch.full((n, K), -float("inf"), device=dev).scatter_reduce(
                0, rows[:, None].expand(-1, K), s, "amax", include_self=True)
            ex = torch.exp(s - mx[rows].detach())
            den = torch.zeros((n, K), device=dev).index_add_(0, rows, ex)
            a = ex / den[rows]
            msg = (a[:, :, None] * Zp[cols].view(-1, K, d)).view(-1, f)
            o = torch.zeros((n, f), device=dev).index_add_(0, rows, msg)
            o.backward(g)

        r["step_multihead"] = median_ms(step_multihead, args.iters, args.warmup)
        r["step_loop"] = median_ms(step_loop, args.iters, args.warmup)
        r["loop_over_multihead"] = r["step_loop"] / r["step_multihead"]
        if not args.no_torch:
            try:
                r["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
                r["torch_native_over_multihead"] = r["step_torch_native"] / r["step_multihead"]
            except RuntimeError as e:                  # report, do not hide
                r["step_torch_native"] = None
                r["step_torch_native_error"] = str(e)[:200]
                torch.cuda.empty_cache()

        # multi-head against the loop: same math, other summation orders -> an fp32 bound, not bits
        o = step_multihead()
        lo = step_loop()
        torch.cuda.synchronize()
        pairs = [(o, torch.cat(lo, 1)), (Zp.grad, torch.cat([x.grad for x in Zs], 1)),
                 (elp.grad, torch.stack([x.grad for x in els], 1)), (erp.grad, torch.stack([x.grad for x in ers], 1))]
        r["max_rel_diff_vs_loop"] = max(float((a - b).abs().max().detach() / (b.abs().max().detach() + 1e-30))
                                        for a, b in pairs)
        r["agrees_with_loop"] = r["max_rel_diff_vs_loop"] <= 1e-4
        res["K%d" % K] = r

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "max_row": int(deg.max()), "iters": args.iters,
              "warmup": args.warmup, "card": card(), "ms": res}
    print("%-28s %s" % ("spmm_ring_fwd", "%.4f" % res["spmm_ring_fwd"]))
    for K, r in res.items():
        if not isinstance(r, dict):
            continue
        for k_, v_ in r.items():
            print("%-4s %-28s %s" % (K, k_, ("%.4g" % v_) if isinstance(v_, float) else v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
