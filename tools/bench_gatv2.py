"""GATv2 attention on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU: what pgcn_forward_gatv2 and
pgcn_backward_gatv2 cost, each new kernel alone, the operator's step next to the PGATMultiHeadAttention step at the same
K, and a PyTorch-native GATv2 step.

    python tools/bench_gatv2.py [--heads 1 4 8] [--iters 20] [--warmup 5] [--config C2]

Per K it reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward              the two entry points
  sddmm_heads                     pgcn_sddmm_heads at the same K (the score kernel gathers the same rows)
  step_gatv2 / step_gat           PGATv2Attention / PGATMultiHeadAttention forward + backward (inputs given, no linear)
and, from one torch.profiler run of forward + backward, the time of each kernel (score, raw softmax forward and backward,
aggregation, row and column backward walks, datt reduction) with the achieved rate of its byte model:
  score          nnz (4 f + 4 + 4 K) + 4 f m        one xl row gathered per entry, xr read once per row, scores written
  softmax_fwd    16 K nnz                           scores read twice, alpha read and written
  softmax_bwd    20 K nnz                           alpha and dalpha read twice, dscore written
  row_bwd        nnz (4 f + 8 + 4 K) + 8 f m        xl gathered, dscore staged, xr read and dxr written once per row
  col_bwd        nnz (8 f + 12 + 8 K) + 8 f (m + h) gZ and xr gathered, alpha and dscore staged, xl read, dxl written
The PyTorch-native step (gathers, leaky_relu, scatter_reduce amax, index_add_, autograd) runs on C2 if it fits in the
card's memory, else on the largest R-MAT of half, a quarter, ... of C2's edges that fits, named in the output, where the
GATv2 step is timed again for the ratio. Prints the card's name and power limit read in the same run, then one JSON line.
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


def kernel_times(torch, fn, names, reps=5):
    """ms per call of each kernel whose name contains one of `names`, from a torch.profiler run of `reps` calls."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in names}
    for ev in prof.key_averages():
        for k, sub in names.items():
            if sub in ev.key:
                out[k] += ev.device_time_total / 1e3 / reps
    return out


def native_step(torch, F, rows, cols, n, xl, xr, att, g, slope):
    K, d = att.shape
    t = xl[cols] + xr[rows]
    s = (F.leaky_relu(t, slope).view(-1, K, d) * att[None]).sum(2)
    mx = torch.full((n, K), -float("inf"), device=xl.device).scatter_reduce(0, rows[:, None].expand(-1, K), s.detach(),
                                                                            "amax")
    ex = torch.exp(s - mx[rows])
    den = torch.zeros((n, K), device=xl.device).index_add_(0, rows, ex)
    alpha = ex / den[rows]
    out = torch.zeros((n, K * d), device=xl.device).index_add_(0, rows, alpha.repeat_interleave(d, 1) * xl[cols])
    out.backward(g)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--heads", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-torch", action="store_true", help="skip the PyTorch-native step")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from pgcn_b200 import cabi, graphio, plan as planmod
    from pgcn_b200.op import PGATMultiHeadAttention, PGATv2Attention
    if not torch.cuda.is_available():
        raise SystemExit("bench_gatv2.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, _, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    nnz = lp.nnz()
    plan = planmod.PgcnPlan(lp, max(f, 32), device=dev)
    plan.autotune(f)
    plan.bind_values()
    lib = cabi.load()
    st = lambda: torch.cuda.current_stream().cuda_stream
    call = lambda rc: cabi.check(rc, plan.handle)
    gen = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *s: torch.rand(s, device=dev, generator=gen) * 2 - 1
    xl, xr, g = rnd(n, f), rnd(n, f), rnd(n, f)
    Z, dxl, dxr = (torch.empty((n, f), device=dev) for _ in range(3))
    results = {}
    names = {"score": "gatv2_score", "softmax_fwd": "edge_softmax_raw_kernel", "aggregate": "spmm_heads_kernel",
             "sddmm": "sddmm", "softmax_bwd": "edge_softmax_raw_backward", "row_bwd": "gatv2_row_backward",
             "col_bwd": "gatv2_col_backward", "datt": "gatv2_datt", "fixup": "spmm_fixup"}
    for K in args.heads:
        att = rnd(K, f // K) * 0.3
        datt = torch.empty_like(att)
        alpha = torch.empty((nnz, K), device=dev)
        work = torch.empty_like(alpha)
        fwd = lambda: call(lib.pgcn_forward_gatv2(plan.handle, K, xl.data_ptr(), xr.data_ptr(), att.data_ptr(), 0.2,
                                                  alpha.data_ptr(), Z.data_ptr(), None, f, st()))
        bwd = lambda: call(lib.pgcn_backward_gatv2(plan.handle, K, alpha.data_ptr(), g.data_ptr(), xl.data_ptr(), None,
                                                   xr.data_ptr(), att.data_ptr(), 0.2, work.data_ptr(),
                                                   dxl.data_ptr(), dxr.data_ptr(), datt.data_ptr(), f, st()))
        r = {"forward": median_ms(fwd, args.iters, args.warmup), "backward": median_ms(bwd, args.iters, args.warmup)}
        r["sddmm_heads"] = median_ms(lambda: call(lib.pgcn_sddmm_heads(plan.handle, K, g.data_ptr(), xl.data_ptr(), None,
                                                                       work.data_ptr(), f, st())),
                                     args.iters, args.warmup)
        kt = kernel_times(torch, lambda: (fwd(), bwd()), names)
        if K == 1:
            kt["sddmm"] = kernel_times(torch, lambda: call(lib.pgcn_sddmm_heads(
                plan.handle, K, g.data_ptr(), xl.data_ptr(), None, work.data_ptr(), f, st())), {"sddmm": "sddmm"})["sddmm"]
        r["kernels_ms"] = kt
        r["score_over_sddmm"] = kt["score"] / max(kt["sddmm"], 1e-9)
        XL, XR, AT = (x.clone().requires_grad_(True) for x in (xl, xr, att))

        def step_v2():
            XL.grad = XR.grad = AT.grad = None
            PGATv2Attention.apply(plan, XL, XR, AT, 0.2).backward(g)

        el, er = rnd(n, K).requires_grad_(True), rnd(n, K).requires_grad_(True)

        def step_gat():
            XL.grad = el.grad = er.grad = None
            PGATMultiHeadAttention.apply(plan, XL, el, er, 0.2).backward(g)

        r["step_gatv2"] = median_ms(step_v2, args.iters, args.warmup)
        r["step_gat"] = median_ms(step_gat, args.iters, args.warmup)
        r["gatv2_over_gat"] = r["step_gatv2"] / r["step_gat"]
        model = {"score": nnz * (4 * f + 4 + 4 * K) + 4 * f * n, "softmax_fwd": 16 * K * nnz,
                 "softmax_bwd": 20 * K * nnz, "row_bwd": nnz * (4 * f + 8 + 4 * K) + 8 * f * n,
                 "col_bwd": nnz * (8 * f + 12 + 8 * K) + 8 * f * (n + lp.h)}
        r["bytes"] = model
        r["gbps"] = {k: model[k] / kt[k] / 1e6 for k in model if kt.get(k)}
        results["K%d" % K] = r
        print("K=%d " % K + json.dumps(r), flush=True)

    native = {}
    if not args.no_torch:
        K = args.heads[-1]
        att = rnd(K, f // K) * 0.3
        cur_A, cur_lp, cur_plan, label = A, lp, plan, args.config
        m_edges = nnz
        while True:
            rows = torch.from_numpy(np.repeat(np.arange(cur_lp.m, dtype=np.int64),
                                              np.diff(cur_lp.rowptr.astype(np.int64)))).to(dev)
            cols = torch.from_numpy(cur_lp.colidx.astype(np.int64)).to(dev)
            nn_ = cur_lp.m
            XL, XR, AT = (x.clone().requires_grad_(True) for x in (xl[:nn_], xr[:nn_], att))
            gg = g[:nn_]
            try:
                ms = median_ms(lambda: native_step(torch, F, rows, cols, nn_, XL, XR, AT, gg, 0.2), 3, 1)
                break
            except torch.cuda.OutOfMemoryError:
                del rows, cols, XL, XR, AT
                torch.cuda.empty_cache()
                m_edges //= 2
                label = "R-MAT %d vertices / %d edges" % (n, m_edges)
                cur_A = graphio.synthetic_graph(n, m_edges, seed=1)
                cur_lp = planmod.build_local_plan(cur_A, np.zeros(n, dtype=np.int64), 0, 1)
                if cur_plan is not plan:
                    cur_plan.close()
                cur_plan = planmod.PgcnPlan(cur_lp, f, device=dev)
                cur_plan.bind_values()
        XL2, XR2, AT2 = (x.clone().requires_grad_(True) for x in (xl[:nn_], xr[:nn_], att))
        ours = median_ms(lambda: PGATv2Attention.apply(cur_plan, XL2, XR2, AT2, 0.2).backward(gg), args.iters,
                         args.warmup)
        native = {"graph": label, "nnz": cur_lp.nnz(), "heads": K, "step_torch_native": ms, "step_gatv2": ours,
                  "native_over_gatv2": ms / ours}
        print("native " + json.dumps(native), flush=True)
        if cur_plan is not plan:
            cur_plan.close()

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "iters": args.iters, "warmup": args.warmup,
              "card": card(), "heads": results, "native": native}
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
