"""Max aggregation on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU: what pgcn_forward_max and
pgcn_backward_max cost, next to the sum aggregation's register-kernel and ring launches and a PyTorch-native max step.

    python tools/bench_max.py [--iters 30] [--warmup 10] [--config C2]

Reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward_max / backward_max      the two entry points
  spmm_register_fwd / _bwd        pgcn_spmm forward / transposed with the plan option kernel = 4 (the register kernel)
  spmm_ring_fwd / _bwd            pgcn_spmm forward / transposed on the default ring kernel
  step_torch_native               gather [nnz, f], scatter_reduce("amax", include_self=False), autograd backward
and the achieved rates of the byte models (DESIGN.md §4):
  forward_max    the register SpMM's compulsory bytes (pgcn_algorithmic_bytes spmm_fwd) + 4 f m for arg
  backward_max   per transposed entry 8 B of indices, 4 B of value map and 8 f B gathered (gZ and arg rows, no reuse),
                 plus 4 f (m + h) written
It checks that the max values equal the PyTorch baseline bit for bit and, on tie-free inputs (every column of H a
permutation of 1 .. n, so no row's max ties the baseline's zero-initialised output either), that the gradients agree
within the fp32 bound of summing the same terms in another order. Prints the card's name and power limit read in the
same run, then one JSON line.
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
    ap.add_argument("--no-torch", action="store_true", help="skip the PyTorch-native step")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_max.py needs a CUDA device")
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
    call = lambda rc: cabi.check(rc, plan.handle)
    # tie-free: every column a permutation of 1 .. n (exact in fp32)
    gen = torch.Generator(device=dev).manual_seed(1)
    H = torch.argsort(torch.rand((n, f), device=dev, generator=gen), dim=0).to(torch.float32) + 1
    g = torch.rand((n, f), device=dev, generator=gen) * 2 - 1
    Z = torch.empty((n, f), device=dev)
    arg = torch.empty((n, f), dtype=torch.int32, device=dev)
    G = torch.empty((n, f), device=dev)
    out = torch.empty((n, f), device=dev)
    res = {}
    res["forward_max"] = median_ms(lambda: call(lib.pgcn_forward_max(plan.handle, H.data_ptr(), Z.data_ptr(),
                                                                     arg.data_ptr(), f, st())), args.iters, args.warmup)
    res["backward_max"] = median_ms(lambda: call(lib.pgcn_backward_max(plan.handle, arg.data_ptr(), g.data_ptr(),
                                                                       G.data_ptr(), f, st())), args.iters, args.warmup)
    spmm = lambda tr, x: call(lib.pgcn_spmm(plan.handle, tr, x.data_ptr(), None, out.data_ptr(), None, f, st()))
    kernel = plan.get_option("kernel")
    plan.set_option("kernel", 4)
    res["spmm_register_fwd"] = median_ms(lambda: spmm(0, H), args.iters, args.warmup)
    res["spmm_register_bwd"] = median_ms(lambda: spmm(1, g), args.iters, args.warmup)
    plan.set_option("kernel", kernel)
    res["spmm_ring_fwd"] = median_ms(lambda: spmm(0, H), args.iters, args.warmup)
    res["spmm_ring_bwd"] = median_ms(lambda: spmm(1, g), args.iters, args.warmup)
    res["forward_over_register_sum"] = res["forward_max"] / res["spmm_register_fwd"]
    res["backward_over_register_sum"] = res["backward_max"] / res["spmm_register_bwd"]

    b = plan.algorithmic_bytes(f)
    bytes_fwd = b["spmm_fwd"] + 4 * f * lp.m
    bytes_bwd = nnz * (8 + 4 + 8 * f) + 4 * f * (lp.m + lp.h)
    rates = {"forward_max_gbps": bytes_fwd / res["forward_max"] / 1e6,
             "backward_max_gbps": bytes_bwd / res["backward_max"] / 1e6}

    check = {}
    if not args.no_torch:
        rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
        cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
        idx = rows[:, None].expand(-1, f)
        Hp = H.clone().requires_grad_(True)

        def step_torch_native():
            Hp.grad = None
            o = torch.zeros((n, f), device=dev).scatter_reduce(0, idx, Hp[cols], "amax", include_self=False)
            o.backward(g)
            return o

        try:
            res["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
            res["step_max"] = res["forward_max"] + res["backward_max"]
            res["torch_native_over_max"] = res["step_torch_native"] / res["step_max"]
            o = step_torch_native()
            torch.cuda.synchronize()
            check["values_bit_identical"] = bool(torch.equal(o.detach().view(torch.int32), Z.view(torch.int32)))
            # the same terms summed in another order: the fp32 bound 2 (d + 2) 2^-24 sum|terms| per element, with d the
            # column's entry count and sum|terms| the routed gradient of |g|
            mag = torch.empty_like(G)
            ga = g.abs()
            call(lib.pgcn_backward_max(plan.handle, arg.data_ptr(), ga.data_ptr(), mag.data_ptr(), f, st()))
            cdeg = torch.from_numpy(np.diff(lp.t_rowptr.astype(np.int64))[:n].astype(np.float32)).to(dev)[:, None]
            err = (Hp.grad - G).abs()
            check["grad_max_rel_diff"] = float(err.max() / (Hp.grad.abs().max() + 1e-30))
            check["grad_within_fp32_bound"] = bool((err <= 2 * (cdeg + 2) * 2.0 ** -24 * mag + 1e-30).all())
        except RuntimeError as e:                      # report, do not hide
            res["step_torch_native"] = None
            res["step_torch_native_error"] = str(e)[:200]
            torch.cuda.empty_cache()

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "max_row": int(deg.max()), "iters": args.iters,
              "warmup": args.warmup, "card": card(), "ms": res, "gbps": rates, "bytes": {"forward_max": bytes_fwd,
              "backward_max": bytes_bwd}, "check": check}
    for k_, v_ in list(res.items()) + list(rates.items()) + list(check.items()):
        print("%-28s %s" % (k_, ("%.4g" % v_) if isinstance(v_, float) else v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
