"""Edge values on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU: what setting the values, the
SDDMM of their gradient and a weighted aggregation step cost, next to the forward SpMM they are built around.

    python tools/bench_edge_values.py [--iters 30] [--warmup 10] [--config C2]

Reports the median over `iters` launches (each timed with CUDA events, after `warmup` untimed ones) of
  set_values            pgcn_plan_set_values (every record set of the plan rewritten)
  spmm_fwd              the forward SpMM launch (pgcn_spmm, transpose = 0)
  sddmm                 pgcn_sddmm, also as gathered TB/s at 4 f bytes (512 B at f = 128) per edge
  torch_sampled_addmm   torch.sparse.sampled_addmm on the same CSR (the library baseline; no product path uses it)
  step_pspmm            PSpMM forward + backward
  step_weighted         PSpMMWeighted forward + backward with dvals, the same unmodified values every step (they stay
                        resident: forward, backward, SDDMM, no rewrite)
  step_weighted_new_values   the same with other values every step, as after an optimizer update (+ one set_values)
and the card's name and power limit beside them. Prints one JSON line last.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["name"], out["power_limit_w"] = q[0].strip(), float(q[1])
    except Exception:
        pass
    return out


def median_ms(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, plan as planmod
    from pgcn_b200.op import PSpMM, PSpMMWeighted
    if not torch.cuda.is_available():
        raise SystemExit("bench_edge_values.py needs a CUDA device")
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
    lib = cabi.load()
    st = lambda: torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    H = torch.rand((n, f), device=dev, generator=gen) * 2 - 1
    gZ = torch.rand((n, f), device=dev, generator=gen) * 2 - 1
    Z = torch.empty((n, f), device=dev)
    v = torch.rand(nnz, device=dev, generator=gen) + 0.5
    dv = torch.empty(nnz, device=dev)
    res = {}

    res["set_values"] = median_ms(lambda: plan.set_values(v), args.iters, args.warmup)
    plan.set_values(None)
    res["spmm_fwd"] = median_ms(lambda: cabi.check(lib.pgcn_spmm(plan.handle, 0, H.data_ptr(), None, Z.data_ptr(), None,
                                                                 f, st()), plan.handle), args.iters, args.warmup)
    res["sddmm"] = median_ms(lambda: cabi.check(lib.pgcn_sddmm(plan.handle, gZ.data_ptr(), H.data_ptr(), None, dv.data_ptr(),
                                                               f, st()), plan.handle), args.iters, args.warmup)
    d1 = dv.clone()
    cabi.check(lib.pgcn_sddmm(plan.handle, gZ.data_ptr(), H.data_ptr(), None, dv.data_ptr(), f, st()), plan.handle)
    torch.cuda.synchronize()
    res["sddmm_bit_identical_runs"] = bool(torch.equal(d1, dv))
    res["sddmm_gathered_TBps"] = nnz * 4.0 * f / (res["sddmm"] * 1e-3) / 1e12
    res["sddmm_over_spmm_fwd"] = res["sddmm"] / res["spmm_fwd"]

    # library baseline: sampled dense-dense product on the same CSR (cuSPARSE SDDMM through torch)
    rowptr = torch.from_numpy(lp.rowptr.astype(np.int64)).to(dev)
    col = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    S = torch.sparse_csr_tensor(rowptr, col, torch.zeros(nnz, device=dev), size=(n, n))
    Ht = H.t()
    try:
        res["torch_sampled_addmm"] = median_ms(lambda: torch.sparse.sampled_addmm(S, gZ, Ht), args.iters, args.warmup)
        ref = torch.sparse.sampled_addmm(S, gZ, Ht).values()
        res["sddmm_max_abs_diff_vs_torch"] = float((ref - dv).abs().max())
    except RuntimeError as e:                      # report, do not hide
        res["torch_sampled_addmm"] = None
        res["torch_sampled_addmm_error"] = str(e)[:200]
    del S

    g = torch.rand((n, f), device=dev, generator=gen) * 2 - 1
    x = H.clone().requires_grad_(True)
    vw = v.clone().requires_grad_(True)

    def step_plain():
        x.grad = None
        PSpMM.apply(plan, x).backward(g)

    def step_weighted():
        x.grad = None
        vw.grad = None
        PSpMMWeighted.apply(plan, vw, x).backward(g)

    # values that change every step, as after an optimizer update: two tensors in turn, so every step rewrites them
    vs = [v.clone().requires_grad_(True), (v * 0.5).requires_grad_(True)]
    turn = [0]

    def step_weighted_new_values():
        w = vs[turn[0] % 2]
        turn[0] += 1
        x.grad = None
        w.grad = None
        PSpMMWeighted.apply(plan, w, x).backward(g)
    res["step_pspmm"] = median_ms(step_plain, args.iters, args.warmup)
    res["step_weighted"] = median_ms(step_weighted, args.iters, args.warmup)
    res["step_weighted_new_values"] = median_ms(step_weighted_new_values, args.iters, args.warmup)

    out = {"config": args.config, "n": n, "nnz": nnz, "f": f, "iters": args.iters, "warmup": args.warmup,
           "card": card(), "ms": {k: v for k, v in res.items()}}
    for k_, v_ in res.items():
        print("%-28s %s" % (k_, ("%.4f" % v_) if isinstance(v_, float) else v_))
    print("card: %s, power limit %s W" % (out["card"]["name"], out["card"]["power_limit_w"]))
    print(json.dumps(out))
    plan.close()


if __name__ == "__main__":
    main()
