"""Sparse graph attention on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU: what the edge
softmax kernels and one attention step cost, next to the weighted aggregation step they are built on and a
PyTorch-native sparse attention on the same CSR.

    python tools/bench_attention.py [--iters 30] [--warmup 10] [--config C2]

Reports the median over `iters` calls (each timed with CUDA events, after `warmup` untimed ones) of
  edge_softmax            pgcn_edge_softmax, also as achieved GB/s over SOFTMAX_BYTES_PER_EDGE
  edge_softmax_backward   pgcn_edge_softmax_backward, over BACKWARD_BYTES_PER_EDGE
  spmm_fwd                the forward SpMM launch (pgcn_spmm), for scale
  step_attention          PGATAttention forward + backward (gradients of Z, el and er)
  step_weighted_new_values   PSpMMWeighted forward + backward with other values every step
  step_torch_native       the same attention in PyTorch ops on the same CSR: gather, leaky_relu, scatter_reduce amax,
                          exp, index_add_ for the softmax and for the aggregation (gathered rows
                          scaled by alpha), autograd (a baseline; no product path uses it)
and whether two attention steps give bit-identical outputs and gradients, with the card's name and power limit
beside them. Prints one JSON line last.
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

# Compulsory traffic per stored edge (fp32 / int32 words), as the kernels in csrc/attention.cuh move it:
#   forward:  column word + er[col] gather + score written + score read back twice + alpha written    = 24 B
#   backward: alpha + dalpha (row sum), then alpha + dalpha + column + er[col] + dpre written           = 28 B
SOFTMAX_BYTES_PER_EDGE = 24
BACKWARD_BYTES_PER_EDGE = 28


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from pgcn_b200 import cabi, graphio, plan as planmod
    from pgcn_b200.op import PGATAttention, PSpMMWeighted
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a CUDA device")
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
    el, er = rnd(n), rnd(n)
    alpha, dalpha, dpre = torch.empty(nnz, device=dev), rnd(nnz), torch.empty(nnz, device=dev)
    d_el = torch.empty(n, device=dev)
    out = torch.empty((n, f), device=dev)
    res = {}

    res["edge_softmax"] = median_ms(lambda: cabi.check(lib.pgcn_edge_softmax(
        plan.handle, el.data_ptr(), er.data_ptr(), None, 0.2, alpha.data_ptr(), st()), plan.handle),
        args.iters, args.warmup)
    res["edge_softmax_backward"] = median_ms(lambda: cabi.check(lib.pgcn_edge_softmax_backward(
        plan.handle, el.data_ptr(), er.data_ptr(), None, alpha.data_ptr(), dalpha.data_ptr(), 0.2, dpre.data_ptr(),
        d_el.data_ptr(), st()), plan.handle), args.iters, args.warmup)
    res["edge_softmax_GBps"] = nnz * SOFTMAX_BYTES_PER_EDGE / (res["edge_softmax"] * 1e-3) / 1e9
    res["edge_softmax_backward_GBps"] = nnz * BACKWARD_BYTES_PER_EDGE / (res["edge_softmax_backward"] * 1e-3) / 1e9
    plan.set_values(None)
    res["spmm_fwd"] = median_ms(lambda: cabi.check(lib.pgcn_spmm(plan.handle, 0, Z.data_ptr(), None, out.data_ptr(),
                                                                 None, f, st()), plan.handle), args.iters, args.warmup)

    Zp, elp, erp = (t.clone().requires_grad_(True) for t in (Z, el, er))

    def step_attention():
        for t in (Zp, elp, erp):
            t.grad = None
        o = PGATAttention.apply(plan, Zp, elp, erp, 0.2)
        o.backward(g)
        return o

    vs = [(torch.rand(nnz, device=dev, generator=gen) + 0.5).requires_grad_(True) for _ in range(2)]
    turn = [0]

    def step_weighted_new_values():
        w = vs[turn[0] % 2]
        turn[0] += 1
        Zp.grad = None
        w.grad = None
        PSpMMWeighted.apply(plan, w, Zp).backward(g)

    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)

    def step_torch_native():
        for t in (Zp, elp, erp):
            t.grad = None
        s = F.leaky_relu(elp[rows] + erp[cols], 0.2)
        mx = torch.full((n,), -float("inf"), device=dev).scatter_reduce(0, rows, s, "amax", include_self=True)
        ex = torch.exp(s - mx[rows].detach())
        den = torch.zeros(n, device=dev).index_add_(0, rows, ex)
        a = ex / den[rows]
        # torch.sparse.mm(S, Z) on the same CSR would be the natural call, but its backward to S's values builds a dense
        # n x n gradient (3.7 TiB on C2): the aggregation is a gather and index_add_ instead (nnz x f floats, 8.7 GB)
        o = torch.zeros((n, f), device=dev).index_add_(0, rows, a[:, None] * Zp[cols])
        o.backward(g)

    res["step_attention"] = median_ms(step_attention, args.iters, args.warmup)
    res["step_weighted_new_values"] = median_ms(step_weighted_new_values, args.iters, args.warmup)
    try:
        res["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
    except RuntimeError as e:                      # report, do not hide
        res["step_torch_native"] = None
        res["step_torch_native_error"] = str(e)[:200]
    res["attention_over_weighted"] = res["step_attention"] / res["step_weighted_new_values"]
    if res["step_torch_native"]:
        res["torch_native_over_attention"] = res["step_torch_native"] / res["step_attention"]

    runs = []
    for _ in range(2):
        o = step_attention()
        torch.cuda.synchronize()
        runs.append([t.detach().clone() for t in (o, Zp.grad, elp.grad, erp.grad)])
    res["bit_identical_runs"] = all(torch.equal(a, b) for a, b in zip(*runs))

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "max_row": int(deg.max()),
              "long_rows": int((deg > 1024).sum()), "iters": args.iters, "warmup": args.warmup, "card": card(),
              "ms": res}
    for k_, v_ in res.items():
        print("%-28s %s" % (k_, ("%.4f" % v_) if isinstance(v_, float) else v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
