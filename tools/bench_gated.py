"""Gated aggregation on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU: what the three gated walks
cost, next to the register-kernel sum aggregation at width 2f, which gathers the same bytes per entry, and a
PyTorch-native gated step.

    python tools/bench_gated.py [--iters 30] [--warmup 10] [--config C2]

Reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward_rows / backward_cols   pgcn_gated_forward, pgcn_gated_backward_rows, pgcn_gated_backward_cols
  spmm_register_2f                          pgcn_spmm forward at width 2f with the plan option kernel = 4
  step_torch_native                         gather K[row], Q[col], V[col], sigmoid, index_add_, autograd backward
and the achieved rates of the byte models (DESIGN.md §4):
  forward        per entry 4 B of index + 8f B gathered (Q and V rows); per row 4f B of K read and 4f B of Z written
  backward_rows  the forward's bytes plus 4f B of gZ read per row (dK written in place of Z)
  backward_cols  per transposed entry 4 B of index + 8f B gathered (K and gZ rows); per column 8f B of [Q | V] read
                 and 8f B of [dQ | dV] written
It checks that the native step's output and gradients lie within the fp32 bound 2 (d + 16) 2^-24 sum|terms| of the
kernels' (the same terms summed in another order, d the row's or column's entry count; for dK and dQ sum|terms| also
holds |V eta gZ|, since torch's sigmoid backward forms 1 - y from the rounded y), or prints the native step's error if
it fails, e.g. for memory. Prints the card's name and power limit read in the same run, then
one JSON line.
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
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--no-torch", action="store_true", help="skip the PyTorch-native step")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_gated.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, _, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    cdeg = np.diff(lp.t_rowptr.astype(np.int64))
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    lib, glib = cabi.load(), cabi.load_gated()
    st = lambda: torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    K, Q, V, g = ((torch.randn((n, f), device=dev, generator=gen) * s) for s in (2.0, 2.0, 1.0, 1.0))
    QV = torch.cat([Q, V], 1)
    Z, dK = torch.empty((n, f), device=dev), torch.empty((n, f), device=dev)
    dQV = torch.empty((n, 2 * f), device=dev)
    w1, w2 = torch.empty((fwd.nslots, f), device=dev), torch.empty((tr.nslots, 2 * f), device=dev)
    chk = cabi.check_gated
    res = {}
    res["forward"] = median_ms(lambda: chk(glib.pgcn_gated_forward(C.byref(fwd.c), n, 0, K.data_ptr(), QV.data_ptr(),
                                                                   None, Z.data_ptr(), w1.data_ptr(), f, st())),
                               args.iters, args.warmup)
    res["backward_rows"] = median_ms(lambda: chk(glib.pgcn_gated_backward_rows(
        C.byref(fwd.c), n, 0, K.data_ptr(), QV.data_ptr(), None, g.data_ptr(), dK.data_ptr(), w1.data_ptr(), f,
        st())), args.iters, args.warmup)
    res["backward_cols"] = median_ms(lambda: chk(glib.pgcn_gated_backward_cols(
        C.byref(tr.c), n, 0, K.data_ptr(), QV.data_ptr(), None, g.data_ptr(), dQV.data_ptr(), w2.data_ptr(), f,
        st())), args.iters, args.warmup)
    plan.set_option("kernel", 4)
    out2 = torch.empty((n, 2 * f), device=dev)
    res["spmm_register_2f"] = median_ms(lambda: cabi.check(lib.pgcn_spmm(plan.handle, 0, QV.data_ptr(), None,
                                                                         out2.data_ptr(), None, 2 * f, st()),
                                                           plan.handle), args.iters, args.warmup)
    res["forward_over_register_2f"] = res["forward"] / res["spmm_register_2f"]
    res["step_gated"] = res["forward"] + res["backward_rows"] + res["backward_cols"]

    bytes_ = {"forward": nnz * (4 + 8 * f) + n * 8 * f,
              "backward_rows": nnz * (4 + 8 * f) + n * 12 * f,
              "backward_cols": nnz * (4 + 8 * f) + n * 16 * f}
    rates = {name + "_gbps": b / res[name] / 1e6 for name, b in bytes_.items()}

    check = {}
    if not args.no_torch:
        rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
        cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
        leaves = [x.clone().requires_grad_(True) for x in (K, Q, V)]

        def step_torch_native():
            for u in leaves:
                u.grad = None
            Kp, Qp, Vp = leaves
            o = torch.zeros((n, f), device=dev).index_add_(0, rows, torch.sigmoid(Kp[rows] + Qp[cols]) * Vp[cols])
            o.backward(g)
            return o

        try:
            res["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
            res["torch_native_over_gated"] = res["step_torch_native"] / res["step_gated"]
            o = step_torch_native().detach()
            with torch.no_grad():
                eta = torch.sigmoid(K[rows] + Q[cols])
                ds = eta * (1 - eta)
                d_r = torch.from_numpy(deg.astype(np.float32)).to(dev)[:, None]
                d_c = torch.from_numpy(cdeg[:n].astype(np.float32)).to(dev)[:, None]
                z = lambda: torch.zeros((n, f), device=dev)
                # torch's sigmoid backward takes y (1 - y) from the rounded y: up to 2^-24 y of absolute error in
                # 1 - y, so its dK and dQ terms carry up to 2^-24 |V eta gZ| more
                mags = {"Z": z().index_add_(0, rows, (eta * V[cols]).abs()),
                        "dK": z().index_add_(0, rows, (V[cols] * ds).abs() + (V[cols] * eta).abs()) * g.abs(),
                        "dQ": z().index_add_(0, cols, (g[rows] * ds).abs() + (g[rows] * eta).abs()) * V.abs(),
                        "dV": z().index_add_(0, cols, (eta * g[rows]).abs())}
                pairs = {"Z": (o, Z, d_r), "dK": (leaves[0].grad, dK, d_r), "dQ": (leaves[1].grad, dQV[:, :f], d_c),
                         "dV": (leaves[2].grad, dQV[:, f:], d_c)}
                for name, (a, b, d) in pairs.items():
                    err = (a - b).abs()
                    check[name + "_max_rel_diff"] = float(err.max() / (a.abs().max() + 1e-30))
                    check[name + "_within_fp32_bound"] = bool((err <= 2 * (d + 16) * 2.0 ** -24 * mags[name] +
                                                               1e-30).all())
        except RuntimeError as e:                      # report, do not hide
            res["step_torch_native"] = None
            res["step_torch_native_error"] = str(e)[:300]
            torch.cuda.empty_cache()

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "max_row": int(deg.max()), "max_col": int(cdeg.max()),
              "chunk": int(glib.pgcn_gated_chunk()), "split_rows": int(fwd.c.nsplits), "split_cols": int(tr.c.nsplits),
              "iters": args.iters, "warmup": args.warmup, "card": card(), "ms": res, "gbps": rates, "bytes": bytes_,
              "check": check}
    for k_, v_ in list(res.items()) + list(rates.items()) + list(check.items()):
        print("%-32s %s" % (k_, ("%.4g" % v_) if isinstance(v_, float) else v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
