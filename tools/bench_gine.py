"""GINE on C2 (R-MAT 1 M vertices / 16 M edges + self loops), one GPU: what the two GINE walks cost at f = 64 and 128,
and the fused step against a PyTorch-native step.

    python tools/bench_gine.py [--iters 20] [--warmup 5] [--config C2] [--widths 64,128] [--native-widths 128,64]

Reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward     pgcn_gine_forward, pgcn_gine_backward (dE written)
  backward_no_dE         pgcn_gine_backward with dE = NULL
  step_gine              forward + backward
  step_op                op.aggregate_gine + op.aggregate_gine_backward (allocations included)
  step_torch_native      X[col] + E, relu, index_add_, autograd backward to X and E
and the achieved rates of the byte models (model bytes over time):
  forward         per entry 8f + 4 B (E read, X[j] gathered, the index); per row 4f B (Z written)
  backward        per transposed entry 12f + 8 B (E read, gZ[i] gathered, dE written, the index and the permutation);
                  per column 8f B (X read, dX written)
  backward_no_dE  per transposed entry 8f + 8 B; per column 8f B
The native step runs at the widest of --native-widths that fits in memory, next to the fused step at that width; its Z
and dX must lie within twice the kernels' first-order fp32 bound (tests/gine_oracle.py's, evaluated here on the device)
and its dE must have the kernels' bits. Prints the card's name and power limit read in the same run, then one JSON
line.
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

U32 = 2.0 ** -24


def bounds(torch, rows, cols, n, deg, cdeg, X, E, dE):
    """The kernels' first-order fp32 error bound of Z and dX (gine_oracle.terms' propagation, fp32 on the device)."""
    z = lambda: torch.zeros((n, X.shape[1]), device=X.device)
    pre = X[cols] + E
    msg = torch.relu(pre)
    eZ = z().index_add_(0, rows, U32 * pre.abs()) + deg[:, None] * U32 * z().index_add_(0, rows, msg)
    eX = (cdeg[:, None] + 2) * U32 * z().index_add_(0, cols, dE.abs())
    return {"Z": 2 * eZ, "dX": 2 * eX}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--widths", default="64,128")
    ap.add_argument("--native-widths", default="128,64")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_gine.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = graphio.CONFIGS[args.config][0]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    cdeg = np.diff(lp.t_rowptr.astype(np.int64))
    widths = [int(x) for x in args.widths.split(",")]
    native_widths = [int(x) for x in args.native_widths.split(",")]
    plan = planmod.PgcnPlan(lp, max(widths + native_widths), device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    perm = plan.transposed_entries()
    lib = cabi.load_gine()
    st = lambda: torch.cuda.current_stream().cuda_stream
    chk = cabi.check_gine
    out = {"config": args.config, "n": n, "nnz": nnz, "max_row": int(deg.max()), "max_col": int(cdeg.max()),
           "split_rows": int(fwd.c.nsplits), "split_cols": int(tr.c.nsplits), "iters": args.iters,
           "warmup": args.warmup, "card": card(), "widths": {}}

    def kernels(f):
        gen = torch.Generator(device=dev).manual_seed(f)
        X, gZ = (torch.randn((n, f), device=dev, generator=gen) for _ in range(2))
        E = torch.randn((nnz, f), device=dev, generator=gen)
        Z, dX = torch.empty((n, f), device=dev), torch.empty((n, f), device=dev)
        dE = torch.empty((nnz, f), device=dev)
        w1, w2 = torch.empty((fwd.nslots, f), device=dev), torch.empty((tr.nslots, f), device=dev)
        p = lambda x: None if x is None else x.data_ptr()

        def backward(de):
            return lambda: chk(lib.pgcn_gine_backward(C.byref(tr.c), p(perm), n, 0, p(X), None, p(E), p(gZ), p(de),
                                                      p(dX), p(w2), f, st()))
        calls = {"forward": lambda: chk(lib.pgcn_gine_forward(C.byref(fwd.c), n, 0, p(X), None, p(E), p(Z), p(w1), f,
                                                              st())),
                 "backward_no_dE": backward(None),
                 "backward": backward(dE)}
        res = {name: median_ms(fn, args.iters, args.warmup) for name, fn in calls.items()}
        res["step_gine"] = res["forward"] + res["backward"]

        def step_op():
            Zo, Xh = op.aggregate_gine(plan, X, E)
            return op.aggregate_gine_backward(plan, X, Xh, E, gZ)
        res["step_op"] = median_ms(step_op, args.iters, args.warmup)
        bytes_ = {"forward": nnz * (8 * f + 4) + n * 4 * f,
                  "backward": nnz * (12 * f + 8) + n * 8 * f,
                  "backward_no_dE": nnz * (8 * f + 8) + n * 8 * f}
        rates = {name + "_tbps": b / res[name] / 1e9 for name, b in bytes_.items()}
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        return res, rates, bytes_, dict(X=X, E=E, gZ=gZ, Z=Z, dX=dX, dE=dE)

    for f in widths:
        res, rates, bytes_, state = kernels(f)
        out["widths"][f] = {"ms": res, "tbps": rates, "bytes": bytes_}
        del state
        torch.cuda.empty_cache()

    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    dr = torch.from_numpy(deg.astype(np.float32)).to(dev)
    dc = torch.from_numpy(cdeg[:n].astype(np.float32)).to(dev)
    native = {"errors": {}}
    for f in native_widths:
        k = leaves = None
        torch.cuda.empty_cache()
        try:
            res, _, _, k = kernels(f)
            leaves = [k[x].clone().requires_grad_(True) for x in ("X", "E")]

            def step_torch_native():
                for u in leaves:
                    u.grad = None
                X, E = leaves
                Z = torch.zeros((n, f), device=dev).index_add_(0, rows, torch.relu(X[cols] + E))
                Z.backward(k["gZ"])
                return Z
            ms = median_ms(step_torch_native, args.iters, args.warmup)
            Zn = step_torch_native().detach()
        except RuntimeError as err:                        # report, do not hide
            native["errors"][f] = str(err)[:200]
            k = leaves = None
            continue
        native.update({"f": f, "step_torch_native": ms, "step_gine": res["step_gine"], "step_op": res["step_op"],
                       "torch_native_over_gine": ms / res["step_gine"], "torch_native_over_op": ms / res["step_op"]})
        check = {"dE_bit_equal": bool(torch.equal(leaves[1].grad.view(torch.int32), k["dE"].view(torch.int32)))}
        got = {"Z": Zn, "dX": leaves[0].grad}
        check.update({name + "_within_2x_fp32_bound": True for name in got})
        check.update({name + "_max_abs_diff": 0.0 for name in got})
        leaves[1].grad = None
        with torch.no_grad():
            for c0 in range(0, f, 16):                     # 16 features at a time: the bound's [nnz, .] temporaries
                c = slice(c0, min(f, c0 + 16))
                bnd = bounds(torch, rows, cols, n, dr, dc, k["X"][:, c], k["E"][:, c], k["dE"][:, c])
                for name, a in got.items():
                    err = (a[:, c] - k[name][:, c]).abs()
                    check[name + "_within_2x_fp32_bound"] &= bool((err <= 2 * bnd[name] + 1e-30).all())
                    check[name + "_max_abs_diff"] = max(check[name + "_max_abs_diff"], float(err.max()))
                del bnd
        native["check"] = check
        break
    out["native"] = native

    for f, w in out["widths"].items():
        for k_, v_ in list(w["ms"].items()) + list(w["tbps"].items()):
            print("f=%-4d %-28s %.4g" % (f, k_, v_))
    for k_, v_ in native.items():
        print("native %-28s %s" % (k_, v_))
    print("card: %s, power limit %s W" % (out["card"]["name"], out["card"]["power_limit_w"]))
    print(json.dumps(out))
    plan.close()


if __name__ == "__main__":
    main()
