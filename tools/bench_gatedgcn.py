"""GatedGCN on C2 (R-MAT 1 M vertices / 16 M edges + self loops), one GPU: what the three GatedGCN walks cost at
f = 64 and 128, and the fused step against a PyTorch-native step.

    python tools/bench_gatedgcn.py [--iters 20] [--warmup 5] [--config C2] [--widths 64,128] [--native-widths 64,32]

Reports the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward_rows / backward_cols   pgcn_gatedgcn_forward, _backward_rows, _backward_cols (gE given)
  step_gatedgcn                             their sum
  step_op                                   op.aggregate_gatedgcn + op.aggregate_gatedgcn_backward (allocations included)
  step_torch_native                         gathers Dx[row], Ex[col], Bx[col], sigmoid, index_add_, autograd backward
and the achieved rates of the byte models (model bytes over time):
  forward        per entry 16f + 4 B (Ce read, ehat written, [Ex | Bx] row gathered, its index); per row 12f B
                 (Dx read, Z and den written)
  backward_rows  per entry 16f + 4 B (ehat, gE and the Bx half read, dCe written, the index); per row 20f B (gZ, den,
                 Z read, dDx and U written)
  backward_cols  per transposed entry 12f + 8 B (ehat, dCe, U gathered, the index and the permutation); per column
                 8f B ([dEx | dBx] written)
The native step runs at the widest of --native-widths that fits in memory, next to the fused step at that width; its
outputs and gradients must lie within twice the kernels' first-order fp32 bound (tests/gatedgcn_oracle.py's, evaluated
here on the device from the kernels' own outputs). Prints the card's name and power limit read in the same run, then
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

EPS = 1e-6
U32 = 2.0 ** -24
CONST = 16


def bounds(torch, rows, cols, n, deg, cdeg, e, B, Z, den, U, gE):
    """The kernels' first-order fp32 error bound per output (gatedgcn_oracle.terms' propagation, fp32 on the device)."""
    z = lambda: torch.zeros((n, e.shape[1]), device=e.device)
    s = torch.sigmoid(e)
    ds = s * (1 - s)
    q = den + EPS
    d_r, d_c = deg[:, None], cdeg[:, None]
    eden = (d_r + CONST) * U32 * den
    enum = (d_r + CONST) * U32 * z().index_add_(0, rows, (s * B[cols]).abs())
    eq = eden + U32 * q
    eZ = enum / q + Z.abs() * eq / q + U32 * Z.abs()
    eU = U.abs() * (eq / q + U32)
    diff = B[cols] - Z[rows]
    dsig = U[rows] * diff
    edsig = U[rows].abs() * (eZ[rows] + U32 * diff.abs()) + diff.abs() * eU[rows] + U32 * dsig.abs()
    del diff
    dce = gE + dsig * ds
    edce = ds * edsig + dsig.abs() * CONST * U32 * ds + U32 * dce.abs()
    del edsig
    su = (s * U[rows]).abs()
    esu = CONST * U32 * su + s * eU[rows] + U32 * su
    return {"Z": 2 * eZ, "dCe": 2 * edce,
            "dDx": 2 * (z().index_add_(0, rows, edce) + d_r * U32 * z().index_add_(0, rows, dce.abs())),
            "dEx": 2 * (z().index_add_(0, cols, edce) + (d_c + 2) * U32 * z().index_add_(0, cols, dce.abs())),
            "dBx": 2 * (z().index_add_(0, cols, esu) + (d_c + 2) * U32 * z().index_add_(0, cols, su))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--widths", default="64,128")
    ap.add_argument("--native-widths", default="64,32")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_gatedgcn.py needs a CUDA device")
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
    plan = planmod.PgcnPlan(lp, 2 * max(widths + native_widths), device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    perm = plan.transposed_entries()
    nlib = cabi.load_gatedgcn()
    st = lambda: torch.cuda.current_stream().cuda_stream
    chk = cabi.check_gatedgcn
    out = {"config": args.config, "n": n, "nnz": nnz, "max_row": int(deg.max()), "max_col": int(cdeg.max()),
           "split_rows": int(fwd.c.nsplits), "split_cols": int(tr.c.nsplits), "iters": args.iters,
           "warmup": args.warmup, "card": card(), "widths": {}}

    def kernels(f):
        gen = torch.Generator(device=dev).manual_seed(f)
        Dx, Ex, Bx, gZ = (torch.randn((n, f), device=dev, generator=gen) for _ in range(4))
        Ce, gE = torch.randn((nnz, f), device=dev, generator=gen), torch.randn((nnz, f), device=dev, generator=gen)
        EB = torch.cat([Ex, Bx], 1)
        Z, den, U, dDx = (torch.empty((n, f), device=dev) for _ in range(4))
        Ehat, dCe = torch.empty((nnz, f), device=dev), torch.empty((nnz, f), device=dev)
        dEB = torch.empty((n, 2 * f), device=dev)
        w1, w2 = torch.empty((fwd.nslots, 2 * f), device=dev), torch.empty((tr.nslots, 2 * f), device=dev)
        p = lambda x: x.data_ptr()
        calls = {
            "forward": lambda: chk(nlib.pgcn_gatedgcn_forward(C.byref(fwd.c), n, 0, p(Dx), p(EB), None, p(Ce), EPS,
                                                              p(Z), p(den), p(Ehat), p(w1), f, st())),
            "backward_rows": lambda: chk(nlib.pgcn_gatedgcn_backward_rows(
                C.byref(fwd.c), n, 0, p(EB), None, p(Ehat), p(gE), p(Z), p(den), p(gZ), EPS, p(U), p(dCe), p(dDx),
                p(w1), f, st())),
            "backward_cols": lambda: chk(nlib.pgcn_gatedgcn_backward_cols(
                C.byref(tr.c), p(perm), n, 0, p(Ehat), p(dCe), p(U), p(dEB), p(w2), f, st()))}
        res = {name: median_ms(fn, args.iters, args.warmup) for name, fn in calls.items()}
        res["step_gatedgcn"] = res["forward"] + res["backward_rows"] + res["backward_cols"]

        def step_op():
            Zo, Eo, do, EBo, EBh = op.aggregate_gatedgcn(plan, Dx, Ex, Bx, Ce)
            return op.aggregate_gatedgcn_backward(plan, Eo, EBo, EBh, Zo, do, gZ, gE)
        res["step_op"] = median_ms(step_op, args.iters, args.warmup)
        bytes_ = {"forward": nnz * (16 * f + 4) + n * 12 * f,
                  "backward_rows": nnz * (16 * f + 4) + n * 20 * f,
                  "backward_cols": nnz * (12 * f + 8) + n * 8 * f}
        rates = {name + "_tbps": b / res[name] / 1e9 for name, b in bytes_.items()}
        for name, fn in calls.items():
            fn()
        torch.cuda.synchronize()
        state = dict(Dx=Dx, Ex=Ex, Bx=Bx, gZ=gZ, Ce=Ce, gE=gE, Z=Z, den=den, U=U, Ehat=Ehat, dCe=dCe, dDx=dDx,
                     dEx=dEB[:, :f], dBx=dEB[:, f:])
        return res, rates, bytes_, state

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
        res, _, _, k = kernels(f)
        leaves = [k[x].clone().requires_grad_(True) for x in ("Dx", "Ex", "Bx", "Ce")]

        def step_torch_native():
            for u in leaves:
                u.grad = None
            D, E, B, Ce = leaves
            e = (D[rows] + E[cols]) + Ce
            s = torch.sigmoid(e)
            z = torch.zeros((n, f), device=dev)
            Z = z.index_add(0, rows, s * B[cols]) / (z.index_add(0, rows, s) + EPS)
            torch.autograd.backward([Z, e], [k["gZ"], k["gE"]])
            return Z
        try:
            ms = median_ms(step_torch_native, args.iters, args.warmup)
            Zn = step_torch_native().detach()
        except RuntimeError as err:                        # report, do not hide
            native["errors"][f] = str(err)[:200]
            leaves = None
            torch.cuda.empty_cache()
            continue
        native.update({"f": f, "step_torch_native": ms, "step_gatedgcn": res["step_gatedgcn"], "step_op": res["step_op"],
                       "torch_native_over_gatedgcn": ms / res["step_gatedgcn"],
                       "torch_native_over_op": ms / res["step_op"]})
        got = {"Z": Zn, "dDx": leaves[0].grad, "dEx": leaves[1].grad, "dBx": leaves[2].grad, "dCe": leaves[3].grad}
        check = {name + "_within_2x_fp32_bound": True for name in got}
        check.update({name + "_max_abs_diff": 0.0 for name in got})
        with torch.no_grad():
            for c0 in range(0, f, 16):                     # 16 features at a time: the bound's [nnz, .] temporaries
                c = slice(c0, min(f, c0 + 16))
                bnd = bounds(torch, rows, cols, n, dr, dc, *(k[x][:, c] for x in ("Ehat", "Bx", "Z", "den", "U", "gE")))
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
