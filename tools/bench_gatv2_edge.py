"""GATv2 attention with edge features on C2 (R-MAT 1 M vertices / 16 M edges + self loops), one GPU, heads K in
{1, 4, 8}: what the three fused kernels cost, next to op.PGATv2Attention without edges and a PyTorch-native
GATv2Conv(edge_dim) step.

    python tools/bench_gatv2_edge.py [--iters 20] [--warmup 5] [--config C2] [--heads 1,4,8] [--widths 128,64]
                                     [--native-width 64]

Reports, per width f and K, the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward_rows / backward_cols   pgcn_gatv2_edge_forward, _backward_rows, _backward_cols
  step                                      op.aggregate_gatv2_edge + op.aggregate_gatv2_edge_backward (with dE): the
                                            three walks, the exchange calls and the operator's allocations
  step_p03                                  the same with attention dropout p = 0.3 (the mask drawn inline)
  noedge_step                               op.PGATv2Attention forward + backward (autograd) on the same XL, XR, att
  step_torch_native                         (at the native width) gathers XR[row], XL[col], adds E, LeakyReLU, a scatter
                                            softmax, index_add_, autograd for XL, XR, att and E
The byte model (DESIGN.md §4): the forward gathers 4 B of index + 4f B (XL[j]) and streams 4f B of E per entry, and
reads 4f B of XR and writes 4f B of Z per row; the row walk reads the same per entry and writes g (4f B) and [P | ds]
(8K B), and reads 12f B (XR, gZ, Z) and writes 4f B (dXR) per row; the column walk reads 8 B of index and perm,
gathers 4f B of gZ and reads 4f B of g and 4K B of P per transposed entry and writes 4f B of dXL per column. The native
step's outputs and gradients are compared with the fused kernels' (largest difference relative to the largest
magnitude). Prints the card's name and power limit read in the same run, then one JSON line.
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

SLOPE = 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--heads", default="1,4,8")
    ap.add_argument("--widths", default="128,64")
    ap.add_argument("--native-width", type=int, default=64, help="width of the PyTorch-native step; 0 skips it")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_gatv2_edge.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = graphio.CONFIGS[args.config][0]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    widths = [int(x) for x in args.widths.split(",")]
    plan = planmod.PgcnPlan(lp, max(widths), device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    gid = plan.global_ids()
    perm = plan.transposed_entries()
    lib = cabi.load_gatv2_edge()
    cabi.check_gatv2_edge(lib.pgcn_gatv2_edge_load())
    st = lambda: torch.cuda.current_stream().cuda_stream
    chk = cabi.check_gatv2_edge
    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    res, rates, check = {}, {}, {}

    for f in widths:
        gen = torch.Generator(device=dev).manual_seed(1)
        XL, XR, g = (torch.randn((n, f), device=dev, generator=gen) for _ in range(3))
        E = torch.randn((nnz, f), device=dev, generator=gen) * 0.5
        for heads in [int(x) for x in args.heads.split(",")]:
            att = torch.randn((heads, f // heads), device=dev, generator=gen) * 0.3
            Z, L, dXR, D = (torch.empty(s, device=dev) for s in ((n, f), (n, heads), (n, f), (n, heads)))
            dXL = torch.empty((n, f), device=dev)
            PS, G = torch.empty((nnz, 2 * heads), device=dev), torch.empty((nnz, f), device=dev)
            datt = torch.empty(f, device=dev)
            w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev)
            w1 = torch.empty((lib.pgcn_gatv2_edge_work_rows(C.byref(fwd.c)), f), device=dev)
            w2 = torch.empty((tr.nslots, f), device=dev)
            head = (n, 0, heads, XL.data_ptr(), None, XR.data_ptr(), att.data_ptr(), E.data_ptr(), SLOPE,
                    gid.data_ptr(), None, 0, 1.0)
            fw = lambda: chk(lib.pgcn_gatv2_edge_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                         w0.data_ptr(), f, st()))
            rw = lambda: chk(lib.pgcn_gatv2_edge_backward_rows(
                C.byref(fwd.c), *head, g.data_ptr(), Z.data_ptr(), L.data_ptr(), dXR.data_ptr(), D.data_ptr(),
                PS.data_ptr(), G.data_ptr(), datt.data_ptr(), w1.data_ptr(), f, st()))
            cw = lambda: chk(lib.pgcn_gatv2_edge_backward_cols(
                C.byref(tr.c), perm.data_ptr(), n, 0, heads, g.data_ptr(), PS.data_ptr(), G.data_ptr(), dXL.data_ptr(),
                w2.data_ptr(), f, st()))
            it, wu = args.iters, args.warmup
            r = {"forward": median_ms(fw, it, wu), "backward_rows": median_ms(rw, it, wu),
                 "backward_cols": median_ms(cw, it, wu)}
            drop = op.EdgeDropout(0.3, 12345, dev)

            def step(d=None):
                Zs, Ls, XLh, snap = op.aggregate_gatv2_edge(plan, XL, XR, att, E, SLOPE, d)
                return (Zs,) + op.aggregate_gatv2_edge_backward(plan, XL, XLh, XR, att, E, Zs, Ls, g, SLOPE, d, snap)

            r["step"] = median_ms(step, it, wu)
            r["step_p03"] = median_ms(lambda: step(drop), it, wu)
            nl = [x.clone().requires_grad_(True) for x in (XL, XR, att)]

            def noedge_step():
                for u in nl:
                    u.grad = None
                op.PGATv2Attention.apply(plan, *nl, SLOPE).backward(g)

            r["noedge_step"] = median_ms(noedge_step, it, wu)
            r["step_over_noedge_step"] = r["step"] / r["noedge_step"]
            del nl
            fw(), rw(), cw()                                  # the outputs without dropout, kept for the check
            torch.cuda.synchronize()
            K = heads
            bytes_ = {"forward": nnz * (4 + 8 * f) + n * 8 * f,
                      "backward_rows": nnz * (4 + 12 * f + 8 * K) + n * 16 * f,
                      "backward_cols": nnz * (8 + 8 * f + 4 * K) + n * 4 * f}
            rates["f%d_K%d" % (f, heads)] = {name + "_gbps": b / r[name] / 1e6 for name, b in bytes_.items()}
            ck = {}
            if f == args.native_width:
                d = f // heads
                idx = rows[:, None].expand(-1, heads)
                leaves = [x.clone().requires_grad_(True) for x in (XL, XR, att, E)]

                def step_torch_native():
                    for u in leaves:
                        u.grad = None
                    XLp, XRp, ap_, Ep = leaves
                    t = (XRp[rows] + XLp[cols]) + Ep
                    s = (F.leaky_relu(t, SLOPE).view(-1, heads, d) * ap_[None]).sum(2)
                    mx = torch.full((n, heads), -float("inf"), device=dev).scatter_reduce(0, idx, s.detach(), "amax")
                    e = torch.exp(s - mx[rows])
                    al = e / torch.zeros((n, heads), device=dev).index_add(0, rows, e)[rows]
                    msg = (al[:, :, None] * XLp[cols].view(-1, heads, d)).reshape(-1, f)
                    o = torch.zeros((n, f), device=dev).index_add(0, rows, msg)
                    o.backward(g)
                    return o

                try:
                    r["step_torch_native"] = median_ms(step_torch_native, it, wu)
                    r["torch_native_over_fused"] = r["step_torch_native"] / r["step"]
                    o = step_torch_native().detach()
                    nat = {"Z": o, "dXL": leaves[0].grad, "dXR": leaves[1].grad, "datt": leaves[2].grad.reshape(-1),
                           "dE": leaves[3].grad}
                    fused = {"Z": Z, "dXL": dXL, "dXR": dXR, "datt": datt, "dE": G}
                    for name in fused:
                        err = (nat[name] - fused[name]).abs()
                        ck["native_" + name + "_max_rel_diff"] = float(err.max() / (nat[name].abs().max() + 1e-30))
                    del o, nat
                except RuntimeError as e:                  # report, do not hide
                    r["step_torch_native"] = None
                    r["step_torch_native_error"] = str(e)[:300]
                del leaves
            res["f%d_K%d" % (f, heads)] = r
            check["f%d_K%d" % (f, heads)] = ck
            del Z, L, dXR, D, dXL, PS, G, w0, w1, w2
            torch.cuda.empty_cache()
        del XL, XR, g, E
        torch.cuda.empty_cache()

    result = {"config": args.config, "n": n, "nnz": nnz, "max_row": int(deg.max()), "split_rows": int(fwd.c.nsplits),
              "split_cols": int(tr.c.nsplits), "iters": args.iters, "warmup": args.warmup, "card": card(), "ms": res,
              "gbps": rates, "check": check}
    for k_, v_ in res.items():
        for a, b in list(v_.items()) + list(rates[k_].items()) + list(check[k_].items()):
            print("%-8s %-32s %s" % (k_, a, ("%.4g" % b) if isinstance(b, float) else b))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
