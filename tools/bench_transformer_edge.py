"""Graph transformer attention with edge features on C2 (R-MAT 1 M vertices / 16 M edges + self loops), one GPU, heads
K in {1, 4, 8}: what the three fused kernels cost, next to the attention without edges and a PyTorch-native
TransformerConv(edge_dim) step.

    python tools/bench_transformer_edge.py [--iters 20] [--warmup 5] [--config C2] [--heads 1,4,8] [--widths 128,64]
                                           [--native-width 64]

Reports, per width f and K, the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward_rows / backward_cols   pgcn_transformer_edge_forward, _backward_rows (with dE), _backward_cols
  step                                      the three in a row (forward + backward)
  step_p01                                  the same with attention dropout p = 0.1 (the mask drawn inline)
  noedge_forward / noedge_cols / noedge_step  pgcn_transformer_* without edges on the same plan and inputs
  step_torch_native                         (at the native width) gathers q[row], k[col] + E, v[col] + E, a scatter
                                            softmax, index_add_, autograd for Q, K, V and E
The byte model (DESIGN.md §4): the forward gathers 4 B of index + 8f B ([k | v]) and streams 4f B of E per entry, and
reads 4f B of q and writes 4f B of Z per row; the row walk streams E and writes dE (8f B) and [P | ds] (8K B) per entry
besides the forward's gathers, and reads 4f B of gZ and 4f B of Z per row; the column walk reads 8 B of index and perm,
gathers 8f B (q and gZ) and 8K B of [P | ds] per transposed entry and writes 8f B per column. The native step's outputs
and gradients are compared with the fused kernels' (largest difference relative to the largest magnitude). Prints the
card's name and power limit read in the same run, then one JSON line.
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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--heads", default="1,4,8")
    ap.add_argument("--widths", default="128,64")
    ap.add_argument("--native-width", type=int, default=64, help="width of the PyTorch-native step; 0 skips it")
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "pgcn_b200_cache"))
    args = ap.parse_args()

    import torch
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_transformer_edge.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = graphio.CONFIGS[args.config][0]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    widths = [int(x) for x in args.widths.split(",")]
    plan = planmod.PgcnPlan(lp, 2 * max(widths), device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    gid = plan.global_ids()
    perm = plan.transposed_entries()
    elib, tlib = cabi.load_transformer_edge(), cabi.load_transformer()
    cabi.check_transformer_edge(elib.pgcn_transformer_edge_load())
    st = lambda: torch.cuda.current_stream().cuda_stream
    chk, tchk = cabi.check_transformer_edge, cabi.check_transformer
    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    res, rates, check = {}, {}, {}

    for f in widths:
        gen = torch.Generator(device=dev).manual_seed(1)
        Q, K, V, g = ((torch.randn((n, f), device=dev, generator=gen) * s) for s in (1.5, 1.5, 1.0, 1.0))
        E = torch.randn((nnz, f), device=dev, generator=gen) * 0.5
        KV = torch.cat([K, V], 1)
        for heads in [int(x) for x in args.heads.split(",")]:
            sc = op.transformer_scale(f, heads)
            Z, L, dQ, D = (torch.empty(s, device=dev) for s in ((n, f), (n, heads), (n, f), (n, heads)))
            dKV = torch.empty((n, 2 * f), device=dev)
            PS = torch.empty((nnz, 2 * heads), device=dev)
            dE = torch.empty((nnz, f), device=dev)
            w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev)
            w1, w2 = torch.empty((fwd.nslots, f), device=dev), torch.empty((tr.nslots, 2 * f), device=dev)
            drop = op.EdgeDropout(0.1, 12345, dev)

            def calls(dargs):
                head = (n, 0, heads, Q.data_ptr(), KV.data_ptr(), None, E.data_ptr(), sc, gid.data_ptr()) + dargs
                return (lambda: chk(elib.pgcn_transformer_edge_forward(C.byref(fwd.c), *head, Z.data_ptr(),
                                                                       L.data_ptr(), w0.data_ptr(), f, st())),
                        lambda: chk(elib.pgcn_transformer_edge_backward_rows(
                            C.byref(fwd.c), *head, g.data_ptr(), Z.data_ptr(), L.data_ptr(), dQ.data_ptr(),
                            D.data_ptr(), PS.data_ptr(), dE.data_ptr(), w1.data_ptr(), f, st())),
                        lambda: chk(elib.pgcn_transformer_edge_backward_cols(
                            C.byref(tr.c), perm.data_ptr(), n, 0, heads, Q.data_ptr(), g.data_ptr(), PS.data_ptr(),
                            sc, dKV.data_ptr(), w2.data_ptr(), f, st())))

            def plain_calls():
                head = (n, 0, heads, Q.data_ptr(), KV.data_ptr(), None, sc, gid.data_ptr(), None, 0, 1.0)
                return (lambda: tchk(tlib.pgcn_transformer_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                                   w0.data_ptr(), f, st())),
                        lambda: tchk(tlib.pgcn_transformer_backward_rows(
                            C.byref(fwd.c), *head, g.data_ptr(), Z.data_ptr(), L.data_ptr(), dQ.data_ptr(),
                            D.data_ptr(), w1.data_ptr(), f, st())),
                        lambda: tchk(tlib.pgcn_transformer_backward_cols(
                            C.byref(tr.c), *head, g.data_ptr(), L.data_ptr(), D.data_ptr(), dKV.data_ptr(),
                            w2.data_ptr(), f, st())))

            it, wu = args.iters, args.warmup
            pf, pr, pc = plain_calls()
            r = {"noedge_forward": median_ms(pf, it, wu), "noedge_backward_rows": median_ms(pr, it, wu),
                 "noedge_backward_cols": median_ms(pc, it, wu)}
            r["noedge_step"] = median_ms(lambda: (pf(), pr(), pc()), it, wu)
            fw, rw, cw = calls((None, 0, 1.0))
            r["forward"] = median_ms(fw, it, wu)
            r["backward_rows"] = median_ms(rw, it, wu)
            r["backward_cols"] = median_ms(cw, it, wu)
            r["step"] = median_ms(lambda: (fw(), rw(), cw()), it, wu)
            snap = drop.draw()
            dfw, drw, dcw = calls((snap.data_ptr(), drop.threshold, drop.scale))
            r["step_p01"] = median_ms(lambda: (dfw(), drw(), dcw()), it, wu)
            # the aim: the no-edge forward plus streaming E at 3 TB/s
            r["forward_aim"] = r["noedge_forward"] + nnz * 4 * f / 3e12 * 1e3
            r["cols_over_noedge_cols"] = r["backward_cols"] / r["noedge_backward_cols"]
            fw(), rw(), cw()                                  # the outputs at p = 0, kept for the check
            torch.cuda.synchronize()
            bytes_ = {"forward": nnz * (4 + 12 * f) + n * 8 * f,
                      "backward_rows": nnz * (4 + 20 * f + 8 * heads) + n * 16 * f,
                      "backward_cols": nnz * (8 + 8 * f + 8 * heads) + n * 8 * f,
                      "noedge_forward": nnz * (4 + 8 * f) + n * 8 * f,
                      "noedge_backward_cols": nnz * (4 + 8 * f + 8 * heads) + n * 16 * f}
            rates["f%d_K%d" % (f, heads)] = {name + "_gbps": b / r[name] / 1e6 for name, b in bytes_.items()}
            ck = {}
            if f == args.native_width:
                Cw = f // heads
                idx = rows[:, None].expand(-1, heads)
                leaves = [x.clone().requires_grad_(True) for x in (Q, K, V, E)]

                def step_torch_native():
                    for u in leaves:
                        u.grad = None
                    Qp, Kp, Vp, Ep = leaves
                    s = (Qp[rows].view(-1, heads, Cw) * (Kp[cols] + Ep).view(-1, heads, Cw)).sum(2) * sc
                    mx = torch.full((n, heads), -float("inf"), device=dev).scatter_reduce(0, idx, s.detach(), "amax")
                    e = torch.exp(s - mx[rows])
                    al = e / torch.zeros((n, heads), device=dev).index_add(0, rows, e)[rows]
                    msg = (al[:, :, None] * (Vp[cols] + Ep).view(-1, heads, Cw)).reshape(-1, f)
                    o = torch.zeros((n, f), device=dev).index_add(0, rows, msg)
                    o.backward(g)
                    return o

                try:
                    r["step_torch_native"] = median_ms(step_torch_native, it, wu)
                    r["torch_native_over_fused"] = r["step_torch_native"] / r["step"]
                    o = step_torch_native().detach()
                    nat = {"Z": o, "dQ": leaves[0].grad, "dK": leaves[1].grad, "dV": leaves[2].grad, "dE": leaves[3].grad}
                    fused = {"Z": Z, "dQ": dQ, "dK": dKV[:, :f], "dV": dKV[:, f:], "dE": dE}
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
            del Z, L, dQ, D, dKV, PS, dE, w0, w1, w2
            torch.cuda.empty_cache()
        del Q, K, V, g, E, KV
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
