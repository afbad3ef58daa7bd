"""Graph transformer attention on C2 (R-MAT 1 M vertices / 16 M edges + self loops, f = 128), one GPU, heads K in
{1, 4, 8}: what the three fused kernels cost, next to the composed path of existing kernels, a PyTorch-native
TransformerConv step and, for context, the gated step.

    python tools/bench_transformer.py [--iters 30] [--warmup 10] [--config C2] [--heads 1,4,8] [--no-torch]

Reports, per K, the median over `iters` calls (CUDA events, after `warmup` untimed calls) of
  forward / backward_rows / backward_cols   pgcn_transformer_forward, _backward_rows, _backward_cols
  step                                      the three in a row (forward + backward)
  step_p01                                  the same with attention dropout p = 0.1 (the mask drawn inline)
  step_composed                             pgcn_sddmm_heads (scores), a torch scatter softmax, pgcn_forward_heads
                                            (Z); pgcn_backward_heads (dV), pgcn_sddmm_heads (dalpha), the torch softmax
                                            backward, pgcn_forward_heads / pgcn_backward_heads (dQ, dK)
  step_torch_native                         gathers q[row], k[col], v[col], a scatter softmax, index_add_, autograd
and once the gated step (pgcn_gated_forward + both backward walks at f). The byte model (DESIGN.md §4): the forward
gathers 4 B of index + 8f B ([k | v]) per entry and reads 4f B of q and writes 4f B of Z per row; the row walk adds 4f
B of gZ and 4f B of Z per row; the column walk gathers 8f B (q and gZ) + 8K B (L and D) per transposed entry and reads
and writes 8f B per column. The native step's output and gradients are checked against the fused kernels' within twice
the fp32 bound of tests/test_transformer_attention.py, with the magnitudes evaluated in fp32 on the device. Prints
the card's name and power limit read in the same run, then one JSON line.
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

EPS = 2.0 ** -24
CONST = 16


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
    from pgcn_b200 import cabi, graphio, op, plan as planmod
    if not torch.cuda.is_available():
        raise SystemExit("bench_transformer.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, _, f, _, _ = graphio.CONFIGS[args.config]
    A = graphio.config_graph(args.config, cache_dir=args.cache)
    lp = planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)
    del A
    nnz = lp.nnz()
    deg = np.diff(lp.rowptr.astype(np.int64))
    cdeg = np.diff(lp.t_rowptr.astype(np.int64))
    plan = planmod.PgcnPlan(lp, max(2 * f, 32), device=dev)
    plan.bind_values()
    fwd, tr = plan.gated_walks()
    gid = plan.global_ids()
    tlib, glib = cabi.load_transformer(), cabi.load_gated()
    st = lambda: torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    Q, K, V, g = ((torch.randn((n, f), device=dev, generator=gen) * s) for s in (1.5, 1.5, 1.0, 1.0))
    KV = torch.cat([K, V], 1)
    rows = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    cols = torch.from_numpy(lp.colidx.astype(np.int64)).to(dev)
    d_r = torch.from_numpy(deg.astype(np.float32)).to(dev)
    d_c = torch.from_numpy(cdeg[:n].astype(np.float32)).to(dev)
    chk = cabi.check_transformer
    res, rates, check = {}, {}, {}

    # the gated step at the same width, for context
    Z0, dK0, dQV0 = torch.empty((n, f), device=dev), torch.empty((n, f), device=dev), torch.empty((n, 2 * f), device=dev)
    gw1, gw2 = torch.empty((fwd.nslots, f), device=dev), torch.empty((tr.nslots, 2 * f), device=dev)

    def gated_step():
        cabi.check_gated(glib.pgcn_gated_forward(C.byref(fwd.c), n, 0, K.data_ptr(), KV.data_ptr(), None,
                                                 Z0.data_ptr(), gw1.data_ptr(), f, st()))
        cabi.check_gated(glib.pgcn_gated_backward_rows(C.byref(fwd.c), n, 0, K.data_ptr(), KV.data_ptr(), None,
                                                       g.data_ptr(), dK0.data_ptr(), gw1.data_ptr(), f, st()))
        cabi.check_gated(glib.pgcn_gated_backward_cols(C.byref(tr.c), n, 0, K.data_ptr(), KV.data_ptr(), None,
                                                       g.data_ptr(), dQV0.data_ptr(), gw2.data_ptr(), f, st()))

    res["gated_forward"] = median_ms(lambda: cabi.check_gated(glib.pgcn_gated_forward(
        C.byref(fwd.c), n, 0, K.data_ptr(), KV.data_ptr(), None, Z0.data_ptr(), gw1.data_ptr(), f, st())),
        args.iters, args.warmup)
    res["gated_step"] = median_ms(gated_step, args.iters, args.warmup)
    del Z0, dK0, dQV0, gw1, gw2

    for heads in [int(x) for x in args.heads.split(",")]:
        sc = op.transformer_scale(f, heads)
        Cw = f // heads
        Z, L, dQ, D = (torch.empty(s, device=dev) for s in ((n, f), (n, heads), (n, f), (n, heads)))
        dKV = torch.empty((n, 2 * f), device=dev)
        w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev)
        w1, w2 = torch.empty((fwd.nslots, f), device=dev), torch.empty((tr.nslots, 2 * f), device=dev)
        drop = op.EdgeDropout(0.1, 12345, dev)

        def calls(dargs):
            head = (n, 0, heads, Q.data_ptr(), KV.data_ptr(), None, sc, gid.data_ptr()) + dargs
            return (lambda: chk(tlib.pgcn_transformer_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                              w0.data_ptr(), f, st())),
                    lambda: chk(tlib.pgcn_transformer_backward_rows(C.byref(fwd.c), *head, g.data_ptr(), Z.data_ptr(),
                                                                    L.data_ptr(), dQ.data_ptr(), D.data_ptr(),
                                                                    w1.data_ptr(), f, st())),
                    lambda: chk(tlib.pgcn_transformer_backward_cols(C.byref(tr.c), *head, g.data_ptr(), L.data_ptr(),
                                                                    D.data_ptr(), dKV.data_ptr(), w2.data_ptr(), f,
                                                                    st())))

        fw, rw, cw = calls((None, 0, 1.0))
        r = {"forward": median_ms(fw, args.iters, args.warmup), "backward_rows": median_ms(rw, args.iters, args.warmup),
             "backward_cols": median_ms(cw, args.iters, args.warmup)}
        r["step"] = median_ms(lambda: (fw(), rw(), cw()), args.iters, args.warmup)
        snap = drop.draw()
        dfw, drw, dcw = calls((snap.data_ptr(), drop.threshold, drop.scale))
        r["step_p01"] = median_ms(lambda: (dfw(), drw(), dcw()), args.iters, args.warmup)
        r["p01_over_p0"] = r["step_p01"] / r["step"]
        r["forward_over_gated_forward"] = r["forward"] / res["gated_forward"]
        fw(), rw(), cw()                                  # the outputs at p = 0, kept for the checks
        torch.cuda.synchronize()
        bytes_ = {"forward": nnz * (4 + 8 * f) + n * 8 * f, "backward_rows": nnz * (4 + 8 * f) + n * 16 * f,
                  "backward_cols": nnz * (4 + 8 * f + 8 * heads) + n * 16 * f}
        rates[heads] = {name + "_gbps": b / r[name] / 1e6 for name, b in bytes_.items()}

        # the composed path
        S, dal = torch.empty((nnz, heads), device=dev), torch.empty((nnz, heads), device=dev)
        Zc, dQc, dKc, dVc = (torch.empty((n, f), device=dev) for _ in range(4))
        idx = rows[:, None].expand(-1, heads)

        def composed():
            op._call(plan, dev, "pgcn_sddmm_heads", heads, Q.data_ptr(), K.data_ptr(), None, S.data_ptr(), f)
            s = S * sc
            mx = torch.full((n, heads), -float("inf"), device=dev).scatter_reduce(0, idx, s, "amax")
            e = torch.exp(s - mx[rows])
            al = (e / torch.zeros((n, heads), device=dev).index_add_(0, rows, e)[rows]).contiguous()
            op._call(plan, dev, "pgcn_forward_heads", heads, al.data_ptr(), V.data_ptr(), Zc.data_ptr(), None, f)
            op._call(plan, dev, "pgcn_backward_heads", heads, al.data_ptr(), g.data_ptr(), dVc.data_ptr(), f)
            op._call(plan, dev, "pgcn_sddmm_heads", heads, g.data_ptr(), V.data_ptr(), None, dal.data_ptr(), f)
            ds = al * dal
            ds = (ds - al * torch.zeros((n, heads), device=dev).index_add_(0, rows, ds)[rows]).contiguous()
            op._call(plan, dev, "pgcn_forward_heads", heads, ds.data_ptr(), K.data_ptr(), dQc.data_ptr(), None, f)
            op._call(plan, dev, "pgcn_backward_heads", heads, ds.data_ptr(), Q.data_ptr(), dKc.data_ptr(), f)
            dQc.mul_(sc)
            dKc.mul_(sc)

        r["step_composed"] = median_ms(composed, args.iters, args.warmup)
        r["composed_over_fused"] = r["step_composed"] / r["step"]
        del S, dal

        # the fp32 bound of the tests, magnitudes on the device in fp32: per entry the score error sigma, the row's
        # envelope ef, the backward's p error eb
        with torch.no_grad():
            qh, kh = Q[rows].view(-1, heads, Cw), K[cols].view(-1, heads, Cw)
            s = (qh * kh).sum(2) * sc
            sig = (Cw + 6) * EPS * sc * (qh * kh).abs().sum(2)
            del qh, kh
            mx = torch.full((n, heads), -float("inf"), device=dev).scatter_reduce(0, idx, s, "amax")
            E = torch.zeros((n, heads), device=dev).scatter_reduce(0, idx, sig + 2 * (s - mx[rows]).abs() * EPS,
                                                                   "amax")
            ef = (10 * d_r[:, None] + CONST) * EPS + 2 * E
            p = torch.exp(s - L[rows])
            eb = sig + (ef + (mx.abs() + 2 * (L - mx).abs()) * EPS)[rows] + ((s - L[rows]).abs() + CONST) * EPS
            del s, sig
            ex = lambda x: x.repeat_interleave(Cw, 1)
            vh = V[cols]
            mags = {"Z": torch.zeros((n, f), device=dev).index_add_(0, rows, ex(p) * vh.abs()) * ex(ef)}
            gv = (g[rows] * vh).view(-1, heads, Cw)
            del vh
            dp, adp = gv.sum(2), gv.abs().sum(2)
            del gv
            # D = <gZ, Z>: its dot-product error and the error Z carries
            dD = ((Cw + 6) * EPS * (g * Z).abs() + g.abs() * mags["Z"]).view(n, heads, Cw).sum(2)
            mds = p * (dp.abs() + D[rows].abs())
            e_ds = ex(mds * eb + p * ((Cw + 6) * EPS * adp + dD[rows]))
            del dp, adp
            mags["dQ"] = sc * torch.zeros((n, f), device=dev).index_add_(
                0, rows, K[cols].abs() * (e_ds + ex(mds) * (d_r[rows, None] + CONST) * EPS))
            mags["dK"] = sc * torch.zeros((n, f), device=dev).index_add_(
                0, cols, Q[rows].abs() * (e_ds + ex(mds) * (d_c[cols, None] + CONST) * EPS))
            del e_ds, mds
            mags["dV"] = torch.zeros((n, f), device=dev).index_add_(
                0, cols, g[rows].abs() * ex(p * (eb + (d_c[cols, None] + CONST) * EPS)))
            del p, eb
        fused = {"Z": Z, "dQ": dQ, "dK": dKV[:, :f], "dV": dKV[:, f:]}
        comp = {"Z": Zc, "dQ": dQc, "dK": dKc, "dV": dVc}
        ck = {}
        for name in fused:
            err = (comp[name] - fused[name]).abs()
            ck["composed_" + name + "_within_2x_bound"] = bool((err <= 2 * mags[name] + 1e-30).all())
        del Zc, dQc, dKc, dVc
        torch.cuda.empty_cache()

        if not args.no_torch:
            leaves = [x.clone().requires_grad_(True) for x in (Q, K, V)]

            def step_torch_native():
                for u in leaves:
                    u.grad = None
                Qp, Kp, Vp = leaves
                s = (Qp[rows].view(-1, heads, Cw) * Kp[cols].view(-1, heads, Cw)).sum(2) * sc
                mx = torch.full((n, heads), -float("inf"), device=dev).scatter_reduce(0, idx, s.detach(), "amax")
                e = torch.exp(s - mx[rows])
                al = e / torch.zeros((n, heads), device=dev).index_add(0, rows, e)[rows]
                msg = (al[:, :, None] * Vp[cols].view(-1, heads, Cw)).reshape(-1, f)
                o = torch.zeros((n, f), device=dev).index_add(0, rows, msg)
                o.backward(g)
                return o

            try:
                r["step_torch_native"] = median_ms(step_torch_native, args.iters, args.warmup)
                r["torch_native_over_fused"] = r["step_torch_native"] / r["step"]
                o = step_torch_native().detach()
                nat = {"Z": o, "dQ": leaves[0].grad, "dK": leaves[1].grad, "dV": leaves[2].grad}
                for name in fused:
                    err = (nat[name] - fused[name]).abs()
                    ck["native_" + name + "_max_rel_diff"] = float(err.max() / (nat[name].abs().max() + 1e-30))
                    ck["native_" + name + "_within_2x_bound"] = bool((err <= 2 * mags[name] + 1e-30).all())
                del o, nat
            except RuntimeError as e:                  # report, do not hide
                r["step_torch_native"] = None
                r["step_torch_native_error"] = str(e)[:300]
            del leaves
            torch.cuda.empty_cache()
        res[heads] = r
        check[heads] = ck
        del mags, Z, L, dQ, D, dKV, w0, w1, w2
        torch.cuda.empty_cache()

    result = {"config": args.config, "n": n, "nnz": nnz, "f": f, "max_row": int(deg.max()), "max_col": int(cdeg.max()),
              "split_rows": int(fwd.c.nsplits), "split_cols": int(tr.c.nsplits), "iters": args.iters,
              "warmup": args.warmup, "card": card(), "ms": res, "gbps": rates, "check": check}
    for k_, v_ in res.items():
        if isinstance(v_, dict):
            for a, b in list(v_.items()) + list(rates[k_].items()) + list(check[k_].items()):
                print("K=%d %-32s %s" % (k_, a, ("%.4g" % b) if isinstance(b, float) else b))
        else:
            print("%-38s %.4g" % (k_, v_))
    print("card: %s, power limit %s W" % (result["card"]["name"], result["card"]["power_limit_w"]))
    print(json.dumps(result))
    plan.close()


if __name__ == "__main__":
    main()
