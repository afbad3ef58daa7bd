"""Graph transformer attention on the H100 path: pgcn_transformer_forward / _backward_rows / _backward_cols,
op.PTransformerAttention and PTRANSFORMER.py.

The fp32 bound. Per entry e = (i, j) and head h of width C, the kernels form the score s = fl(scale fl(<q, k>)): C
products summed on a lane and over a butterfly of at most 32 lanes, then the scale, so s carries at most
sigma_e = (C + 6) 2^-24 scale sum_c |q k| of absolute error, which enters every p = exp(s - .) relatively. The forward
keeps an online softmax: a term's weight exp(s - m) takes one rounding of s - m (|s - m| 2^-24 absolute in the
exponent) and expf's 2 ulp; each later rescale of the running max, at most d of them for a row of d entries, multiplies
it by a rounded expf(m_old - m_new) (2 ulp, one rounding of an argument whose magnitudes add up to at most |s - m|,
one rounding of the product); the sums of the accumulator and of the normaliser take d roundings each; the quotient
one. A chunked row merges its chunks with the same operations. So each normalised weight w = M p carries at most
eps_f = (10 d + C0) 2^-24 + 2 max_e (sigma_e + 2 |s_e - m| 2^-24) relative error, and
    |Z - Z64| <= eps_f sum_e |w_e v_j|,      |L - L64| <= (|m| + 2 |log l|) 2^-24 + eps_f.
The backward's p = expf(s - L) then carries eps_b = sigma_e + tol_L + (|s - L| + C0) 2^-24 relative error; dp =
<gZ, v> and D = <gZ, Z> are dot products of C terms ((C + 6) 2^-24 sum|terms|, and D also the error of Z), and
ds = p (M dp - D) takes a few more roundings. Each gradient element is a sum of d terms (the row's for dQ, the global
column's for dK and dV, whose halo partials add at most k - 1 <= 2 roundings at their owner):
    |dQ - dQ64| <= scale sum_e |k_j| (|ds|' (d + C0) 2^-24 + err(ds_e)),   |ds|' = p (M |dp| + |D|),
dK likewise with |q_i|, and |dV - dV64| <= sum_e M p |gZ_i| (eps_b + (d + C0) 2^-24). tests/transformer_oracle.py
evaluates these per element from fp64 magnitude sums; C0 = CONST below is the one constant, and 1e-30 covers exact
zeros.

  * the forward and the three gradients against fp64 for every valid (f, heads), f in 1 .. 256, heads 1, 2, 4, 8, on
    gemat11, the hub graph (a split row of 3000 entries, empty rows, rows of one entry) and a local plan with
    duplicated entries, with and without dropout (p = 0.3); run-to-run bits; every operand 4 bytes into its buffer (the
    scalar instances) gives the vector instances' bits;
  * the same graph walked with a chunk of 4 stays within the bound;
  * the mask read back through V = I on karate equals tests/dropout_oracle.keep bit for bit; the backward uses the
    forward's counter and the next call draws a new one;
  * +-inf and NaN in q, k or v: NaN and +-inf exactly where the fp32 NumPy restatement has them;
  * torch.profiler, in a process of its own, sees every instance of tests/transformer_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport, with and without dropout, within the bound of the one-rank fp64 result; on
    two GPUs NCCL gives the peer transport's bits;
  * PTransformerAttention's autograd in both layouts on one rank and on three; CUDA-graph capture with dropout on one
    and two ranks, and a capture before the first eager call refused before it enqueues work;
  * the composed path (pgcn_sddmm_heads, a torch softmax, pgcn_forward_heads / pgcn_backward_heads) agrees within the
    bound;
  * PTRANSFORMER.py follows the fp64 loss curve, and the layer on 3 ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import dropout_oracle as do
import transformer_oracle as tro
from harness import (EPS, ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, op, plan as planmod
from pgcn_b200.op import (EdgeDropout, PTransformerAttention, aggregate_transformer, aggregate_transformer_backward,
                          transformer_scale)
from test_max_aggregation import with_duplicates

pytestmark = pytest.mark.gpu
CONST = 16
KEY = 0x0123456789ABCDEF
P = 0.3
FH = [(f, k) for f in (1, 3, 4, 8, 12, 64, 128, 136, 256) for k in (1, 2, 4, 8) if f % k == 0]


def one_rank_plan(case, f):
    """A bound one-rank plan of width 2f on problem(case) ("dup": gemat11 with duplicated entries)."""
    A, _, _ = problem("gemat11_k1" if case == "dup" else case)
    lp = planmod.build_local_plan(A, np.zeros(A.shape[0], dtype=np.int64), 0, 1)
    if case == "dup":
        lp = with_duplicates(lp)
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev())
    plan.bind_values()
    return plan


def inputs(n, f, seed):
    rs = np.random.RandomState(seed)
    return tuple((rs.standard_normal((n, f)) * s).astype(np.float32) for s in (1.5, 1.5, 1.0, 1.0))   # Q, K, V, gZ


def global_entries(lp):
    """(global row, global column) of the local plan's entries."""
    rows, cols = tro.entries(lp.rowptr, lp.colidx)
    return lp.owned[rows], np.concatenate([lp.owned, lp.halo])[cols]


def mask(lp, heads, p, counter):
    return None if p == 0 else do.weights(*global_entries(lp), heads, p, KEY, counter).numpy()


def reference(lp, Q, K, V, gZ, heads, p=0.0, counter=1):
    """{name: (fp64 value, bound)} of a one-rank plan (h = 0) on global inputs."""
    f = Q.shape[1]
    return tro.attention(lp.rowptr, lp.colidx, lp.m, Q, K, V, gZ, heads, transformer_scale(f, heads), CONST,
                         mask(lp, heads, p, counter))


def within(got, ref, what):
    val, tol = ref
    g = got.detach().cpu().numpy().astype(np.float64)
    err = np.abs(g - val)
    bad = ~(err <= tol)
    if np.isneginf(val).any():                      # L of rows without entries: -inf either way
        bad &= ~(np.isneginf(val) & np.isneginf(g))
    assert not bad.any(), "%s: %d elements beyond the fp32 bound, worst err %.3e" % (
        what, int(bad.sum()), float(np.nanmax(np.where(bad, err, 0))))


def run_all(plan, Q, KV, KVh, gZ, f, heads, drop=None, snap=None, walks=None):
    """(Z, L, dQ, D, dKV) from the three C calls, outputs NaN-filled first; walks default to the plan's."""
    fwd, tr = walks or plan.gated_walks()
    lib, lp = cabi.load_transformer(), plan.lp
    gid = plan.global_ids()
    nan = lambda *s: torch.full(s, float("nan"), device=dev())
    Z, L, dQ, D, dKV = nan(lp.m, f), nan(lp.m, heads), nan(lp.m, f), nan(lp.m, heads), nan(lp.m + lp.h, 2 * f)
    w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev())
    w1 = torch.empty((fwd.nslots, f), device=dev())
    w2 = torch.empty((tr.nslots, 2 * f), device=dev())
    hp = KVh.data_ptr() if KVh is not None else None
    sc = transformer_scale(f, heads)
    dargs = (None, 0, 1.0) if drop is None else (snap.data_ptr(), drop.threshold, drop.scale)
    head = (lp.m, lp.h, heads, Q.data_ptr(), KV.data_ptr(), hp, sc, gid.data_ptr()) + dargs
    cabi.check_transformer(lib.pgcn_transformer_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                        w0.data_ptr(), f, stream()))
    cabi.check_transformer(lib.pgcn_transformer_backward_rows(C.byref(fwd.c), *head, gZ.data_ptr(), Z.data_ptr(),
                                                              L.data_ptr(), dQ.data_ptr(), D.data_ptr(), w1.data_ptr(),
                                                              f, stream()))
    cabi.check_transformer(lib.pgcn_transformer_backward_cols(C.byref(tr.c), *head, gZ.data_ptr(), L.data_ptr(),
                                                              D.data_ptr(), dKV.data_ptr(), w2.data_ptr(), f,
                                                              stream()))
    torch.cuda.synchronize()
    return Z, L, dQ, D, dKV


def check_one_rank(plan, ins, f, heads, p=0.0, walks=None, shift=False):
    """Run the three calls on (Q, K, V, gZ) with a fresh draw at counter 1, check every output against fp64."""
    lp = plan.lp
    Qn, Kn, Vn, gn = ins
    ops = [t(Qn), t(np.concatenate([Kn, Vn], 1)), t(gn)]
    if shift:
        ops = [shifted(x) for x in ops]
    Q, KV, gZ = ops
    drop = EdgeDropout(p, KEY, dev()) if p > 0 else None
    snap = drop.draw() if drop else None
    Z, L, dQ, D, dKV = run_all(plan, Q, KV, None, gZ, f, heads, drop, snap, walks)
    ref = reference(lp, Qn, Kn, Vn, gn, heads, p)
    for name, got in (("Z", Z), ("L", L), ("dQ", dQ), ("dK", dKV[:, :f]), ("dV", dKV[:, f:])):
        within(got, ref[name], "%s f=%d heads=%d p=%g" % (name, f, heads, p))
    return Z, L, dQ, D, dKV


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("f,heads", FH)
@pytest.mark.parametrize("case", ["gemat11_k1", "hub", "dup"])
def test_within_fp32_of_fp64_run_to_run_and_scalar_bits(case, f, heads, p):
    if case != "gemat11_k1" and (f, heads) not in ((3, 1), (8, 8), (128, 4), (136, 8), (256, 2)):
        pytest.skip("the hub and duplicate plans run a subset of the widths")
    plan = one_rank_plan(case, f)
    lp = plan.lp
    if case == "hub":
        deg = np.diff(lp.rowptr.astype(np.int64))
        assert deg.max() > cabi.load_gated().pgcn_gated_chunk() and (deg == 0).any() and (deg == 1).any()
        assert plan.gated_walks()[0].nslots > 0
    ins = inputs(lp.m, f, f + heads + len(case))
    first = check_one_rank(plan, ins, f, heads, p)
    again = check_one_rank(plan, ins, f, heads, p)
    scalar = check_one_rank(plan, ins, f, heads, p, shift=True)
    for a, b, s in zip(first, again, scalar):
        assert np.array_equal(bits(a), bits(b)) and np.array_equal(bits(a), bits(s))
    plan.close()


@pytest.mark.parametrize("f,heads", [(4, 1), (5, 1), (64, 4), (136, 8)])
def test_forced_small_chunk_stays_within_the_bound(f, heads):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    ins = inputs(lp.m, f, 9)
    for p in (0.0, P):
        check_one_rank(plan, ins, f, heads, p)
        check_one_rank(plan, ins, f, heads, p, walks=small)
    plan.close()


@pytest.mark.parametrize("heads", [1, 2])
def test_mask_read_back_through_v_identity_equals_the_oracle(heads):
    """V = I on karate (f = n = 34): Z[i, j] = M alpha of entry (i, j) for the head that holds column j, so Z is zero
    exactly where the mask drops."""
    A, _, _ = problem("karate")
    n = f = A.shape[0]
    plan = one_rank_plan("karate", f)
    lp = plan.lp
    rows, cols = tro.entries(lp.rowptr, lp.colidx)
    assert len(set(zip(rows.tolist(), cols.tolist()))) == len(rows)        # no duplicates
    rs = np.random.RandomState(4)
    Q, K = (t(rs.standard_normal((n, f)).astype(np.float32)) for _ in range(2))
    V = torch.eye(n, device=dev())
    drop = EdgeDropout(0.5, KEY, dev())
    Qr, Kr, Vr = (x.clone().requires_grad_(True) for x in (Q, K, V))
    Z = PTransformerAttention.apply(plan, Qr, Kr, Vr, heads, None, drop)
    assert int(drop.state[1]) == 1
    gi, gj = global_entries(lp)
    C = f // heads
    keep = do.keep(gi, gj, heads, 0.5, KEY, 1)
    got = Z.detach().cpu().numpy()[rows, cols] != 0
    assert np.array_equal(got, keep[np.arange(len(rows)), cols // C])
    # the backward draws nothing and uses the forward's counter
    gn = rs.standard_normal((n, f)).astype(np.float32)
    Z.backward(t(gn))
    assert int(drop.state[1]) == 1
    ref = tro.attention(lp.rowptr, lp.colidx, n, Q.cpu().numpy(), K.cpu().numpy(), np.eye(n, dtype=np.float32), gn,
                        heads, transformer_scale(f, heads), CONST, mask(lp, heads, 0.5, 1))
    for name, got in (("dQ", Qr.grad), ("dK", Kr.grad), ("dV", Vr.grad)):
        within(got, ref[name], "%s heads=%d" % (name, heads))
    # a second call draws counter 2
    Z2 = PTransformerAttention.apply(plan, Q, K, V, heads, None, drop)
    assert int(drop.state[1]) == 2
    keep2 = do.keep(gi, gj, heads, 0.5, KEY, 2)
    got2 = Z2.cpu().numpy()[rows, cols] != 0
    assert np.array_equal(got2, keep2[np.arange(len(rows)), cols // C]) and not np.array_equal(got2, got)
    plan.close()


@pytest.mark.parametrize("f,heads", [(5, 1), (8, 2)])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values(case, f, heads):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    Qn, Kn, Vn, gn = inputs(lp.m, f, 3 * f)
    rs = np.random.RandomState(f)
    for x in (Qn, Kn, Vn):
        u = rs.uniform(size=x.shape)
        x[u < 0.004] = np.inf
        x[(u >= 0.004) & (u < 0.008)] = -np.inf
        x[(u >= 0.008) & (u < 0.01)] = np.nan
    Z, L, dQ, _, dKV = run_all(plan, t(Qn), t(np.concatenate([Kn, Vn], 1)), None, t(gn), f, heads)
    fwd = plan.gated_walks()[0]
    ref = tro.fp32_reference(lp.rowptr, lp.colidx, lp.m, Qn, Kn, Vn, gn, heads, transformer_scale(f, heads),
                             fwd.items.cpu().numpy(), fwd.splits.cpu().numpy())
    has = np.diff(lp.rowptr.astype(np.int64)) > 0
    for name, got in (("Z", Z), ("L", L), ("dQ", dQ), ("dK", dKV[:, :f]), ("dV", dKV[:, f:])):
        g, w = got.cpu().numpy(), ref[name]
        if name == "L":
            g, w = g[has], w[has]
        assert np.isnan(w).any(), name
        assert np.array_equal(np.isnan(g), np.isnan(w)), "%s: %d NaN differ" % (name, int((np.isnan(g) != np.isnan(w)).sum()))
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    plan.close()


def key(name):
    """Instance name without return type, parameter list, casts and spaces, bools as 0 / 1: the manifest's and the
    profiler's spellings of one instance give the same key."""
    s = name.strip()
    for a, b in (("(int)", ""), ("(bool)", ""), ("true", "1"), ("false", "0")):
        s = s.replace(a, b)
    if s.startswith("void "):
        s = s[5:]
    return s.split("(")[0].replace(" ", "")


def _instances_worker(rank, k):
    """The keys of the transformer kernels torch.profiler sees while every instance runs (vector and scalar, split
    rows through the delta and fixup kernels), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for f, heads, shift in ((8, 2, False), (6, 2, False), (8, 2, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        walks = (planmod.GatedWalk(lp.rowptr, lp.colidx, 64, dev()),
                 planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 64, dev()))
        assert walks[0].c.nsplits > 0 and walks[1].c.nsplits > 0
        ins = inputs(lp.m, f, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                check_one_rank(plan, ins, f, heads, P, walks=walks, shift=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "transformer_" in e.name}
            if len(names) == 7:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    # in a process of its own: a profiler session leaves the profiler attached to the process, and later sessions in
    # it then lose the records of their first kernels
    with open(os.path.join(ROOT, "tests", "transformer_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


def rank_inputs(lps, arrays):
    return [[t(a[lp.owned]) for a in arrays] for lp in lps]


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("case,f,heads", [("gemat11_k2", 64, 4), ("gemat11_k2", 6, 2), ("gemat11_k3_hp", 16, 1),
                                          ("gemat11_k3_hp", 136, 8)])
def test_multi_rank_within_the_bound_of_one_rank(case, f, heads, p):
    A, pv, k = problem(case)
    n = A.shape[0]
    ins_n = inputs(n, f, f + k)
    one = one_rank_plan(case, f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = rank_inputs(lps, ins_n)
    drops = [EdgeDropout(p, KEY, dev()) for _ in plans]

    def step(r):
        Q, K, V, g = ins[r]
        Z, L, KV, KVh, snap = aggregate_transformer(plans[r], Q, K, V, heads, drop=drops[r])
        return (Z, L) + aggregate_transformer_backward(plans[r], Q, KV, KVh, Z, L, g, heads, drop=drops[r], snap=snap)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs; counters 1 and 2
        ref = reference(one.lp, *ins_n, heads, p, rep + 1)
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "L", "dQ", "dK", "dV"), out[r]):
                val, tol = ref[name]
                within(got, (val[lp.owned], tol[lp.owned]), "%s %s rank %d rep %d" % (case, name, r, rep))
        if first is None:
            first = [[bits(x) for x in o] for o in out]
        elif p == 0:
            assert all(np.array_equal(a, bits(b)) for fo, o in zip(first, out) for a, b in zip(fo, o))
    for p_ in plans + [one]:
        p_.close()


def _nccl_worker(rank, k, port, transport):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=k, device_id=torch.device("cuda", rank))
    A, pv, _ = problem("gemat11_k2")
    n, f = A.shape[0], 64
    p = planmod.build_plan(A, pv, rank, k, 2 * f, device=torch.device("cuda", rank))
    used = p.init_comm(transport=transport)
    p.bind_values()
    own = p.lp.owned
    Q, K, V, g = (torch.from_numpy(a[own]).cuda().requires_grad_(True) for a in inputs(n, f, 1))
    Z = PTransformerAttention.apply(p, Q, K, V, 4, None, EdgeDropout(P, KEY, torch.device("cuda", rank)))
    Z.backward(g.detach())
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), Q.grad, K.grad, V.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29881, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29882, "p2p"))
    for r in range(2):
        assert a[r][0] == "nccl" and b[r][0] == "p2p"
        for x, y in zip(a[r][1], b[r][1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("layout", ["local", "global"])
def test_autograd_one_rank(layout):
    f, heads = 32, 4
    plan = one_rank_plan("hub", f)
    plan.layout = layout
    lp = plan.lp
    Qn, Kn, Vn, gn = inputs(lp.m, f, 4)
    Q, K, V = (t(a).requires_grad_(True) for a in (Qn, Kn, Vn))
    Z = PTransformerAttention.apply(plan, Q, K, V, heads)
    Z.backward(t(gn))
    ref = reference(lp, Qn, Kn, Vn, gn, heads)
    for name, got in (("Z", Z), ("dQ", Q.grad), ("dK", K.grad), ("dV", V.grad)):
        within(got, ref[name], "%s %s" % (layout, name))
    plan.close()


def test_autograd_three_ranks_and_global_layout():
    A, pv, k = problem("gemat11_k3_hp")
    n, f, heads = A.shape[0], 16, 2
    ins_n = inputs(n, f, 3)
    one = one_rank_plan("gemat11_k3_hp", f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    for counter, layout in enumerate(("local", "global"), 1):
        ref = reference(one.lp, *ins_n, heads, P, counter)
        for p in plans:
            p.layout = layout
        if counter == 1:
            drops = [EdgeDropout(P, KEY, dev()) for _ in plans]
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [[t(pick(a, lp)).requires_grad_(True) for a in ins_n[:3]] for lp in lps]
        Z = run_ranks(plans, lambda r: PTransformerAttention.apply(plans[r], *leaves[r], heads, None, drops[r]),
                      streams)
        run_ranks(plans, lambda r: Z[r].backward(t(pick(ins_n[3], lps[r]))), streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "dQ", "dK", "dV"), [Z[r]] + [x.grad for x in leaves[r]]):
                val, tol = ref[name]
                if layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                    within(got, (val, tol), "global %s rank %d" % (name, r))
                else:
                    within(got, (val[lp.owned], tol[lp.owned]), "local %s rank %d" % (name, r))
    for p in plans + [one]:
        p.close()


def follower(drop):
    """A second EdgeDropout whose next use draws with the counter `drop` used last."""
    ref = EdgeDropout(drop.p, KEY, dev())
    ref.state.copy_(drop.state)
    ref.state[1:].sub_(1)
    return ref


def test_one_rank_capture_with_dropout_and_refusal_before_the_first_eager_call():
    f, heads = 64, 4
    plan = one_rank_plan("hub", f)
    m = plan.lp.m
    Q, K, V, g = (torch.zeros((m, f), device=dev()) for _ in range(4))
    drop = EdgeDropout(P, KEY, dev())

    def step(Q, K, V, g, drop):
        Z, L, KV, KVh, snap = aggregate_transformer(plan, Q, K, V, heads, drop=drop)
        dQ, dK, dV = aggregate_transformer_backward(plan, Q, KV, KVh, Z, L, g, heads, drop=drop, snap=snap)
        return dict(Z=Z, L=L, dQ=dQ, dK=dK, dV=dV)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    with pytest.raises(RuntimeError, match="gated_walks"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(Q, K, V, g, drop)
    assert plan.launch_count() == launches and plan._gated_walks is None and int(drop.state[1]) == 0
    ins = [tuple(t(a) for a in inputs(m, f, 20 + i)) for i in range(3)]

    def load(i):
        for dst, src in zip((Q, K, V, g), ins[i]):
            dst.copy_(src)

    plan.prepare(2 * f)
    step(*ins[0], None)                                   # the first eager call builds the walks and the ids
    check_one_rank_capture(plan, lambda: step(Q, K, V, g, drop), load, lambda i: step(*ins[i], follower(drop)))
    assert int(drop.state[1]) == 4                        # one draw per replay, none at capture
    plan.close()


def test_global_ids_capture_is_refused():
    plan = one_rank_plan("hub", 8)
    plan.gated_walks()
    with pytest.raises(RuntimeError, match="global_ids"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=torch.cuda.Stream()):
            plan.global_ids()
    ids = plan.global_ids().cpu().numpy()
    assert ids.dtype == np.int32 and np.array_equal(ids, np.concatenate([plan.lp.owned, plan.lp.halo]))
    plan.close()


def test_two_rank_capture_with_dropout_over_the_peer_transport():
    A, pv, k = problem("gemat11_k2")
    f, n, heads = 64, A.shape[0], 2
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    for p in plans:
        p.prepare(2 * f)
        p.gated_walks()
        p.global_ids()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, f, 30 + i) for i in range(3)]
    made = []

    def buffers(r):
        b = {name: torch.zeros((lps[r].m, f), device=dev()) for name in ("x", "k", "v", "g")}
        b["drop"] = EdgeDropout(P, KEY, dev())
        made.append(b)
        return b

    def load(bufs, i):
        for r, lp in enumerate(lps):
            for name, a in zip(("x", "k", "v", "g"), ins[i]):
                bufs[r][name].copy_(t(a[lp.owned]))
            if bufs[r] is not made[r]:                    # eager buffers draw with the counter the replay just used
                bufs[r]["drop"] = follower(made[r]["drop"])
        torch.cuda.synchronize()

    def step(r, b):
        Z, L, KV, KVh, snap = aggregate_transformer(plans[r], b["x"], b["k"], b["v"], heads, drop=b["drop"])
        dQ, dK, dV = aggregate_transformer_backward(plans[r], b["x"], KV, KVh, Z, L, b["g"], heads, drop=b["drop"],
                                                    snap=snap)
        return dict(Z=Z, dQ=dQ, dK=dK, dV=dV)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for r in range(k):
        assert int(made[r]["drop"].state[1]) == 4
    for p in plans:
        p.close()


@pytest.mark.parametrize("f,heads", [(64, 4), (128, 8), (24, 1)])
def test_composed_path_agrees_within_the_bound(f, heads):
    """pgcn_sddmm_heads for the scores, a torch softmax per row, pgcn_forward_heads / pgcn_backward_heads for the
    aggregation and dV, pgcn_sddmm_heads again for dalpha: an independent GPU implementation of the same layer."""
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    Qn, Kn, Vn, gn = inputs(lp.m, f, 77)
    ref = reference(lp, Qn, Kn, Vn, gn, heads)
    Q, K, V, g = (t(a) for a in (Qn, Kn, Vn, gn))
    rows = torch.from_numpy(tro.entries(lp.rowptr, lp.colidx)[0]).to(dev())
    sc = transformer_scale(f, heads)
    C_ = f // heads
    nnz = lp.nnz()
    S = torch.empty((nnz, heads), device=dev())
    op._call(plan, dev(), "pgcn_sddmm_heads", heads, Q.data_ptr(), K.data_ptr(), None, S.data_ptr(), f)
    S = S * sc
    mx = torch.full((lp.m, heads), -float("inf"), device=dev()).scatter_reduce(0, rows[:, None].expand(-1, heads), S,
                                                                               "amax")
    e = torch.exp(S - mx[rows])
    den = torch.zeros((lp.m, heads), device=dev()).index_add(0, rows, e)
    alpha = (e / den[rows]).contiguous()
    Z = torch.empty((lp.m, f), device=dev())
    op._call(plan, dev(), "pgcn_forward_heads", heads, alpha.data_ptr(), V.data_ptr(), Z.data_ptr(), None, f)
    dV = torch.empty((lp.m, f), device=dev())
    op._call(plan, dev(), "pgcn_backward_heads", heads, alpha.data_ptr(), g.data_ptr(), dV.data_ptr(), f)
    dalpha = torch.empty((nnz, heads), device=dev())
    op._call(plan, dev(), "pgcn_sddmm_heads", heads, g.data_ptr(), V.data_ptr(), None, dalpha.data_ptr(), f)
    D = torch.zeros((lp.m, heads), device=dev()).index_add(0, rows, alpha * dalpha)
    ds = (alpha * (dalpha - D[rows])).contiguous()
    dQ = torch.empty((lp.m, f), device=dev())
    op._call(plan, dev(), "pgcn_forward_heads", heads, ds.data_ptr(), K.data_ptr(), dQ.data_ptr(), None, f)
    dK = torch.empty((lp.m, f), device=dev())
    op._call(plan, dev(), "pgcn_backward_heads", heads, ds.data_ptr(), Q.data_ptr(), dK.data_ptr(), f)
    dQ, dK = dQ * sc, dK * sc
    torch.cuda.synchronize()
    fused = run_all(plan, Q, torch.cat([K, V], 1), None, g, f, heads)
    # both lie within the bound of fp64, so within twice the bound of each other
    for name, comp, fu in (("Z", Z, fused[0]), ("dQ", dQ, fused[2]), ("dK", dK, fused[4][:, :f]),
                           ("dV", dV, fused[4][:, f:])):
        val, tol = ref[name]
        within(comp, (val, 4 * tol), "composed %s" % name)
        within(fu, (comp.detach().cpu().numpy().astype(np.float64), 5 * tol), "fused vs composed %s" % name)
    plan.close()


def test_cli_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PTRANSFORMER.py", ["--heads", "2"], 29791)
    assert_follows(lines, tro.intended_training(karate(), 2, 4, 7, heads=2))


def test_cli_attn_dropout_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PTRANSFORMER.py", ["--attn-dropout", "0.5"], 29792)
    assert_follows(lines, tro.intended_training(karate(), 2, 4, 7, p=0.5))


def test_layer_on_three_ranks_follows_the_one_rank_curve():
    """transformer.run's training loop with the three ranks of karate_k3 in this process (peer transport), against the
    same loop on one rank and against the fp64 oracle with gradients averaged over three ranks."""
    import torch.nn as nn
    import torch.nn.functional as F
    from pgcn_b200.transformer import PTRANSFORMER
    A, pv, k = problem("karate")
    n, f, L, epochs, heads = A.shape[0], 4, 2, 50, 2

    def train(plans, lps):
        kk = len(plans)
        streams = [torch.cuda.Stream(device=dev()) for _ in plans]
        models, opts = [], []
        for p in plans:
            torch.manual_seed(7)
            m = nn.Sequential(*[PTRANSFORMER(p, f, f, heads) for _ in range(L)]).to(dev())
            models.append(m)
            opts.append(torch.optim.Adam(m.parameters(), lr=1e-3))
        H = [t(np.repeat(lp.owned.astype(np.float32)[:, None], f, axis=1)) for lp in lps]
        y = [torch.from_numpy(lp.owned % f).to(dev()) for lp in lps]
        losses = []
        for _ in range(epochs):
            logits = run_ranks(plans, lambda r: models[r](H[r]), streams)
            loss = [F.nll_loss(F.log_softmax(logits[r], 1), y[r], reduction="sum") / n for r in range(kk)]
            for o in opts:
                o.zero_grad()
            run_ranks(plans, lambda r: loss[r].backward(), streams)
            with torch.no_grad():
                for ps in zip(*[m.parameters() for m in models]):
                    avg = sum(q.grad for q in ps) / kk
                    for q in ps:
                        q.grad.copy_(avg)
            for o in opts:
                o.step()
            losses.append(float(sum(float(x) for x in loss)))
        return losses

    lp1 = [planmod.build_local_plan(A, np.zeros(n, dtype=np.int64), 0, 1)]
    one = [planmod.PgcnPlan(lp1[0], 2 * f, device=dev())]
    one[0].bind_values()
    curve1 = train(one, lp1)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    curve3 = train(plans, lps)
    np.testing.assert_allclose(curve1, tro.intended_training(A, L, f, 7, heads=heads), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, tro.intended_training(A, L, f, 7, k=3, heads=heads), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
    for p in plans + one:
        p.close()
