"""Graph transformer attention with edge features on the H100 path: pgcn_transformer_edge_forward / _backward_rows /
_backward_cols, op.PTransformerEdgeAttention and PTRANSFORMER.py --edge-values.

The fp32 bound is tests/test_transformer_attention.py's, with the roundings of k + E and v + E added
(tests/transformer_edge_oracle.py), and CONST = 16 as there.

  * the forward, the three node gradients and dE against fp64 for the transformer tests' (f, heads), on gemat11, the hub
    graph and a plan with duplicated entries, with and without dropout (p = 0.3); run-to-run bits; E 4 bytes into its
    buffer (the scalar instances) gives the vector instances' bits; without dE every other output keeps its bits;
  * the same graph walked with a chunk of 4 stays within the bound;
  * with E = 0, Z, L, dQ, dK and dV equal op.aggregate_transformer's (torch.equal), with and without dropout;
  * +-inf and NaN in E: NaN and +-inf exactly where the fp32 NumPy restatement has them;
  * a graph with nnz * f > 2^31;
  * torch.profiler, in a process of its own, sees every instance of tests/transformer_edge_kernel_instances.txt;
  * 2 and 3 ranks over the peer transport, with and without dropout, within the bound of the one-rank fp64 result; on
    two GPUs NCCL gives the peer transport's bits;
  * PTransformerEdgeAttention's autograd in both layouts on one rank and on three; E without a gradient; CUDA-graph
    capture with dropout on one and two ranks, and a capture before the first eager call refused before it enqueues
    work;
  * PTRANSFORMER.py --edge-values follows the fp64 loss curve (with --heads 2, with --attn-dropout), and the layer on 3
    ranks follows the one-rank curve.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import transformer_edge_oracle as teo
import transformer_oracle as tro
from harness import (ROOT, assert_follows, bits, check_one_rank_capture, check_two_rank_capture, dev, karate,
                     linked_plans, problem, run_cli, run_ranks, shifted, spawn_ranks, stream, t)
from pgcn_b200 import cabi, plan as planmod
from pgcn_b200.op import (EdgeDropout, PTransformerEdgeAttention, aggregate_transformer,
                          aggregate_transformer_backward, aggregate_transformer_edge,
                          aggregate_transformer_edge_backward, transformer_scale)
from test_gatedgcn import edge_rows
from test_transformer_attention import (FH, follower, global_entries, inputs, key, mask, one_rank_plan, within)

pytestmark = pytest.mark.gpu
CONST = 16
KEY = 0x0123456789ABCDEF
P = 0.3


def edge_term(lp, f):
    """E of the local entries as a function of their global (row, column) and feature, so that every partition of a
    graph gives each entry the same E (duplicated entries share it)."""
    gi, gj = global_entries(lp)
    c = np.arange(f)
    return (np.sin(0.37 * gi[:, None] + 1.13 * gj[:, None] + 0.71 * c) * 0.8).astype(np.float32)


def reference(lp, Q, K, V, E, gZ, heads, p=0.0, counter=1):
    """{name: (fp64 value, bound)} of a one-rank plan (h = 0) on global inputs."""
    f = Q.shape[1]
    return teo.attention(lp.rowptr, lp.colidx, lp.m, Q, K, V, E, gZ, heads, transformer_scale(f, heads), CONST,
                         mask(lp, heads, p, counter))


def run_all(plan, Q, KV, E, gZ, f, heads, drop=None, snap=None, walks=None, with_dE=True):
    """(Z, L, dQ, D, dKV, PS, dE) from the three C calls, outputs NaN-filled first; walks default to the plan's."""
    fwd, tr = walks or plan.gated_walks()
    perm = plan.transposed_entries()
    lib, lp = cabi.load_transformer_edge(), plan.lp
    cabi.check_transformer_edge(lib.pgcn_transformer_edge_load())
    gid = plan.global_ids()
    nan = lambda *s: torch.full(s, float("nan"), device=dev())
    Z, L, dQ, D, dKV = nan(lp.m, f), nan(lp.m, heads), nan(lp.m, f), nan(lp.m, heads), nan(lp.m + lp.h, 2 * f)
    PS = nan(lp.nnz(), 2 * heads)
    dE = nan(lp.nnz(), f) if with_dE else None
    w0 = torch.empty((fwd.nslots, f + 2 * heads), device=dev())
    w1 = torch.empty((fwd.nslots, f), device=dev())
    w2 = torch.empty((tr.nslots, 2 * f), device=dev())
    sc = transformer_scale(f, heads)
    dargs = (None, 0, 1.0) if drop is None else (snap.data_ptr(), drop.threshold, drop.scale)
    head = (lp.m, lp.h, heads, Q.data_ptr(), KV.data_ptr(), None, E.data_ptr(), sc, gid.data_ptr()) + dargs
    cabi.check_transformer_edge(lib.pgcn_transformer_edge_forward(C.byref(fwd.c), *head, Z.data_ptr(), L.data_ptr(),
                                                                  w0.data_ptr(), f, stream()))
    cabi.check_transformer_edge(lib.pgcn_transformer_edge_backward_rows(
        C.byref(fwd.c), *head, gZ.data_ptr(), Z.data_ptr(), L.data_ptr(), dQ.data_ptr(), D.data_ptr(), PS.data_ptr(),
        None if dE is None else dE.data_ptr(), w1.data_ptr(), f, stream()))
    cabi.check_transformer_edge(lib.pgcn_transformer_edge_backward_cols(
        C.byref(tr.c), perm.data_ptr(), lp.m, lp.h, heads, Q.data_ptr(), gZ.data_ptr(), PS.data_ptr(), sc,
        dKV.data_ptr(), w2.data_ptr(), f, stream()))
    torch.cuda.synchronize()
    return Z, L, dQ, D, dKV, PS, dE


NAMES = ("Z", "L", "dQ", "D", "dK|dV", "PS", "dE")


def check_one_rank(plan, ins, En, f, heads, p=0.0, walks=None, shift_E=False, with_dE=True):
    """Run the three calls on (Q, K, V, gZ) and E with a fresh draw at counter 1, check every output against fp64."""
    lp = plan.lp
    Qn, Kn, Vn, gn = ins
    Q, KV, gZ, E = t(Qn), t(np.concatenate([Kn, Vn], 1)), t(gn), t(En)
    if shift_E:
        E = shifted(E)
    drop = EdgeDropout(p, KEY, dev()) if p > 0 else None
    snap = drop.draw() if drop else None
    out = run_all(plan, Q, KV, E, gZ, f, heads, drop, snap, walks, with_dE)
    Z, L, dQ, D, dKV, PS, dE = out
    ref = reference(lp, Qn, Kn, Vn, En, gn, heads, p)
    checks = [("Z", Z), ("L", L), ("dQ", dQ), ("dK", dKV[:, :f]), ("dV", dKV[:, f:])] + ([("dE", dE)] if with_dE
                                                                                          else [])
    for name, got in checks:
        within(got, ref[name], "%s f=%d heads=%d p=%g" % (name, f, heads, p))
    return out


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
    En = edge_term(lp, f)
    first = check_one_rank(plan, ins, En, f, heads, p)
    again = check_one_rank(plan, ins, En, f, heads, p)
    scalar = check_one_rank(plan, ins, En, f, heads, p, shift_E=True)
    for name, a, b, s in zip(NAMES, first, again, scalar):
        assert np.array_equal(bits(a), bits(b)) and np.array_equal(bits(a), bits(s)), name
    no_dE = check_one_rank(plan, ins, En, f, heads, p, with_dE=False)
    for name, a, b in zip(NAMES[:-1], first, no_dE):
        assert np.array_equal(bits(a), bits(b)), name
    plan.close()


@pytest.mark.parametrize("f,heads", [(4, 1), (5, 1), (64, 4), (136, 8)])
def test_forced_small_chunk_stays_within_the_bound(f, heads):
    plan = one_rank_plan("gemat11_k1", f)
    lp = plan.lp
    small = (planmod.GatedWalk(lp.rowptr, lp.colidx, 4, dev()), planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 4, dev()))
    assert small[0].nslots > 0 and small[1].nslots > 0
    ins = inputs(lp.m, f, 9)
    En = edge_term(lp, f)
    for p in (0.0, P):
        check_one_rank(plan, ins, En, f, heads, p)
        check_one_rank(plan, ins, En, f, heads, p, walks=small)
    plan.close()


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("case,f,heads", [("gemat11_k1", 64, 4), ("gemat11_k1", 6, 2), ("hub", 136, 8),
                                          ("dup", 24, 1)])
def test_zero_edge_term_gives_the_attention_without_edges(case, f, heads, p):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    Q, K, V, g = (t(a) for a in inputs(lp.m, f, 41))
    E = torch.zeros((lp.nnz(), f), device=dev())
    d0, d1 = (EdgeDropout(p, KEY, dev()) for _ in range(2))
    Z0, L0, KV0, KVh0, s0 = aggregate_transformer(plan, Q, K, V, heads, drop=d0)
    grads0 = aggregate_transformer_backward(plan, Q, KV0, KVh0, Z0, L0, g, heads, drop=d0, snap=s0)
    Z1, L1, KV1, KVh1, s1 = aggregate_transformer_edge(plan, Q, K, V, E, heads, drop=d1)
    grads1 = aggregate_transformer_edge_backward(plan, Q, KV1, KVh1, E, Z1, L1, g, heads, drop=d1, snap=s1)
    for name, a, b in zip(("Z", "L", "dQ", "dK", "dV"), (Z0, L0) + grads0, (Z1, L1) + grads1[:3]):
        assert torch.equal(a, b), name
    assert int(d0.state[1]) == int(d1.state[1]) == (1 if p > 0 else 0)
    plan.close()


def fp32_edge_reference(lp, Qn, Kn, Vn, En, gn, heads, items, splits):
    """The kernels' formulas in fp32 (tests/transformer_oracle.fp32_reference on the per-entry keys and values
    kk = k + E, vv = v + E, one column per entry), with the per-entry sums folded back onto the columns and dE."""
    f = Qn.shape[1]
    rows, cols = tro.entries(lp.rowptr, lp.colidx)
    nnz = len(rows)
    f32 = np.float32
    with np.errstate(all="ignore"):
        KK, VV = (Kn[cols] + En).astype(f32), (Vn[cols] + En).astype(f32)
        sc = transformer_scale(f, heads)
        out = tro.fp32_reference(lp.rowptr, np.arange(nnz), nnz, Qn, KK, VV, gn, heads, sc, items, splits)
        C_ = f // heads
        hdot = lambda A, B: (A * B).reshape(len(A), heads, C_).sum(2, dtype=f32)
        s = hdot(Qn[rows], KK) * f32(sc)
        p = np.exp(s - out["L"][rows])
        D = hdot(gn, out["Z"])
        ds = p * (hdot(gn[rows], VV) - D[rows])
        ex = lambda x: np.repeat(x, C_, axis=1)
        out["dE"] = ex(p) * gn[rows] + ex(f32(sc) * ds) * Qn[rows]
        for name in ("dK", "dV"):
            acc = np.zeros((lp.m, f), f32)
            np.add.at(acc, cols, out[name])
            out[name] = acc
    return out


@pytest.mark.parametrize("f,heads", [(5, 1), (8, 2)])
@pytest.mark.parametrize("case", ["hub", "gemat11_k1"])
def test_ieee_special_values_in_E(case, f, heads):
    plan = one_rank_plan(case, f)
    lp = plan.lp
    Qn, Kn, Vn, gn = inputs(lp.m, f, 3 * f)
    En = edge_term(lp, f)
    rs = np.random.RandomState(f)
    u = rs.uniform(size=En.shape)
    En[u < 0.004] = np.inf
    En[(u >= 0.004) & (u < 0.008)] = -np.inf
    En[(u >= 0.008) & (u < 0.01)] = np.nan
    Z, L, dQ, _, dKV, _, dE = run_all(plan, t(Qn), t(np.concatenate([Kn, Vn], 1)), t(En), t(gn), f, heads)
    fwd = plan.gated_walks()[0]
    ref = fp32_edge_reference(lp, Qn, Kn, Vn, En, gn, heads, fwd.items.cpu().numpy(), fwd.splits.cpu().numpy())
    has = np.diff(lp.rowptr.astype(np.int64)) > 0
    for name, got in (("Z", Z), ("L", L), ("dQ", dQ), ("dK", dKV[:, :f]), ("dV", dKV[:, f:]), ("dE", dE)):
        g, w = got.cpu().numpy(), ref[name]
        if name == "L":
            g, w = g[has], w[has]
        assert np.isnan(w).any(), name
        assert np.array_equal(np.isnan(g), np.isnan(w)), "%s: %d NaN differ" % (name, int((np.isnan(g) != np.isnan(w)).sum()))
        assert np.array_equal(np.isposinf(g), np.isposinf(w)) and np.array_equal(np.isneginf(g), np.isneginf(w)), name
    plan.close()


def test_entry_offsets_beyond_2_31():
    """A banded graph with nnz * f > 2^31 (f = 256, 4 heads): the last rows' Z, L, dQ and their entries' dE, and the
    last columns' dK and dV, within the bound of fp64 over the last rows' entries."""
    import scipy.sparse as sp
    m, band, f, heads = 40000, 216, 256, 4
    rows = np.repeat(np.arange(m), band)
    cols = (rows + np.tile(np.arange(band), m)) % m
    A = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(m, m))
    lp = planmod.build_local_plan(A, np.zeros(m, dtype=np.int64), 0, 1)
    nnz = lp.nnz()
    assert nnz * f > 2 ** 31
    plan = planmod.PgcnPlan(lp, 2 * f, device=dev())
    plan.bind_values()
    g = torch.Generator(device=dev()).manual_seed(5)
    Q, K, V, gZ = (torch.randn((m, f), device=dev(), generator=g) for _ in range(4))
    E = torch.randn((nnz, f), device=dev(), generator=g)
    Z, L, KV, KVh, _ = aggregate_transformer_edge(plan, Q, K, V, E, heads)
    dQ, dK, dV, dE = aggregate_transformer_edge_backward(plan, Q, KV, KVh, E, Z, L, gZ, heads)
    torch.cuda.synchronize()
    last = 400                                                      # rows m - 400 .. m - 1
    e0 = int(lp.rowptr[m - last])
    sub_ptr = lp.rowptr[m - last:].astype(np.int64) - e0
    sub_col = lp.colidx[e0:]
    cpu = lambda x: x.cpu().numpy()
    ref = teo.attention(sub_ptr, sub_col, m, cpu(Q[m - last:]), cpu(K), cpu(V), cpu(E[e0:]), cpu(gZ[m - last:]), heads,
                        transformer_scale(f, heads), CONST, dcol=np.full(m, band))
    for name, got in (("Z", Z[m - last:]), ("L", L[m - last:]), ("dQ", dQ[m - last:]), ("dE", dE[e0:])):
        within(got, ref[name], "nnz*f > 2^31: " + name)
    done = slice(m - 100, m)                                        # every entry of these columns is in the last rows
    for name, got in (("dK", dK), ("dV", dV)):
        val, tol = ref[name]
        within(got[done], (val[done], tol[done]), "nnz*f > 2^31: " + name)
    plan.close()


def _instances_worker(rank, k):
    """The keys of the kernels torch.profiler sees while every instance runs (vector and scalar, split rows through the
    delta and fixup kernels), each launch's outputs checked against fp64."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for f, heads, shift in ((8, 2, False), (6, 2, False), (8, 2, True)):
        plan = one_rank_plan("hub", f)
        lp = plan.lp
        walks = (planmod.GatedWalk(lp.rowptr, lp.colidx, 64, dev()),
                 planmod.GatedWalk(lp.t_rowptr, lp.t_colidx, 64, dev()))
        assert walks[0].c.nsplits > 0 and walks[1].c.nsplits > 0
        ins = inputs(lp.m, f, f)
        En = edge_term(lp, f)
        for _ in range(3):            # torch.profiler now and then loses a session's activity records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                check_one_rank(plan, ins, En, f, heads, P, walks=walks, shift_E=shift)
                torch.cuda.synchronize()
            names = {key(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "transformer_edge_" in e.name}
            if len(names) == 7:
                break
        seen |= names
        plan.close()
    return sorted(seen)


def test_profiler_sees_every_instance_of_the_manifest():
    with open(os.path.join(ROOT, "tests", "transformer_edge_kernel_instances.txt")) as fh:
        want = sorted({key(ln) for ln in fh if ln.strip()})
    assert spawn_ranks(_instances_worker, 1) == {0: want}


# ---- several ranks ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("case,f,heads", [("gemat11_k2", 64, 4), ("gemat11_k2", 6, 2), ("gemat11_k3_hp", 16, 1),
                                          ("gemat11_k3_hp", 136, 8)])
def test_multi_rank_within_the_bound_of_one_rank(case, f, heads, p):
    A, pv, k = problem(case)
    n = A.shape[0]
    ins_n = inputs(n, f, f + k)
    one = one_rank_plan(case, f)
    lp1 = one.lp
    E1 = edge_term(lp1, f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    pos = [edge_rows(lp1, lp) for lp in lps]
    ins = [[t(a[lp.owned]) for a in ins_n] + [t(edge_term(lp, f))] for lp in lps]
    drops = [EdgeDropout(p, KEY, dev()) for _ in plans]

    def step(r):
        Q, K, V, g, E = ins[r]
        Z, L, KV, KVh, snap = aggregate_transformer_edge(plans[r], Q, K, V, E, heads, drop=drops[r])
        return (Z, L) + aggregate_transformer_edge_backward(plans[r], Q, KV, KVh, E, Z, L, g, heads, drop=drops[r],
                                                            snap=snap)

    first = None
    for rep in range(2):                                  # both epoch parities of the peer slabs; counters 1 and 2
        ref = reference(lp1, *ins_n[:3], E1, ins_n[3], heads, p, rep + 1)
        out = run_ranks(plans, step, streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "L", "dQ", "dK", "dV", "dE"), out[r]):
                val, tol = ref[name]
                sel = pos[r] if name == "dE" else lp.owned
                within(got, (val[sel], tol[sel]), "%s %s rank %d rep %d" % (case, name, r, rep))
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
    E = torch.from_numpy(edge_term(p.lp, f)).cuda().requires_grad_(True)
    Z = PTransformerEdgeAttention.apply(p, Q, K, V, E, 4, None, EdgeDropout(P, KEY, torch.device("cuda", rank)))
    Z.backward(g.detach())
    torch.cuda.synchronize()
    dist.barrier()
    p.close()
    dist.destroy_process_group()
    return used, [x.cpu().numpy() for x in (Z.detach(), Q.grad, K.grad, V.grad, E.grad)]


@pytest.mark.multigpu
def test_two_gpus_nccl_gives_the_peer_transport_bits():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    a = spawn_ranks(_nccl_worker, 2, (29883, "nccl"))
    b = spawn_ranks(_nccl_worker, 2, (29884, "p2p"))
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
    En = edge_term(lp, f)
    Q, K, V, E = (t(a).requires_grad_(True) for a in (Qn, Kn, Vn, En))
    Z = PTransformerEdgeAttention.apply(plan, Q, K, V, E, heads)
    Z.backward(t(gn))
    ref = reference(lp, Qn, Kn, Vn, En, gn, heads)
    for name, got in (("Z", Z), ("dQ", Q.grad), ("dK", K.grad), ("dV", V.grad), ("dE", E.grad)):
        within(got, ref[name], "%s %s" % (layout, name))
    # E without a gradient: the same node gradients, and none for E
    Q2, K2, V2 = (t(a).requires_grad_(True) for a in (Qn, Kn, Vn))
    E2 = t(En)
    Z2 = PTransformerEdgeAttention.apply(plan, Q2, K2, V2, E2, heads)
    Z2.backward(t(gn))
    assert E2.grad is None
    for a, b in ((Z, Z2), (Q.grad, Q2.grad), (K.grad, K2.grad), (V.grad, V2.grad)):
        assert torch.equal(a, b)
    plan.close()


def in_eager_process(worker):
    """worker(0, 1) in a spawned process of its own with CUDA_MODULE_LOADING=EAGER, its result returned. Several ranks
    in one process share one device wait: with lazy loading, the first launch of a torch or cuBLAS kernel chosen for one
    rank's shapes waits for the device, where an earlier rank's exchange waits for this rank's half, which the blocked
    thread never enqueues. Ranks in separate processes, as in a real job, do not share that wait."""
    old = os.environ.get("CUDA_MODULE_LOADING")
    os.environ["CUDA_MODULE_LOADING"] = "EAGER"
    try:
        return spawn_ranks(worker, 1)[0]
    finally:
        if old is None:
            del os.environ["CUDA_MODULE_LOADING"]
        else:
            os.environ["CUDA_MODULE_LOADING"] = old


def test_autograd_three_ranks_and_global_layout():
    assert in_eager_process(_autograd_three_ranks_worker)


def _autograd_three_ranks_worker(rank, k):
    A, pv, k = problem("gemat11_k3_hp")
    n, f, heads = A.shape[0], 16, 2
    ins_n = inputs(n, f, 3)
    one = one_rank_plan("gemat11_k3_hp", f)
    E1 = edge_term(one.lp, f)
    lps = [planmod.build_local_plan(A, pv, r, k) for r in range(k)]
    pos = [edge_rows(one.lp, lp) for lp in lps]
    plans = linked_plans(lps, 2 * f, 1)
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    for counter, layout in enumerate(("local", "global"), 1):
        ref = reference(one.lp, *ins_n[:3], E1, ins_n[3], heads, P, counter)
        for p in plans:
            p.layout = layout
        if counter == 1:
            drops = [EdgeDropout(P, KEY, dev()) for _ in plans]
        pick = (lambda a, lp: a[lp.owned]) if layout == "local" else (lambda a, lp: np.where(
            (pv == lp.rank)[:, None], a, np.float32(7.0)))               # non-owned rows are ignored
        leaves = [[t(pick(a, lp)).requires_grad_(True) for a in ins_n[:3]] + [t(E1[q]).requires_grad_(True)]
                  for lp, q in zip(lps, pos)]
        Z = run_ranks(plans, lambda r: PTransformerEdgeAttention.apply(plans[r], *leaves[r], heads, None, drops[r]),
                      streams)
        run_ranks(plans, lambda r: Z[r].backward(t(pick(ins_n[3], lps[r]))), streams)
        for r, lp in enumerate(lps):
            for name, got in zip(("Z", "dQ", "dK", "dV", "dE"), [Z[r]] + [x.grad for x in leaves[r]]):
                val, tol = ref[name]
                if name == "dE":
                    within(got, (val[pos[r]], tol[pos[r]]), "%s dE rank %d" % (layout, r))
                elif layout == "global":
                    val, tol = np.where((pv == r)[:, None], val, 0.0), np.where((pv == r)[:, None], tol, 0.0)
                    within(got, (val, tol), "global %s rank %d" % (name, r))
                else:
                    within(got, (val[lp.owned], tol[lp.owned]), "local %s rank %d" % (name, r))
    for p in plans + [one]:
        p.close()
    return True


def test_one_rank_capture_with_dropout_and_refusal_before_the_first_eager_call():
    f, heads = 64, 4
    plan = one_rank_plan("hub", f)
    m, nnz = plan.lp.m, plan.lp.nnz()
    Q, K, V, g = (torch.zeros((m, f), device=dev()) for _ in range(4))
    E = torch.zeros((nnz, f), device=dev())
    drop = EdgeDropout(P, KEY, dev())

    def step(Q, K, V, E, g, drop):
        Z, L, KV, KVh, snap = aggregate_transformer_edge(plan, Q, K, V, E, heads, drop=drop)
        dQ, dK, dV, dE = aggregate_transformer_edge_backward(plan, Q, KV, KVh, E, Z, L, g, heads, drop=drop, snap=snap)
        return dict(Z=Z, L=L, dQ=dQ, dK=dK, dV=dV, dE=dE)

    s = torch.cuda.Stream()
    launches = plan.launch_count()
    plan.gated_walks()                                    # the walks and ids exist; the transposed entries do not yet
    plan.global_ids()
    with pytest.raises(RuntimeError, match="transposed_entries"):
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            step(Q, K, V, E, g, drop)
    assert plan.launch_count() == launches and plan._transposed_entries is None and int(drop.state[1]) == 0
    ins = [tuple(t(a) for a in inputs(m, f, 20 + i)) + (t(edge_term(plan.lp, f) * (i + 1)),) for i in range(3)]

    def load(i):
        for dst, src in zip((Q, K, V, g, E), (ins[i][0], ins[i][1], ins[i][2], ins[i][3], ins[i][4])):
            dst.copy_(src)

    plan.prepare(2 * f)
    step(*ins[0][:3], ins[0][4], ins[0][3], None)         # the first eager call builds the transposed entries
    check_one_rank_capture(plan, lambda: step(Q, K, V, E, g, drop), load,
                           lambda i: step(*ins[i][:3], ins[i][4], ins[i][3], follower(drop)))
    assert int(drop.state[1]) == 4                        # one draw per replay, none at capture
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
        p.transposed_entries()
    streams = [torch.cuda.Stream(device=dev()) for _ in plans]
    ins = [inputs(n, f, 30 + i) for i in range(3)]
    made = []

    def buffers(r):
        b = {name: torch.zeros((lps[r].m, f), device=dev()) for name in ("x", "k", "v", "g")}
        b["e"] = torch.zeros((lps[r].nnz(), f), device=dev())
        b["drop"] = EdgeDropout(P, KEY, dev())
        made.append(b)
        return b

    def load(bufs, i):
        for r, lp in enumerate(lps):
            for name, a in zip(("x", "k", "v", "g"), ins[i]):
                bufs[r][name].copy_(t(a[lp.owned]))
            bufs[r]["e"].copy_(t(edge_term(lp, f) * (i + 1)))
            if bufs[r] is not made[r]:                    # eager buffers draw with the counter the replay just used
                bufs[r]["drop"] = follower(made[r]["drop"])
        torch.cuda.synchronize()

    def step(r, b):
        Z, L, KV, KVh, snap = aggregate_transformer_edge(plans[r], b["x"], b["k"], b["v"], b["e"], heads,
                                                         drop=b["drop"])
        dQ, dK, dV, dE = aggregate_transformer_edge_backward(plans[r], b["x"], KV, KVh, b["e"], Z, L, b["g"], heads,
                                                             drop=b["drop"], snap=snap)
        return dict(Z=Z, dQ=dQ, dK=dK, dV=dV, dE=dE)

    check_two_rank_capture(plans, streams, buffers, load, step)
    for r in range(k):
        assert int(made[r]["drop"].state[1]) == 4
    for p in plans:
        p.close()


# ---- the command line ------------------------------------------------------------------------------------------------

def test_cli_edge_values_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PTRANSFORMER.py", ["--edge-values", "--heads", "2"], 29793)
    assert_follows(lines, teo.intended_training(karate(), 2, 4, 7, heads=2))


def test_cli_edge_values_attn_dropout_follows_the_fp64_loss_curve(tmp_path):
    lines = run_cli(tmp_path, "PTRANSFORMER.py", ["--edge-values", "--attn-dropout", "0.5"], 29794)
    assert_follows(lines, teo.intended_training(karate(), 2, 4, 7, p=0.5))


def _three_rank_worker(rank, k):
    """transformer.run's training loop with --edge-values on one rank and on the three ranks of karate_k3 in this
    process (peer transport): (one-rank curve, three-rank curve)."""
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
            m = nn.Sequential(*[PTRANSFORMER(p, f, f, heads, edge_values=True) for _ in range(L)]).to(dev())
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
    for p in plans + one:
        p.close()
    return curve1, curve3


def test_edge_values_layer_on_three_ranks_follows_the_one_rank_curve():
    """The layer with --edge-values on one rank and on three, against the fp64 oracle with gradients averaged over
    three ranks, the ranks in a process of their own (in_eager_process: lin_edge's backward launches cuBLAS kernels
    chosen for each rank's entry count)."""
    A, _, _ = problem("karate")
    curve1, curve3 = in_eager_process(_three_rank_worker)
    np.testing.assert_allclose(curve1, teo.intended_training(A, 2, 4, 7, heads=2), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, teo.intended_training(A, 2, 4, 7, k=3, heads=2), rtol=1e-3, atol=6e-5)
    np.testing.assert_allclose(curve3, curve1, rtol=1e-3, atol=6e-5)
