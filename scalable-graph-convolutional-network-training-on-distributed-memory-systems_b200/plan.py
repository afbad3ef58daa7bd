"""Loader-side plan of the PGCN path: what GPU/PGCN.py:37-64 and :175-182 compute, vectorised.

The reference walks every nnz in interpreted Python on every rank (GPU/PGCN.py:41-45) and keeps an
n x n COO with global indices (:53-64). Here the same information is produced with O(nnz) NumPy:

  * `compute_communication_maps` / `get_partition_of_adjacency_matrix`: same names, arguments and
    return meaning as the reference functions (dicts of sorted global ids per peer; the owned rows
    of A) — drop-in for callers that want the reference's data structures;
  * `build_local_plan`: the compact per-rank layout the H100 kernels consume — local CSR (int32)
    over the column space [own | halo grouped by source peer, sorted by global id], its transpose,
    send_idx / send_off / recv_off. Sender order == receiver order because both sides sort by
    global id (the invariant GPU/PGCN.py:47-48 relies on);
  * `PgcnPlan`: owns the device-side plan (C-ABI handle) and the host stats the reference keeps in
    device counters (GPU/PGCN.py:78-83).
"""
import collections
import ctypes as C

import numpy as np
import scipy.sparse as sp

from . import cabi


def _coo(A):
    A = A.tocoo() if sp.issparse(A) else sp.coo_matrix(A)
    return A


def compute_communication_maps(A, partvec, rank, size):
    """Vectorised GPU/PGCN.py:37-51.

    Returns (send_map, recv_map): dicts keyed by every OTHER rank (possibly empty arrays), values
    sorted int64 global vertex ids. recv_map[p] = columns owned by p referenced by my rows;
    send_map[p] = my columns referenced by rows of p. send_map_r[p] == recv_map_p[r].
    """
    A = _coo(A)
    pv = np.asarray(partvec, dtype=np.int64)
    n = A.shape[0]
    prow, pcol = pv[A.row], pv[A.col]
    cross = prow != pcol
    # I receive column j from part[j] when one of my rows references it
    mine = cross & (prow == rank)
    rkeys = np.unique(pcol[mine] * n + A.col[mine].astype(np.int64))
    # I send my column j to part[i] for every foreign row i that references it
    theirs = cross & (pcol == rank)
    skeys = np.unique(prow[theirs] * n + A.col[theirs].astype(np.int64))
    send_map, recv_map = {}, {}
    for p in range(size):
        if p == rank:
            continue
        lo, hi = np.searchsorted(rkeys, [p * n, (p + 1) * n])
        recv_map[p] = rkeys[lo:hi] - p * n
        lo, hi = np.searchsorted(skeys, [p * n, (p + 1) * n])
        send_map[p] = skeys[lo:hi] - p * n
    return send_map, recv_map


def get_partition_of_adjacency_matrix(A, partvec, rank):
    """Vectorised GPU/PGCN.py:53-64: the entries of A whose ROW is owned by `rank`, global indices,
    global shape, duplicates kept. Returns scipy COO (float32)."""
    A = _coo(A)
    pv = np.asarray(partvec, dtype=np.int64)
    keep = pv[A.row] == rank
    return sp.coo_matrix((A.data[keep].astype(np.float32), (A.row[keep], A.col[keep])), shape=A.shape)


# the reference's spelling (GPU/PGCN.py:53)
get_partitiont_of_adjacency_matrix = get_partition_of_adjacency_matrix


class LocalPlan:
    """Host-side arrays of one rank (all NumPy, no device state)."""

    def __init__(self):
        self.n = 0; self.k = 1; self.rank = 0
        self.m = 0; self.h = 0; self.S = 0
        self.owned = None        # int64[m] global ids of my rows, ascending
        self.halo = None         # int64[h] global ids of halo rows, [peer0 | peer1 | ...], ascending inside
        self.rowptr = self.colidx = self.vals = None
        self.t_rowptr = self.t_colidx = self.t_vals = None
        self.send_idx = None     # int32[S] local row ids
        self.send_gid = None     # int64[S] global ids (wire order)
        self.send_off = None     # int64[k+1]
        self.recv_off = None     # int64[k+1]

    # --- the reference's views -----------------------------------------------------------------
    def send_map(self):
        return {p: self.send_gid[self.send_off[p]:self.send_off[p + 1]] for p in range(self.k) if p != self.rank}

    def recv_map(self):
        return {p: self.halo[self.recv_off[p]:self.recv_off[p + 1]] for p in range(self.k) if p != self.rank}

    def nnz(self):
        return int(self.rowptr[-1])


def build_local_plan(A, partvec, rank, size):
    """Compact per-rank layout (see module docstring). O(nnz) NumPy + scipy COO->CSR."""
    A = _coo(A)
    n = A.shape[0]
    pv = np.asarray(partvec, dtype=np.int64)
    if pv.shape[0] != n:
        raise ValueError("part vector has %d entries, matrix has %d rows" % (pv.shape[0], n))
    if pv.size and (pv.min() < 0 or pv.max() >= size):
        raise KeyError(int(pv.max() if pv.max() >= size else pv.min()))   # the reference's failure mode

    lp = LocalPlan()
    lp.n, lp.k, lp.rank = n, size, rank
    owned = np.flatnonzero(pv == rank).astype(np.int64)
    lp.owned = owned
    lp.m = m = owned.shape[0]
    g2l = np.full(n, -1, dtype=np.int64)
    g2l[owned] = np.arange(m)

    prow, pcol = pv[A.row], pv[A.col]
    mine = prow == rank
    grow, gcol = A.row[mine].astype(np.int64), A.col[mine].astype(np.int64)
    val = A.data[mine].astype(np.float32)
    pc = pcol[mine]

    # halo = distinct foreign columns, grouped by owner then sorted by global id
    foreign = pc != rank
    hkeys = np.unique(pc[foreign] * n + gcol[foreign])
    hpart, hgid = hkeys // n, hkeys % n
    lp.halo = hgid
    lp.h = h = hgid.shape[0]
    lp.recv_off = np.concatenate([[0], np.cumsum(np.bincount(hpart, minlength=size))]).astype(np.int64)

    lcol = g2l[gcol]
    if h:
        lcol[foreign] = m + np.searchsorted(hkeys, pc[foreign] * n + gcol[foreign])
    lrow = g2l[grow]

    csr = sp.coo_matrix((val, (lrow, lcol)), shape=(m, m + h)).tocsr()   # duplicates summed (fp32)
    csr.sort_indices()
    lp.rowptr = csr.indptr.astype(np.int32)
    lp.colidx = csr.indices.astype(np.int32)
    lp.vals = csr.data.astype(np.float32)
    csc = csr.T.tocsr()
    csc.sort_indices()
    lp.t_rowptr = csc.indptr.astype(np.int32)
    lp.t_colidx = csc.indices.astype(np.int32)
    lp.t_vals = csc.data.astype(np.float32)

    # send lists: my columns referenced by rows of peer p, grouped by p, sorted by global id
    theirs = (pcol == rank) & (prow != rank)
    skeys = np.unique(prow[theirs] * n + A.col[theirs].astype(np.int64))
    spart, sgid = skeys // n, skeys % n
    lp.send_gid = sgid
    lp.send_idx = g2l[sgid].astype(np.int32)
    lp.S = int(sgid.shape[0])
    lp.send_off = np.concatenate([[0], np.cumsum(np.bincount(spart, minlength=size))]).astype(np.int64)
    return lp


PLAN_FORMAT_VERSION = 2      # bump when LocalPlan's layout or build_local_plan's ordering / duplicate semantics change

_LP_ARRAYS = ("owned", "halo", "rowptr", "colidx", "vals", "t_rowptr", "t_colidx", "t_vals",
              "send_idx", "send_gid", "send_off", "recv_off")


def save_local_plan(path, lp):
    """Binary cache of one rank's plan (SURVEY.md §8f rank 2): the reference re-reads the .mtx and re-walks
    every nnz on every rank at every start (GPU/PGCN.py:171-176)."""
    np.savez(path, meta=np.array([lp.n, lp.k, lp.rank, lp.m, lp.h, lp.S], dtype=np.int64),
             **{name: getattr(lp, name) for name in _LP_ARRAYS})


def load_local_plan(path):
    z = np.load(path)
    lp = LocalPlan()
    lp.n, lp.k, lp.rank, lp.m, lp.h, lp.S = [int(x) for x in z["meta"]]
    for name in _LP_ARRAYS:
        setattr(lp, name, z[name])
    return lp


def read_local_plan(path_A, path_partvec, rank, size):
    """build_local_plan of the MatrixMarket matrix at path_A and the part vector at path_partvec, which must name a
    part below `size` for every row (GPU/PGCN.py:171-176)."""
    from . import graphio
    A = graphio.read_adjacency(path_A)
    pv = graphio.check_partvec(graphio.read_partvec(path_partvec, A.shape[0]), size)
    return build_local_plan(A, pv, rank, size)


def cached_local_plan(path_A, path_partvec, rank, size, cache_dir):
    """build_local_plan with an on-disk cache keyed by the two input files (size + mtime), rank and size."""
    import hashlib
    import os
    sa, sp_ = os.stat(path_A), os.stat(path_partvec)
    key = hashlib.sha1(repr([PLAN_FORMAT_VERSION, os.path.abspath(path_A), sa.st_size, sa.st_mtime_ns,
                             os.path.abspath(path_partvec), sp_.st_size, sp_.st_mtime_ns,
                             rank, size]).encode()).hexdigest()[:16]
    os.makedirs(cache_dir, exist_ok=True)
    path = os.path.join(cache_dir, "plan_%s_r%dof%d.npz" % (key, rank, size))
    if os.path.exists(path):
        lp = load_local_plan(path)
        if lp.k == size and lp.rank == rank:
            return lp
    lp = read_local_plan(path_A, path_partvec, rank, size)
    tmp = path + ".%d.tmp.npz" % os.getpid()
    save_local_plan(tmp, lp)
    os.replace(tmp, path)
    return lp


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


class PgcnPlan:
    """Device-side plan = the `A` handle handed to PSpMM.apply (SURVEY.md §8b).

    Wraps pgcn_plan_create/destroy and carries the host counters the reference keeps as device
    tensors (GPU/PGCN.py:78-83, :105-106, :113-114): volumes in ROWS, message counts including the
    zero-length ones (the reference sends them, GPU/PGCN.py:101-107).
    """

    def __init__(self, local_plan, f_max, device=None):
        import torch
        self.lp = lp = local_plan
        self.f_max = int(f_max)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._lib = cabi.load()
        self._h = C.c_void_p()
        self.layout = "local"
        self.stats = {"send_volume": 0, "recv_volume": 0, "send_nmsg": 0, "recv_nmsg": 0}
        for name in ("rowptr", "colidx", "vals", "t_rowptr", "t_colidx", "t_vals", "send_idx", "send_off", "recv_off"):
            setattr(lp, name, np.ascontiguousarray(getattr(lp, name)))
        with torch.cuda.device(self.device):
            rc = self._lib.pgcn_plan_create(
                _ptr(lp.rowptr), _ptr(lp.colidx), _ptr(lp.vals), lp.m, lp.h,
                _ptr(lp.t_rowptr), _ptr(lp.t_colidx), _ptr(lp.t_vals),
                _ptr(lp.send_idx), _ptr(lp.send_off), _ptr(lp.recv_off),
                lp.k, lp.rank, self.f_max, C.byref(self._h))
        cabi.check(rc, None)
        self._owned_t = None
        self._edge_index = None
        self._edge_pairs = None
        self._gated_walks = None
        self._global_ids = None
        self._transposed_entries = None
        self._relation_walks = {}        # (_values_key(rel), R) -> (rel, walks): relation_walks' tables per rel and R
        # edge values (bind_values / set_values): which values the records hold, as far as this process knows
        self._bound = False
        self._resident = "creation"      # "creation", a key of the tensor set last, or None: unknown
        self._resident_ref = None        # that tensor, kept alive so that its key cannot be reused
        self._captured = False           # values were set inside a CUDA-graph capture: replays change them unseen

    # -- lifetime ------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.pgcn_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        if not self._h.value:
            raise RuntimeError("plan is closed")
        return self._h

    @property
    def m(self):
        return self.lp.m

    @property
    def n(self):
        return self.lp.n

    def owned_index(self):
        import torch
        if self._owned_t is None:
            self._owned_t = torch.from_numpy(self.lp.owned).to(self.device)
        return self._owned_t

    # -- options / info ------------------------------------------------------------------------
    def set_option(self, name, value):
        cabi.check(self._lib.pgcn_plan_set_option(self.handle, name.encode(), int(value)), self._h)

    def get_option(self, name):
        return int(self._lib.pgcn_plan_get_option(self.handle, name.encode()))

    def autotune(self, f):
        """Pick the fastest edges_per_block for this matrix at width f (set-up work). Returns it."""
        import torch
        with torch.cuda.device(self.device):
            return cabi.check(self._lib.pgcn_plan_autotune(self.handle, int(f)), self._h)

    def prepare(self, f):
        """Set-up work for width f under the current options (pgcn_plan_prepare), so that PSpMM / PSpMMRelu on this
        plan can be captured in a CUDA graph (torch.cuda.graph, torch.cuda.make_graphed_callables). Synchronous. Call it
        again after changing f or an option."""
        import torch
        self.owned_index()                # the "global" layout's index tensor: a host-to-device copy, not capturable
        with torch.cuda.device(self.device):
            cabi.check(self._lib.pgcn_plan_prepare(self.handle, int(f)), self._h)

    # -- edge values ---------------------------------------------------------------------------
    def bind_values(self):
        """Build the maps set_values needs (pgcn_plan_bind_values): synchronous set-up, not capturable; 4 B per edge and
        record set, about 8 B per edge on one rank and 12 B on a split multi-rank plan. Idempotent."""
        import torch
        if self._bound:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("PgcnPlan.bind_values is set-up work and cannot run while a CUDA graph is being captured: "
                               "call it before the capture")
        with torch.cuda.device(self.device):
            cabi.check(self._lib.pgcn_plan_bind_values(self.handle), self._h)
        self._bound = True

    def set_values(self, vals):
        """Aggregate with `vals` (fp32 CUDA [nnz], this plan's local forward CSR order, i.e. lp.colidx's order) from now on,
        stream-ordered on the current stream; None restores the values the plan was created with. Needs bind_values."""
        import torch
        ptr = None
        if vals is not None:
            ptr = check_values(self, vals).data_ptr()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.pgcn_plan_set_values(self.handle, ptr, torch.cuda.current_stream().cuda_stream), self._h)
        if torch.cuda.is_current_stream_capturing():
            # what the device holds after the capture depends on which graphs are replayed: never trust a record again
            self._captured = True
            self._resident, self._resident_ref = None, None
        elif vals is None:
            self._resident, self._resident_ref = "creation", None
        else:
            self._resident, self._resident_ref = _values_key(vals), vals

    def use_values(self, vals):
        """Make `vals` (None: the creation values) the resident values before a launch on the current stream.

        Skips the rewrite when this plan last set the same tensor eagerly and its version counter has not moved since.
        Writes that bypass the counter (`w.data.copy_(...)`, assigning `w.data`, DLPack or raw-pointer kernels) are not
        seen: after such a write call set_values(w) yourself. On a plan that was never bound, None costs nothing and a
        tensor raises (bind_values is synchronous set-up and is not done implicitly). Under CUDA-graph capture, and on a
        plan whose values were ever set inside a capture, it always rewrites, so that a graph never depends on what was
        resident when it was captured or replayed; such a plan pays one set_values launch (0.34 ms on C2, DESIGN.md §6)
        before every later PSpMM / PSpMMRelu forward and backward as well."""
        import torch
        if not self._bound:
            if vals is None:
                return
            raise RuntimeError("edge values need the plan's value maps: call PgcnPlan.bind_values() once (set-up, "
                               "before any CUDA-graph capture) before PSpMMWeighted or set_values")
        if not torch.cuda.is_current_stream_capturing() and not self._captured:
            if vals is None and self._resident == "creation":
                return
            if vals is not None and self._resident_ref is vals and self._resident == _values_key(vals):
                return
        self.set_values(vals)

    def edge_index(self):
        """(row, col) of every forward entry, int64 CUDA tensors in the order of the values set_values takes: rows in
        [0, m) (global id lp.owned[row]), columns in [0, m + h) (own rows, then the halo rows lp.halo[col - m])."""
        import torch
        if self._edge_index is None:
            lp = self.lp
            rows = np.repeat(np.arange(lp.m, dtype=np.int64), np.diff(lp.rowptr.astype(np.int64)))
            self._edge_index = (torch.from_numpy(rows).to(self.device),
                                torch.from_numpy(lp.colidx.astype(np.int64)).to(self.device))
        return self._edge_index

    def edge_pairs(self):
        """(global row, global column) of every forward entry, a CUDA int32 [nnz, 2] tensor in lp.colidx's order (the
        order of edge_index() and of the values set_values takes). Edge dropout (op.EdgeDropout) draws its mask from
        these pairs, so that every partition of the graph draws the same mask. Built on first use by a host-to-device
        copy, which a CUDA graph cannot capture: call it once before capturing a step that uses it."""
        import torch
        if self._edge_pairs is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PgcnPlan.edge_pairs is built by a host-to-device copy, which a CUDA-graph capture "
                                   "cannot hold: call plan.edge_pairs() once before the capture")
            lp = self.lp
            if lp.n > np.iinfo(np.int32).max:
                raise ValueError("n=%d: edge_pairs holds global ids as int32" % lp.n)
            rows = np.repeat(lp.owned, np.diff(lp.rowptr.astype(np.int64)))
            cols = np.concatenate([lp.owned, lp.halo])[lp.colidx]
            pairs = np.stack([rows, cols], 1).astype(np.int32)
            self._edge_pairs = torch.from_numpy(pairs).to(self.device)
        return self._edge_pairs

    def gated_walks(self):
        """(fwd, tr): the GatedWalk of the local forward CSR and of its transpose, the device index arrays and work tables
        of the gated aggregation (op.PSpMMGated, include/pgcn_gated.h) and of the transformer attention
        (op.PTransformerAttention, include/pgcn_transformer.h), which walk the same tables. About 8 B per entry (both index arrays) and 16 B
        per row and per column (the work items), about 170 MB on C2. Built on first use by host-to-device copies, which a
        CUDA graph cannot capture: call it, or the operator once eagerly, before capturing a step that uses it."""
        import torch
        if self._gated_walks is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PgcnPlan.gated_walks is built by host-to-device copies, which a CUDA-graph capture "
                                   "cannot hold: call plan.gated_walks() once before the capture")
            chunk = cabi.load_gated().pgcn_gated_chunk()
            lp = self.lp
            self._gated_walks = (GatedWalk(lp.rowptr, lp.colidx, chunk, self.device),
                                 GatedWalk(lp.t_rowptr, lp.t_colidx, chunk, self.device))
        return self._gated_walks

    def global_ids(self):
        """The global ids of the owned rows, then of the halo rows ([halo by peer] order): a CUDA int32 [m + h] tensor,
        the ids the transformer attention's dropout mask is drawn from (include/pgcn_transformer.h), so that every
        partition draws the same mask. Built on first use by a host-to-device copy, which a CUDA graph cannot capture:
        call it, or the operator once eagerly, before capturing a step that uses it."""
        import torch
        if self._global_ids is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PgcnPlan.global_ids is built by a host-to-device copy, which a CUDA-graph capture "
                                   "cannot hold: call plan.global_ids() once before the capture")
            lp = self.lp
            if lp.n > np.iinfo(np.int32).max:
                raise ValueError("n=%d: global_ids holds global ids as int32" % lp.n)
            ids = np.concatenate([lp.owned, lp.halo]).astype(np.int32)
            self._global_ids = torch.from_numpy(ids).to(self.device)
        return self._global_ids

    def transposed_entries(self):
        """The forward entry of every transposed entry: a CUDA int32 [nnz] tensor `perm` with lp.t_colidx ==
        rows[perm] (rows the forward entries' rows), from a stable sort of the forward entries by column, so duplicated
        entries keep their forward order. GatedGCN's column walk (op.PGatedGCN, include/pgcn_gatedgcn.h) reads the
        per-entry tensors through it. 4 B per entry. Built on first use by a host-to-device copy, which a CUDA graph
        cannot capture: call it, or the operator once eagerly, before capturing a step that uses it."""
        import torch
        if self._transposed_entries is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PgcnPlan.transposed_entries is built by a host-to-device copy, which a CUDA-graph "
                                   "capture cannot hold: call plan.transposed_entries() once before the capture")
            lp = self.lp
            perm = np.argsort(lp.colidx, kind="stable")
            rows = np.repeat(np.arange(lp.m, dtype=np.int32), np.diff(lp.rowptr.astype(np.int64)))
            if not np.array_equal(rows[perm], lp.t_colidx):
                raise ValueError("the plan's transposed CSR is not the stable column sort of its forward CSR")
            self._transposed_entries = torch.from_numpy(perm.astype(np.int32)).to(self.device)
        return self._transposed_entries

    def relation_walks(self, rel, R):
        """RelationWalks (fwd, tr, perm_f, mean, R): the walks of the relational aggregation (op.PRGCN,
        include/pgcn_rgcn.h) for the relation types `rel` (an integer tensor [nnz_local] in edge_pairs() order, values
        in [0, R)), numbering the output rows v = i R + r for row i and relation r:

          perm_f  CUDA int32 [nnz]: the forward entries sorted stably by (row, relation), so a virtual row keeps its
                  entries in forward CSR order; perm_f[e] is the forward entry of sorted entry e
          fwd     GatedWalk over the m R virtual rows with idx = colidx[perm_f]
          tr      GatedWalk over the transposed CSR (m + h columns) with idx = t_colidx R + rel[perm_t], perm_t =
                  transposed_entries()
          mean    CUDA fp32 [nnz] in forward entry order: 1 / c, the fp32 quotient, c the number of entries of the
                  entry's (row, relation) pair (aggr="mean")

        Built on the host on first use and kept per rel tensor (its identity and version, as the edge values are) and
        R; the tables take about 16 B per entry and 16 B per virtual row. Building them copies to the device, which a
        CUDA graph cannot capture: call it, or the operator once eagerly, before capturing a step that uses it."""
        import operator
        import torch
        if isinstance(R, bool):
            raise TypeError("R must be an integer, got %r" % (R,))
        R = operator.index(R)
        if not torch.is_tensor(rel):
            raise TypeError("rel must be an integer tensor, got %s" % type(rel).__name__)
        key = (_values_key(rel), R)
        hit = self._relation_walks.get(key)
        if hit is not None and hit[0] is rel:
            return hit[1]
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("PgcnPlan.relation_walks is built by host-to-device copies, which a CUDA-graph capture "
                               "cannot hold: call plan.relation_walks(rel, R) once before the capture")
        lp = self.lp
        if rel.dtype.is_floating_point or rel.dtype.is_complex or rel.dtype == torch.bool:
            raise TypeError("rel must be an integer tensor, got %s" % rel.dtype)
        nnz = lp.nnz()
        if rel.dim() != 1 or rel.shape[0] != nnz:
            raise ValueError("rel must be [%d] (the plan's local entries, edge_pairs() order), got %s" % (
                nnz, tuple(rel.shape)))
        if R < 1:
            raise ValueError("R=%d: need at least one relation" % R)
        if lp.m * R > np.iinfo(np.int32).max:
            raise ValueError("m R = %d * %d virtual rows exceed 2^31 - 1" % (lp.m, R))
        r = rel.detach().cpu().numpy().astype(np.int64)
        if nnz and (r.min() < 0 or r.max() >= R):
            bad = int(r.min() if r.min() < 0 else r.max())
            raise ValueError("rel holds relation %d, outside [0, R) = [0, %d)" % (bad, R))
        chunk = cabi.load_gated().pgcn_gated_chunk()
        rows = np.repeat(np.arange(lp.m, dtype=np.int64), np.diff(lp.rowptr.astype(np.int64)))
        vrow = rows * R + r
        perm_f = np.argsort(vrow, kind="stable")
        count = np.bincount(vrow, minlength=lp.m * R)
        vptr = np.concatenate([[0], np.cumsum(count)])
        perm_t = self.transposed_entries().cpu().numpy().astype(np.int64)
        mean = np.float32(1.0) / count[vrow].astype(np.float32)
        walks = RelationWalks(GatedWalk(vptr, lp.colidx[perm_f], chunk, self.device),
                              GatedWalk(lp.t_rowptr, lp.t_colidx.astype(np.int64) * R + r[perm_t], chunk, self.device),
                              torch.from_numpy(perm_f.astype(np.int32)).to(self.device),
                              torch.from_numpy(mean).to(self.device), R)
        # a rel tensor changed in place leaves its old tables behind: drop them
        self._relation_walks = {k: v for k, v in self._relation_walks.items() if v[0] is not rel}
        self._relation_walks[key] = (rel, walks)
        return walks

    def algorithmic_bytes(self, f):
        b = cabi.PgcnBytes()
        cabi.check(self._lib.pgcn_algorithmic_bytes(self.handle, int(f), C.byref(b)), self._h)
        return b.as_dict()

    def launch_count(self):
        return int(self._lib.pgcn_launch_count(self.handle))

    # -- communicator --------------------------------------------------------------------------
    def init_comm(self, group=None, transport="auto", nccl_fallback=True):
        """Collective. transport: "nccl" (grouped ncclSend/ncclRecv), "p2p" (peer-memory stores over
        NVLink, single box), or "auto" (p2p when every rank can export/import, else nccl)."""
        import torch
        import torch.distributed as dist
        if self.lp.k == 1:
            return "none"
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised before PgcnPlan.init_comm")
        # collectives of the set-up phase run on whatever backend the process group has
        cdev = self.device if dist.get_backend(group) == "nccl" else torch.device("cpu")
        used = None
        if transport in ("p2p", "auto"):
            blob = C.create_string_buffer(cabi.P2P_HANDLE_BYTES)
            with torch.cuda.device(self.device):
                rc = self._lib.pgcn_p2p_export(self.handle, blob)
            ok = torch.tensor([1 if rc == 0 else 0], device=cdev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
            if int(ok.item()) == 1:
                mine = torch.frombuffer(bytearray(blob.raw), dtype=torch.uint8).to(cdev)
                allb = [torch.empty_like(mine) for _ in range(self.lp.k)]
                dist.all_gather(allb, mine, group=group)
                packed = b"".join(bytes(t.cpu().numpy().tobytes()) for t in allb)
                with torch.cuda.device(self.device):
                    rc = self._lib.pgcn_p2p_import(self.handle, packed)
                ok = torch.tensor([1 if rc == 0 else 0], device=cdev)
                dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
                if int(ok.item()) == 1:
                    dist.barrier(group=group)
                    used = "p2p"
            if used is None:
                # not unanimous: a rank whose own import succeeded must not keep storing into peer slabs while
                # the others talk NCCL (the job would hang) — switch the peer transport off everywhere
                self.set_option("p2p", 0)
                if transport == "p2p":
                    cabi.check(rc if rc < 0 else -5, self._h)
        # the NCCL communicator is always created: it is the transport of the step-by-step entry points
        # (pgcn_exchange) and the fallback of the fused ones for widths the peer-store kernels do not take
        # (f % 4 != 0)
        if used == "p2p" and not nccl_fallback:
            # peer-memory only (e.g. several ranks sharing one device, where NCCL cannot be set up): widths the
            # peer-store kernels do not take (f % 4 != 0) then have no transport and raise
            return used
        ident = torch.zeros(cabi.NCCL_ID_BYTES, dtype=torch.uint8)
        if self.lp.rank == 0:
            buf = C.create_string_buffer(cabi.NCCL_ID_BYTES)
            cabi.check(self._lib.pgcn_comm_unique_id(buf), None)
            ident = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        ident = ident.to(cdev)
        dist.broadcast(ident, src=0, group=group)
        raw = bytes(ident.cpu().numpy().tobytes())
        with torch.cuda.device(self.device):
            cabi.check(self._lib.pgcn_comm_init(self.handle, raw), self._h)
        return used or "nccl"

    def share_comm(self, owner):
        """Borrow `owner`'s NCCL communicator (one plan per mini-batch over one process group)."""
        cabi.check(self._lib.pgcn_comm_share(self.handle, owner.handle), self._h)
        self._comm_owner = owner          # keep it alive

    # -- stats, as the reference counts them (rows, messages incl. empty ones) -------------------
    def count_exchange(self, backward=False):
        lp = self.lp
        out_rows = lp.h if backward else lp.S
        in_rows = lp.S if backward else lp.h
        self.stats["send_volume"] += int(out_rows)
        self.stats["recv_volume"] += int(in_rows)
        self.stats["send_nmsg"] += lp.k - 1
        self.stats["recv_nmsg"] += lp.k - 1


def gated_work_table(rowptr, chunk):
    """(items, splits, nslots) of a CSR's row pointer for the gated kernels: items int32 [nitems, 4] of (row, e0, e1,
    slot), first one per chunk of `chunk` entries of every row longer than `chunk` (slots 0, 1, ... in row and chunk
    order), then one per other row, empty rows included (slot -1); splits int32 [nsplits, 3] of (row, first slot,
    chunks) per split row. The split rows' chunks come first so that the longest work starts first."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    deg = np.diff(rowptr)
    long_rows = np.flatnonzero(deg > chunk)
    nch = -(-deg[long_rows] // chunk)
    first = np.cumsum(nch) - nch
    nslots = int(nch.sum())
    crow = np.repeat(long_rows, nch)
    slot = np.arange(nslots, dtype=np.int64)
    e0 = rowptr[crow] + (slot - np.repeat(first, nch)) * chunk
    e1 = np.minimum(e0 + chunk, rowptr[crow + 1])
    short = np.flatnonzero(deg <= chunk)
    items = np.concatenate([np.stack([crow, e0, e1, slot], 1),
                            np.stack([short, rowptr[short], rowptr[short + 1], np.full(len(short), -1)], 1)])
    splits = np.stack([long_rows, first, nch], 1)
    if rowptr[-1] > np.iinfo(np.int32).max:
        raise ValueError("nnz=%d: the gated work table holds entry offsets as int32" % rowptr[-1])
    return items.astype(np.int32).reshape(-1, 4), splits.astype(np.int32).reshape(-1, 3), nslots


class GatedWalk:
    """One walk of the gated kernels on the device: a CSR's entries `idx` and its work table (gated_work_table), with
    `c`, the pgcn_gated_walk that points at them. `nslots` rows of work memory take the split rows' partial sums."""

    def __init__(self, rowptr, idx, chunk, device):
        import torch
        items, splits, self.nslots = gated_work_table(rowptr, chunk)
        self.rows = len(rowptr) - 1
        self.idx = torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int32)).to(device)
        self.items = torch.from_numpy(items).to(device)
        self.splits = torch.from_numpy(splits).to(device)
        self.c = cabi.PgcnGatedWalk(self.idx.data_ptr(), self.items.data_ptr(), self.splits.data_ptr(), self.rows,
                                    len(items), len(splits), self.nslots)


# The tables of the relational aggregation (PgcnPlan.relation_walks): two GatedWalks, perm_f, the mean weights and R.
RelationWalks = collections.namedtuple("RelationWalks", "fwd tr perm_f mean R")


def _values_key(vals):
    return (id(vals), vals.data_ptr(), vals._version)


def check_values(plan, vals):
    """Edge values for `plan`: fp32 CUDA [nnz] on the plan's device. Returns them contiguous."""
    import torch
    if not torch.is_tensor(vals) or not vals.is_cuda:
        raise RuntimeError("edge values must be a CUDA tensor: the PGCN H100 path has no CPU fallback")
    if vals.dtype != torch.float32:
        raise TypeError("edge values must be float32, got %s" % vals.dtype)
    nnz = plan.lp.nnz()
    if vals.dim() != 1 or vals.shape[0] != nnz:
        raise ValueError("edge values must be [%d] (the plan's nnz), got %s" % (nnz, tuple(vals.shape)))
    if vals.device != plan.device:
        raise ValueError("edge values live on %s, the plan on %s" % (vals.device, plan.device))
    return vals.detach().contiguous()


def link_local_plans(plans):
    """All ranks' plans live in THIS process (one GPU or several): wire their peer-memory transports to each other
    directly — export every arena, import the k blobs into every plan (same-process peers are reached through plain
    device pointers, no IPC). Used by the single-box tests and by smoke(); a multi-process job uses init_comm."""
    import torch
    k = len(plans)
    blobs = []
    for p in plans:
        blob = C.create_string_buffer(cabi.P2P_HANDLE_BYTES)
        with torch.cuda.device(p.device):
            cabi.check(p._lib.pgcn_p2p_export(p.handle, blob), p._h)
        blobs.append(blob.raw)
    packed = b"".join(blobs)
    for p in plans:
        assert p.lp.k == k
        with torch.cuda.device(p.device):
            cabi.check(p._lib.pgcn_p2p_import(p.handle, packed), p._h)
    return "p2p"


def build_plan(A, partvec, rank, size, f_max, device=None):
    """a1 + a2 + buffer allocation of the reference's `run` (GPU/PGCN.py:175-182) in one call."""
    return PgcnPlan(build_local_plan(A, partvec, rank, size), f_max, device=device)
