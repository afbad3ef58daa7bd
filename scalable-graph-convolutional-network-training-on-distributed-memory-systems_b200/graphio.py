"""Input formats of the PGCN path and the synthetic inputs of the benchmark configs.

Formats kept from the reference (SURVEY.md §8b "Input formats"):
  * adjacency: MatrixMarket coordinate file, whatever scipy.io.mmread accepts   GPU/PGCN.py:171
  * part vector: FIRST line of whitespace-separated ints, length n               GPU/PGCN.py:172-173
    (writer: GPU/hypergraph/main.cpp:51-63 — "%d " per vertex then a newline)
Synthetic inputs (SURVEY.md §8d): R-MAT graph, symmetrised, self-loops removed, then the
reference preprocessing A^ = Dr^-1/2 (A + I) Dc^-1/2                  preprocess/GrB-GNN-IDG.py:45-68
"""
import os

import numpy as np
import scipy.sparse as sp
from scipy.io import mmread


def read_adjacency(path):
    """scipy COO (global n x n), exactly what GPU/PGCN.py:171 hands to the plan builder.
    A `.npz` written by save_adjacency_npz is accepted too (fast path for 1e8-edge graphs)."""
    if path.endswith(".npz"):
        z = np.load(path)
        n = int(z["n"])
        return sp.coo_matrix((z["data"], (z["row"], z["col"])), shape=(n, n))
    A = mmread(path)
    return A.tocoo()


def save_adjacency_npz(path, A):
    A = A.tocoo()
    np.savez(path, n=A.shape[0], row=A.row.astype(np.int32), col=A.col.astype(np.int32),
             data=A.data.astype(np.float32))


def read_partvec(path, n=None):
    """First line, whitespace-separated ints (GPU/PGCN.py:172-173)."""
    with open(path) as f:
        pv = np.array(f.readline().split(), dtype=np.int64)
    if n is not None and pv.shape[0] != n:
        raise ValueError("part vector has %d entries, matrix has %d rows" % (pv.shape[0], n))
    return pv


def write_partvec(path, partvec):
    """Same bytes as GPU/hypergraph/main.cpp:51-63."""
    with open(path, "w") as f:
        f.write("".join("%d " % int(p) for p in partvec))
        f.write("\n")


def check_partvec(partvec, size):
    """The reference fails with KeyError on a part id >= size (SURVEY.md §8b); same here, earlier."""
    pv = np.asarray(partvec)
    if pv.size and (pv.min() < 0 or pv.max() >= size):
        bad = int(pv.max() if pv.max() >= size else pv.min())
        raise KeyError(bad)
    return pv


# ------------------------------------------------------------------------------------------
# on-disk formats of the CPU path (GCN-HP/main.cpp writers -> Parallel-GCN/main.c readers)
# ------------------------------------------------------------------------------------------

def read_cpu_config(path):
    """`config`: "nlayers n f ... f fout" (GCN-HP/main.cpp:117-131, parsed by Parallel-GCN/main.c:687-698)."""
    vals = [int(x) for x in open(path).read().split()]
    return {"nlayers": vals[0], "n": vals[1], "widths": vals[2:]}


def read_cpu_matrix_part(path):
    """`A.k` / `Y.k`: header "n nnz_k", then "i j val" with 0-based GLOBAL indices, values printed %.2f
    (GCN-HP/main.cpp:213-249; read by Parallel-GCN/main.c:609-647). Returns (n, row, col, val)."""
    with open(path) as f:
        n, nnz = [int(x) for x in f.readline().split()]
        data = np.loadtxt(f, dtype=np.float64, ndmin=2) if nnz else np.zeros((0, 3))
    if data.shape[0] != nnz:
        raise ValueError("%s: header says %d entries, file has %d" % (path, nnz, data.shape[0]))
    return n, data[:, 0].astype(np.int64), data[:, 1].astype(np.int64), data[:, 2].astype(np.float32)


def read_cpu_rows_part(path):
    """`H.k`: the number of rows of part k, then one owned global row id per line
    (GCN-HP/main.cpp:251-282; Parallel-GCN/main.c:650-684 sets H0 = 1.0 on exactly these rows)."""
    vals = np.array(open(path).read().split(), dtype=np.int64)
    if vals.size == 0 or vals[0] != vals.size - 1:
        raise ValueError("%s: row count does not match" % path)
    return vals[1:]


def read_cpu_conn(path):
    """`conn.k`: "nsend nrecv", then one line per target: "target count id id ..." — the vertices part k
    sends to each target (GCN-HP/main.cpp:147-185; Parallel-GCN/main.c:526-551). Returns {target: ids}."""
    lines = open(path).read().splitlines()
    nsend, _ = [int(x) for x in lines[0].split()]
    out = {}
    for line in lines[1:1 + nsend]:
        v = [int(x) for x in line.split()]
        if len(v) != 2 + v[1]:
            raise ValueError("%s: malformed target line" % path)
        out[v[0]] = np.array(v[2:], dtype=np.int64)
    return out


def read_cpu_buff(path):
    """`buff.k`: "nsend (target count)*" newline "nrecv (source count)*" (GCN-HP/main.cpp:187-209;
    Parallel-GCN/main.c:456-504). Returns ({target: rows_out}, {source: rows_in})."""
    l0, l1 = (open(path).read().split("\n") + [""])[:2]
    a = [int(x) for x in l0.split()]
    b = [int(x) for x in l1.split()]
    send = {a[1 + 2 * i]: a[2 + 2 * i] for i in range(a[0])} if a else {}
    recv = {b[1 + 2 * i]: b[2 + 2 * i] for i in range(b[0])} if b else {}
    return send, recv


def read_cpu_partition(dirpath, k):
    """Everything `gcnhgp -o dir -k k` wrote, as the inputs of the H100 path: the global adjacency (union of the
    A.k blocks, scipy COO) and the part vector (from the H.k row lists), plus the parsed conn/buff files so a
    caller can compare the reference's connectivity with the one the plan builder derives from A.
    Note: the reference derives `conn` from the OUT-entries of a vertex (owner(i) sends i to owner(j) for A[i][j] != 0,
    GCN-HP/main.cpp:154-170) — the transpose of what row-wise aggregation needs; the two agree when the pattern
    is symmetric (which the reference preprocessing produces for symmetric inputs)."""
    rows, cols, vals, n = [], [], [], None
    partvec = None
    conn, buff = [], []
    for r in range(k):
        nn, i, j, v = read_cpu_matrix_part(os.path.join(dirpath, "A.%d" % r))
        n = nn if n is None else n
        if nn != n:
            raise ValueError("A.%d: inconsistent n" % r)
        rows.append(i); cols.append(j); vals.append(v)
        own = read_cpu_rows_part(os.path.join(dirpath, "H.%d" % r))
        if partvec is None:
            partvec = np.full(n, -1, dtype=np.int64)
        if (partvec[own] != -1).any():
            raise ValueError("H.%d: a row is owned twice" % r)
        partvec[own] = r
        if not np.isin(i, own).all():
            raise ValueError("A.%d holds rows that H.%d does not list" % (r, r))
        conn.append(read_cpu_conn(os.path.join(dirpath, "conn.%d" % r)))
        buff.append(read_cpu_buff(os.path.join(dirpath, "buff.%d" % r)))
    if (partvec < 0).any():
        raise ValueError("%d vertices are in no H.k file" % int((partvec < 0).sum()))
    A = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    return {"A": A, "partvec": partvec, "conn": conn, "buff": buff,
            "config": read_cpu_config(os.path.join(dirpath, "config"))}


# ------------------------------------------------------------------------------------------
# synthetic graphs
# ------------------------------------------------------------------------------------------

def rmat_edges(n, n_undirected, abcd=(0.57, 0.19, 0.19, 0.05), seed=1, permute=True):
    """`n_undirected` distinct undirected edges {u,v}, u != v, of an R-MAT graph on n vertices.

    scale = ceil(log2 n); endpoints >= n are dropped; draws continue until enough distinct edges
    exist, then exactly n_undirected are kept. Vertex ids are randomly permuted (Graph500 style)
    unless permute=False, so no locality comes for free from the generator's bit structure.
    """
    rng = np.random.default_rng(seed)
    scale = max(1, int(np.ceil(np.log2(max(n, 2)))))
    a, b, c, _ = abcd
    keys = np.empty(0, dtype=np.int64)
    want = int(n_undirected)
    draw = int(want * 1.25) + 1024
    it = np.int32 if scale <= 30 else np.int64                 # endpoint bits fit 32-bit words up to 2^30 vertices
    while True:
        u = np.zeros(draw, dtype=it)
        v = np.zeros(draw, dtype=it)
        for _ in range(scale):
            r = rng.random(draw)
            ubit = r >= (a + b)
            vbit = ((r >= a) & (r < a + b)) | (r >= a + b + c)
            u <<= 1; u |= ubit
            v <<= 1; v |= vbit
        ok = (u < n) & (v < n) & (u != v)
        u, v = u[ok].astype(np.int64), v[ok].astype(np.int64)
        lo, hi = np.minimum(u, v), np.maximum(u, v)
        before = keys.shape[0]
        # sorted distinct keys (sort + neighbour compare: several times faster than np.unique's hash path at 1e8 keys)
        keys = np.concatenate([keys, lo * n + hi])
        keys.sort()
        if keys.shape[0] > 1:
            keep = np.empty(keys.shape[0], dtype=bool)
            keep[0] = True
            np.not_equal(keys[1:], keys[:-1], out=keep[1:])
            keys = keys[keep]
        if keys.shape[0] >= want:
            break
        # next round: size the draw by the acceptance rate just observed (dense, skewed graphs such as the
        # Reddit-shaped C4 reject most draws as duplicates once the hub neighbourhoods fill up)
        accept = max((keys.shape[0] - before) / float(draw), 0.02)
        draw = int(min((want - keys.shape[0]) / accept * 1.3 + 1024, 4.0e8))
    if keys.shape[0] > want:
        keys = keys[np.sort(rng.permutation(keys.shape[0])[:want])]
    lo, hi = keys // n, keys % n
    if permute:
        perm = rng.permutation(n)
        lo, hi = perm[lo], perm[hi]
    return lo.astype(np.int64), hi.astype(np.int64)


def symmetric_pattern(n, lo, hi):
    """COO pattern with both directions of every undirected edge (values 1.0, no diagonal)."""
    row = np.concatenate([lo, hi])
    col = np.concatenate([hi, lo])
    return sp.coo_matrix((np.ones(row.shape[0], dtype=np.float32), (row, col)), shape=(n, n))


def gcn_normalise(A):
    """A^ = Dr^-1/2 (A + I) Dc^-1/2 with the diagonal of A dropped first
    (preprocess/GrB-GNN-IDG.py:45-68). Returns float32 COO."""
    A = sp.coo_matrix(A)
    keep = A.row != A.col
    n = A.shape[0]
    row = np.concatenate([A.row[keep], np.arange(n)])
    col = np.concatenate([A.col[keep], np.arange(n)])
    dat = np.concatenate([A.data[keep].astype(np.float64), np.ones(n)])
    B = sp.coo_matrix((dat, (row, col)), shape=(n, n))
    col_sum = np.asarray(B.sum(axis=0)).reshape(-1)
    row_sum = np.asarray(B.sum(axis=1)).reshape(-1)
    dc = 1.0 / np.sqrt(col_sum)
    dr = 1.0 / np.sqrt(row_sum)
    val = (dr[B.row] * B.data * dc[B.col]).astype(np.float32)
    return sp.coo_matrix((val, (B.row.astype(np.int64), B.col.astype(np.int64))), shape=(n, n))


def synthetic_graph(n, nnz, abcd=(0.57, 0.19, 0.19, 0.05), seed=1, permute=True):
    """The benchmark adjacency: R-MAT with `nnz` stored entries before +I (nnz/2 undirected edges),
    symmetrised, normalised like the reference preprocessing. nnz(A^) = nnz + n."""
    lo, hi = rmat_edges(n, nnz // 2, abcd=abcd, seed=seed, permute=permute)
    return gcn_normalise(symmetric_pattern(n, lo, hi))


def random_partvec(n, k, seed=1):
    """`rp` vectors: uniform random parts (GPU/hypergraph/main.cpp:134 partition_random)."""
    if k == 1:
        return np.zeros(n, dtype=np.int64)
    return np.random.default_rng(seed).integers(0, k, size=n, dtype=np.int64)


def block_partvec(n, k):
    """Contiguous equal blocks of vertex ids (a cheap stand-in when no partitioner output exists)."""
    return (np.arange(n, dtype=np.int64) * k // max(n, 1)).astype(np.int64)


CONFIGS = {
    # name: (n, nnz before +I, f, layers, abcd)      BASELINE.json "configs" / SURVEY.md §8d
    "C1": (2708, 10556, 16, 2, (0.57, 0.19, 0.19, 0.05)),
    "C2": (1_000_000, 16_000_000, 128, 2, (0.57, 0.19, 0.19, 0.05)),
    "C3": (2_400_000, 62_000_000, 128, 3, (0.45, 0.22, 0.22, 0.11)),
    "C4": (233_000, 114_000_000, 256, 2, (0.57, 0.19, 0.19, 0.05)),
    "C5": (10_000_000, 100_000_000, 128, 3, (0.57, 0.19, 0.19, 0.05)),
}


def config_graph(name, cache_dir=None, seed=1):
    """Adjacency of a named config, cached as .npz under cache_dir when given."""
    n, nnz, _, _, abcd = CONFIGS[name]
    path = None
    if cache_dir:
        os.makedirs(cache_dir, exist_ok=True)
        path = os.path.join(cache_dir, "%s_seed%d.npz" % (name, seed))
        if os.path.exists(path):
            return read_adjacency(path)
    A = synthetic_graph(n, nnz, abcd=abcd, seed=seed)
    if path:
        tmp = path + ".%d.tmp.npz" % os.getpid()
        save_adjacency_npz(tmp, A)
        os.replace(tmp, path)
    return A
