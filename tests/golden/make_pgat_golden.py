"""Generate tests/golden/pgat_*.npz by running the UNMODIFIED reference graph-attention layer (GPU/PGAT.py).

Run in the build container (the reference is mounted read-only there; it does not exist on the GPU machine):
    python tests/golden/make_pgat_golden.py

For every case one gloo process per rank imports the reference module, sets the module globals its `run` sets
(GPU/PGAT.py:160-183: rank, world size, communication maps, buffers, X), builds 1 and 2 PGAT layers with seeded
parameters, and records the rank's logits (n x f), its loss (mean nll over all n rows, labels i % f) and the gradients
of W and a of every layer before averaging. Cases: karate on one rank and on three ranks (the pickled 3-way vector),
and the gcn-normalised gemat11 on one rank. Inputs are seeded uniform [-1, 1) rows (not the reference's H[i] = i,
whose scores of size n saturate every softmax), stored with the parameters, so tests/test_pgat_oracle.py can replay
oracle/pgat_oracle.py's `literal` mode on them without the reference.
"""
import importlib.util
import os
import pickle
import sys

import numpy as np
import scipy.sparse as sp
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F
from scipy.io import mmread

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
SEED = 20261015


def load_reference():
    spec = importlib.util.spec_from_file_location("ref_pgat", os.path.join(REF, "GPU", "PGAT.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def worker(rank, size, port, row, col, val, n, partvec, f, tag):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=size)
    from oracle import pgat_oracle
    ref = load_reference()
    ref.myrank, ref.world_size = rank, size
    ref.device = torch.device("cpu")
    A = sp.coo_matrix((val, (row, col)), shape=(n, n))
    ref.send_map, ref.recv_map = ref.compute_communication_maps(A, partvec, rank, size)
    Ad = ref.get_partitiont_of_adjacency_matrix(A, partvec, rank)
    ref.send_buffers, ref.recv_buffers = {}, {}
    for source, idx in ref.recv_map.items():
        ref.recv_buffers[source] = torch.zeros(len(idx), f)
    for target, idx in ref.send_map.items():
        ref.send_buffers[target] = torch.zeros(len(idx), f)
    H0 = np.random.RandomState(SEED).uniform(-1.0, 1.0, size=(n, f)).astype(np.float32)
    labels = torch.arange(n) % f
    rec = {}
    for L in (1, 2):
        params = pgat_oracle.init_params(L, f, SEED + L)
        ref.X = torch.zeros(n, f)
        H = torch.tensor(H0, requires_grad=True)
        model = nn.Sequential(*[ref.PGAT(Ad, f, f) for _ in range(L)])
        with torch.no_grad():
            for layer, (W, a) in zip(model, params):
                layer.linear.weight.copy_(torch.from_numpy(W))
                layer.attention.copy_(torch.from_numpy(a))
        logits = model(H)
        loss = F.nll_loss(F.log_softmax(logits, 1), labels)
        loss.backward()
        rec["L%d_logits" % L] = logits.detach().numpy()
        rec["L%d_loss" % L] = np.array(float(loss))
        for i, layer in enumerate(model):
            rec["L%d_dW%d" % (L, i)] = layer.linear.weight.grad.numpy()
            rec["L%d_da%d" % (L, i)] = layer.attention.grad.numpy()
    np.savez(os.path.join(HERE, "_tmp_%s_r%d.npz" % (tag, rank)), **rec)
    dist.destroy_process_group()


def run_case(tag, A, partvec, f, port):
    A = sp.coo_matrix(A)
    k = int(max(partvec)) + 1
    n = A.shape[0]
    args = (k, port, A.row, A.col, A.data, n, [int(p) for p in partvec], f, tag)
    mp.spawn(worker, args=args, nprocs=k, join=True)
    out = {"n": np.array(n), "k": np.array(k), "f": np.array(f), "seed": np.array(SEED),
           "row": A.row.astype(np.int32), "col": A.col.astype(np.int32), "val": A.data.astype(np.float64),
           "partvec": np.array(partvec, dtype=np.int32),
           "H": np.random.RandomState(SEED).uniform(-1.0, 1.0, size=(n, f)).astype(np.float32)}
    for r in range(k):
        path = os.path.join(HERE, "_tmp_%s_r%d.npz" % (tag, r))
        z = np.load(path)
        for key in z.files:
            out["r%d_%s" % (r, key)] = z[key]
        os.remove(path)
    np.savez_compressed(os.path.join(HERE, "pgat_%s.npz" % tag), **out)
    print("wrote pgat_%s.npz" % tag)


def main():
    from pgcn_b200 import graphio
    kar = mmread(os.path.join(REF, "GPU/SHP/data/karate/karate.mtx")).tocoo()
    khp = [int(p) for p in pickle.load(open(os.path.join(REF, "GPU/SHP/data/partvec.hp.3"), "rb"))]
    gem = graphio.gcn_normalise(mmread(os.path.join(REF, "GPU/hypergraph/data/gemat11/gemat11.mtx")))
    run_case("karate_k1", kar, [0] * kar.shape[0], 4, 29710)
    run_case("karate_k3", kar, khp, 4, 29711)
    run_case("gemat11_k1", gem, [0] * gem.shape[0], 8, 29712)


if __name__ == "__main__":
    main()
