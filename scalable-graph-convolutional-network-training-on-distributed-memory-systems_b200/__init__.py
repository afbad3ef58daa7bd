"""pgcn_b200 — H100-native drop-in for the PGCN aggregation hot path
(Z = A_local * H + halo exchange; reference GPU/PGCN.py:85-134).

Importable as `pgcn_b200` through the shim at the repo root (the directory name contains
hyphens). Sub-modules: build (nvcc), cabi (ctypes over include/pgcn_b200.h), graphio (formats +
synthetic inputs), plan (loader/plan builder), op (PSpMM autograd op), pgcn (CLI clone),
minibatch (host-side loader of the mini-batch variant).
"""
from . import build, cabi, graphio, plan  # noqa: F401
from .plan import (PgcnPlan, LocalPlan, build_local_plan, build_plan,  # noqa: F401
                   compute_communication_maps, get_partition_of_adjacency_matrix,
                   get_partitiont_of_adjacency_matrix)

__version__ = "0.1"


def __getattr__(name):
    # torch-dependent pieces are imported lazily so `import pgcn_b200` stays cheap
    if name in ("op", "pgcn", "pgat", "minibatch"):
        import importlib
        return importlib.import_module("." + name, __name__)
    if name in ("PSpMM", "PSpMMWeighted", "PGATAttention", "PGATMultiHeadAttention", "aggregate_forward",
                "aggregate_backward"):
        from . import op
        return getattr(op, name)
    raise AttributeError(name)
