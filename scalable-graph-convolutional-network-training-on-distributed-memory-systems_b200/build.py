"""Build the native pieces in-tree (so the .so files travel to the GPU box with the snapshot).

  lib/libpgcn_b200.so     csrc/pgcn_b200.cu (+ spmm_kernels.cuh, spmm_ring.cuh, sddmm.cuh, attention.cuh, spmm_max.cuh, gatv2.cuh)   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo
  lib/libpgcn_dropout.so  csrc/edge_dropout.cu (+ philox.cuh)                                                                        the same flags
  lib/libpgcn_gated.so    csrc/gated.cu (+ gated_math.cuh)                                                                           the same flags
  lib/libpgcn_transformer.so csrc/transformer.cu (+ transformer_math.cuh, philox.cuh, pgcn_gated.h for the walk struct)               the same flags
  lib/libpgcn_transformer_edge.so csrc/transformer_edge.cu (+ transformer_math.cuh, philox.cuh, pgcn_gated.h)                         the same flags
  lib/libpgcn_gatedgcn.so csrc/gatedgcn.cu (+ gated_math.cuh, pgcn_gated.h for the walk struct)                                       the same flags
  lib/libpgcn_gine.so     csrc/gine.cu (+ gated_math.cuh, pgcn_gated.h for the walk struct)                                           the same flags
  lib/libpgcn_rgcn.so     csrc/rgcn.cu (+ gated_math.cuh, pgcn_gated.h for the walk struct)                                           the same flags
  lib/libpgcn_gatv2_edge.so csrc/gatv2_edge.cu (+ transformer_math.cuh, philox.cuh, pgcn_gated.h)                                     the same flags
  (the CPU oracle under oracle/ is built by oracle/build_oracle.py — test infrastructure only)

nvcc cross-compiles without a GPU; `python -m <pkg>.build` or `__graft_entry__.build()` runs this.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
# PGCN_B200_VARIANT=<name> selects lib/libpgcn_b200_<name>.so built with PGCN_B200_DEFS (tuning
# experiments only, e.g. PGCN_B200_VARIANT=occ0 PGCN_B200_DEFS=-DPGCN_OCC=0); default: no suffix.
_VARIANT = os.environ.get("PGCN_B200_VARIANT", "")
LIB = os.path.join(LIBDIR, "libpgcn_b200%s.so" % ("_" + _VARIANT if _VARIANT else ""))
SOURCES = [os.path.join(CSRC, "pgcn_b200.cu")]
# this file too: a library built with other compiler flags (another GPU architecture) is stale
DEPS = SOURCES + [os.path.join(CSRC, "spmm_kernels.cuh"), os.path.join(CSRC, "spmm_ring.cuh"),
                  os.path.join(CSRC, "sddmm.cuh"), os.path.join(CSRC, "attention.cuh"), os.path.join(CSRC, "spmm_max.cuh"),
                  os.path.join(CSRC, "gatv2.cuh"),
                  os.path.join(ROOT, "include", "pgcn_b200.h"), os.path.join(ROOT, "include", "pgcn_b200_halo.h"),
                  os.path.abspath(__file__)]
# the edge-dropout library has its own sources and dependency list: editing one library never rebuilds the other
DROPOUT_LIB = os.path.join(LIBDIR, "libpgcn_dropout.so")
DROPOUT_SOURCES = [os.path.join(CSRC, "edge_dropout.cu")]
DROPOUT_DEPS = DROPOUT_SOURCES + [os.path.join(CSRC, "philox.cuh"), os.path.join(ROOT, "include", "pgcn_dropout.h"),
                                  os.path.abspath(__file__)]
# so has the gated-aggregation library
GATED_LIB = os.path.join(LIBDIR, "libpgcn_gated.so")
GATED_SOURCES = [os.path.join(CSRC, "gated.cu")]
GATED_DEPS = GATED_SOURCES + [os.path.join(CSRC, "gated_math.cuh"), os.path.join(ROOT, "include", "pgcn_gated.h"),
                              os.path.abspath(__file__)]
# and the transformer-attention library, which takes the gated library's walk struct and the dropout's Philox
TRANSFORMER_LIB = os.path.join(LIBDIR, "libpgcn_transformer.so")
TRANSFORMER_SOURCES = [os.path.join(CSRC, "transformer.cu")]
TRANSFORMER_DEPS = TRANSFORMER_SOURCES + [os.path.join(CSRC, "transformer_math.cuh"), os.path.join(CSRC, "philox.cuh"),
                                          os.path.join(ROOT, "include", "pgcn_transformer.h"),
                                          os.path.join(ROOT, "include", "pgcn_gated.h"), os.path.abspath(__file__)]
# and the GatedGCN library, which takes the gated library's walk struct and its gate (gated_math.cuh)
GATEDGCN_LIB = os.path.join(LIBDIR, "libpgcn_gatedgcn.so")
GATEDGCN_SOURCES = [os.path.join(CSRC, "gatedgcn.cu")]
GATEDGCN_DEPS = GATEDGCN_SOURCES + [os.path.join(CSRC, "gated_math.cuh"),
                                    os.path.join(ROOT, "include", "pgcn_gatedgcn.h"),
                                    os.path.join(ROOT, "include", "pgcn_gated.h"), os.path.abspath(__file__)]
# and the transformer attention with edge features, which shares the transformer's lane math (transformer_math.cuh)
TRANSFORMER_EDGE_LIB = os.path.join(LIBDIR, "libpgcn_transformer_edge.so")
TRANSFORMER_EDGE_SOURCES = [os.path.join(CSRC, "transformer_edge.cu")]
TRANSFORMER_EDGE_DEPS = TRANSFORMER_EDGE_SOURCES + [os.path.join(CSRC, "transformer_math.cuh"),
                                                    os.path.join(CSRC, "philox.cuh"),
                                                    os.path.join(ROOT, "include", "pgcn_transformer_edge.h"),
                                                    os.path.join(ROOT, "include", "pgcn_gated.h"),
                                                    os.path.abspath(__file__)]
# and GINE, which takes the gated library's walk struct and its lane loads (gated_math.cuh)
GINE_LIB = os.path.join(LIBDIR, "libpgcn_gine.so")
GINE_SOURCES = [os.path.join(CSRC, "gine.cu")]
GINE_DEPS = GINE_SOURCES + [os.path.join(CSRC, "gated_math.cuh"), os.path.join(ROOT, "include", "pgcn_gine.h"),
                            os.path.join(ROOT, "include", "pgcn_gated.h"), os.path.abspath(__file__)]
# and R-GCN's relational aggregation, which takes the same walk struct and lane loads
RGCN_LIB = os.path.join(LIBDIR, "libpgcn_rgcn.so")
RGCN_SOURCES = [os.path.join(CSRC, "rgcn.cu")]
RGCN_DEPS = RGCN_SOURCES + [os.path.join(CSRC, "gated_math.cuh"), os.path.join(ROOT, "include", "pgcn_rgcn.h"),
                            os.path.join(ROOT, "include", "pgcn_gated.h"), os.path.abspath(__file__)]
# and GATv2 with edge features, which takes the transformer's lane math (transformer_math.cuh) and the same walk struct
GATV2_EDGE_LIB = os.path.join(LIBDIR, "libpgcn_gatv2_edge.so")
GATV2_EDGE_SOURCES = [os.path.join(CSRC, "gatv2_edge.cu")]
GATV2_EDGE_DEPS = GATV2_EDGE_SOURCES + [os.path.join(CSRC, "transformer_math.cuh"), os.path.join(CSRC, "philox.cuh"),
                                        os.path.join(ROOT, "include", "pgcn_gatv2_edge.h"),
                                        os.path.join(ROOT, "include", "pgcn_gated.h"), os.path.abspath(__file__)]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _stale(lib, deps):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def is_stale():
    return _stale(LIB, DEPS)


def dropout_is_stale():
    return _stale(DROPOUT_LIB, DROPOUT_DEPS)


def gated_is_stale():
    return _stale(GATED_LIB, GATED_DEPS)


def transformer_is_stale():
    return _stale(TRANSFORMER_LIB, TRANSFORMER_DEPS)


def gatedgcn_is_stale():
    return _stale(GATEDGCN_LIB, GATEDGCN_DEPS)


def transformer_edge_is_stale():
    return _stale(TRANSFORMER_EDGE_LIB, TRANSFORMER_EDGE_DEPS)


def gine_is_stale():
    return _stale(GINE_LIB, GINE_DEPS)


def rgcn_is_stale():
    return _stale(RGCN_LIB, RGCN_DEPS)


def gatv2_edge_is_stale():
    return _stale(GATV2_EDGE_LIB, GATV2_EDGE_DEPS)


def _compile(lib, sources, defs, verbose):
    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build %s (no prebuilt library either)" % os.path.basename(lib))
    os.makedirs(LIBDIR, exist_ok=True)
    tmp = lib + ".tmp.%d" % os.getpid()
    cmd = [nvcc] + NVCC_FLAGS + defs + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + sources + ["-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        sys.stderr.write(res.stderr)
    os.replace(tmp, lib)
    return lib


def build(force=False, verbose=False):
    """Compile libpgcn_b200.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not is_stale():
        return LIB
    return _compile(LIB, SOURCES, os.environ.get("PGCN_B200_DEFS", "").split() if _VARIANT else [], verbose)


def build_dropout(force=False, verbose=False):
    """Compile libpgcn_dropout.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not dropout_is_stale():
        return DROPOUT_LIB
    return _compile(DROPOUT_LIB, DROPOUT_SOURCES, [], verbose)


def build_gated(force=False, verbose=False):
    """Compile libpgcn_gated.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not gated_is_stale():
        return GATED_LIB
    return _compile(GATED_LIB, GATED_SOURCES, [], verbose)


def build_transformer(force=False, verbose=False):
    """Compile libpgcn_transformer.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not transformer_is_stale():
        return TRANSFORMER_LIB
    return _compile(TRANSFORMER_LIB, TRANSFORMER_SOURCES, [], verbose)


def build_gatedgcn(force=False, verbose=False):
    """Compile libpgcn_gatedgcn.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not gatedgcn_is_stale():
        return GATEDGCN_LIB
    return _compile(GATEDGCN_LIB, GATEDGCN_SOURCES, [], verbose)


def build_transformer_edge(force=False, verbose=False):
    """Compile libpgcn_transformer_edge.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not transformer_edge_is_stale():
        return TRANSFORMER_EDGE_LIB
    return _compile(TRANSFORMER_EDGE_LIB, TRANSFORMER_EDGE_SOURCES, [], verbose)


def build_gine(force=False, verbose=False):
    """Compile libpgcn_gine.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not gine_is_stale():
        return GINE_LIB
    return _compile(GINE_LIB, GINE_SOURCES, [], verbose)


def build_rgcn(force=False, verbose=False):
    """Compile libpgcn_rgcn.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not rgcn_is_stale():
        return RGCN_LIB
    return _compile(RGCN_LIB, RGCN_SOURCES, [], verbose)


def build_gatv2_edge(force=False, verbose=False):
    """Compile libpgcn_gatv2_edge.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not gatv2_edge_is_stale():
        return GATV2_EDGE_LIB
    return _compile(GATV2_EDGE_LIB, GATV2_EDGE_SOURCES, [], verbose)


if __name__ == "__main__":
    force, verbose = "--force" in sys.argv, "-v" in sys.argv
    print(build(force=force, verbose=verbose))
    print(build_dropout(force=force, verbose=verbose))
    print(build_gated(force=force, verbose=verbose))
    print(build_transformer(force=force, verbose=verbose))
    print(build_gatedgcn(force=force, verbose=verbose))
    print(build_transformer_edge(force=force, verbose=verbose))
    print(build_gine(force=force, verbose=verbose))
    print(build_rgcn(force=force, verbose=verbose))
    print(build_gatv2_edge(force=force, verbose=verbose))
