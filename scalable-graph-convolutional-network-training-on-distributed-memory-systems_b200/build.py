"""Build the native pieces in-tree (so the .so files travel to the GPU box with the snapshot).

  lib/libpgcn_b200.so   csrc/pgcn_b200.cu (+ spmm_kernels.cuh, spmm_ring.cuh, sddmm.cuh, attention.cuh, spmm_max.cuh, gatv2.cuh)   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo
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
                  os.path.join(ROOT, "include", "pgcn_b200.h"), os.path.abspath(__file__)]

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


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile libpgcn_b200.so for sm_90a if missing or older than its sources. Returns its path."""
    if not force and not is_stale():
        return LIB
    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libpgcn_b200.so (no prebuilt library either)")
    os.makedirs(LIBDIR, exist_ok=True)
    tmp = LIB + ".tmp.%d" % os.getpid()
    defs = os.environ.get("PGCN_B200_DEFS", "").split() if _VARIANT else []
    cmd = [nvcc] + NVCC_FLAGS + defs + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES + ["-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        sys.stderr.write(res.stderr)
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
