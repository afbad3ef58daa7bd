#!/usr/bin/env python
"""List the kernels of lib/libpgcn_b200.so, one per line, demangled and sorted (tests/kernel_instances.txt).

    python tools/list_kernels.py                 # print the list
    python tools/list_kernels.py --write         # rewrite tests/kernel_instances.txt

The list comes from `cuobjdump -symbols` (the kernel entries, STO_ENTRY) and `cu++filt`, both taken from the toolkit
whose nvcc builds the library. A new kernel instance needs a line in the manifest and a row in the census's route
table (tests/test_kernel_census.py), which launches every listed instance and checks it against fp64.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MANIFEST = os.path.join(ROOT, "tests", "kernel_instances.txt")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def cuda_tool(name):
    """Path of a CUDA toolkit binary next to the nvcc the build uses, or None."""
    from pgcn_b200 import build
    nvcc = build._nvcc()
    cands = [os.path.join(os.path.dirname(nvcc), name)] if nvcc else []
    cands += [shutil.which(name), os.path.join("/usr/local/cuda/bin", name)]
    for c in cands:
        if c and os.path.exists(c):
            return c
    return None


def list_kernels(lib=None):
    """The demangled kernel names of the library, sorted, `[clone ...]` entries dropped."""
    if lib is None:
        from pgcn_b200 import build
        lib = build.LIB
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        raise FileNotFoundError("cuobjdump / cu++filt not found")
    out = subprocess.run([cuobjdump, "-symbols", lib], capture_output=True, text=True, check=True).stdout
    syms = [ln.split()[-1] for ln in out.splitlines() if "STO_ENTRY" in ln]
    names = subprocess.run([cufilt], input="\n".join(syms) + "\n", capture_output=True, text=True,
                           check=True).stdout.splitlines()
    return sorted(set(n.strip() for n in names if n.strip() and "[clone" not in n))


def main():
    text = "".join(n + "\n" for n in list_kernels())
    if "--write" in sys.argv:
        with open(MANIFEST, "w") as fh:
            fh.write(text)
        print("%s: %d kernels" % (MANIFEST, text.count("\n")))
    else:
        sys.stdout.write(text)


if __name__ == "__main__":
    main()
