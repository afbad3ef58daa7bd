#!/usr/bin/env python
"""GINE layers with an edge-feature stream, launched like PGCN.py, PGAT.py, PSAGE.py and PGATEDGCN.py:
    python PGINE.py -a A.mtx -p A.mtx.<k>.<hp|gp|rp> -b nccl -s <k> -l <layers> -f <features> [--seed N]
One process per GPU; rank/size from SLURM_PROCID/SLURM_NPROCS or RANK/WORLD_SIZE (torchrun)."""
import sys

import pgcn_b200  # noqa: F401  (import shim for the hyphenated package directory)
from pgcn_b200.gine import main

if __name__ == "__main__":
    main(sys.argv[1:])
