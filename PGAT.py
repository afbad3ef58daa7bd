#!/usr/bin/env python
"""Drop-in launcher with the reference's name and flags (GPU/PGAT.py):
    python PGAT.py -a A.mtx -p A.mtx.<k>.<hp|gp|rp> -b nccl -s <k> -l <layers> -f <features> [--negative-slope 0.2] [--heads K] [--attn-dropout P] [--v2 [--edge-values]]
One process per GPU; rank/size from SLURM_PROCID/SLURM_NPROCS or RANK/WORLD_SIZE (torchrun)."""
import sys

import pgcn_b200  # noqa: F401  (import shim for the hyphenated package directory)
from pgcn_b200.pgat import main

if __name__ == "__main__":
    main(sys.argv[1:])
