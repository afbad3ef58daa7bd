#!/usr/bin/env python
"""Residual gated graph convolutions (ResGatedGraphConv), launched like PGCN.py, PGAT.py and PSAGE.py:
    python PGATED.py -a A.mtx -p A.mtx.<k>.<hp|gp|rp> -b nccl -s <k> -l <layers> -f <features> [--seed N]
One process per GPU; rank/size from SLURM_PROCID/SLURM_NPROCS or RANK/WORLD_SIZE (torchrun)."""
import sys

import pgcn_b200  # noqa: F401  (import shim for the hyphenated package directory)
from pgcn_b200.gated import main

if __name__ == "__main__":
    main(sys.argv[1:])
