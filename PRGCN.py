#!/usr/bin/env python
"""R-GCN layers over typed edges, launched like PGCN.py, PGAT.py, PSAGE.py, PGATEDGCN.py and PGINE.py:
    python PRGCN.py -a A.mtx -p A.mtx.<k>.<hp|gp|rp> -b nccl -s <k> -l <layers> -f <features> --relations <R>
                    [--bases <B>] [--seed N]
One process per GPU; rank/size from SLURM_PROCID/SLURM_NPROCS or RANK/WORLD_SIZE (torchrun)."""
import sys

import pgcn_b200  # noqa: F401  (import shim for the hyphenated package directory)
from pgcn_b200.rgcn import main

if __name__ == "__main__":
    main(sys.argv[1:])
