"""Scratch timing: the three grid builds (options.binning 1 = cell-wise grid-wide passes, 2 = one CTA per
cloud, 3 = slab build) for single pairs of several sizes and for batches."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from timing import timeit
import pcu_b200 as pcu

I = pcu._pcu_internal

g = torch.Generator(device="cuda").manual_seed(0)
for n in (1024, 4096, 16384, 32768, 65536, 100000, 1000000):
    x = torch.rand((n, 3), generator=g, device="cuda"); y = torch.rand((n, 3), generator=g, device="cuda")
    row = []
    for mode in (1, 2, 3):
        I._set_defaults(binning=mode)
        row.append(timeit(lambda: pcu.chamfer_distance(x, y), it=15, flush=False)[0])
    print("pair n=%7d: passes %.4f ms  one-CTA %.4f ms  slabs %.4f ms" % (n, row[0], row[1], row[2]), flush=True)
for B, n in ((8, 16384), (32, 4096), (64, 65536), (1024, 65536)):
    xb = torch.rand((B, n, 3), generator=g, device="cuda"); yb = torch.rand((B, n, 3), generator=g, device="cuda")
    row = []
    for mode in (1, 2, 3):
        I._set_defaults(binning=mode)
        row.append(timeit(lambda: pcu.batched_chamfer_distance(xb, yb), warm=2, it=5, flush=False)[0])
    print("batch %4d x %6d: passes %.4f ms  one-CTA %.4f ms  slabs %.4f ms" % (B, n, row[0], row[1], row[2]), flush=True)
    del xb, yb
I._set_defaults()
