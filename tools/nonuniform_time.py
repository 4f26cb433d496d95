"""Chamfer timing on non-uniform clouds (sphere surface, planar patch, gaussian blobs) vs uniform."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from timing import timeit
import pcu_b200 as pcu

n = 1000000
g = torch.Generator(device="cuda").manual_seed(0)
def sphere(): v = torch.randn((n, 3), generator=g, device="cuda"); return v / v.norm(dim=1, keepdim=True) * 0.5
def plane(): v = torch.rand((n, 3), generator=g, device="cuda"); v[:, 2] = 0.3 + 0.001 * v[:, 2]; return v
def blobs(): c = torch.rand((64, 3), generator=g, device="cuda"); return c[torch.randint(0, 64, (n,), generator=g, device="cuda")] + 0.01 * torch.randn((n, 3), generator=g, device="cuda")
for name, mk in (("uniform", lambda: torch.rand((n, 3), generator=g, device="cuda")), ("sphere", sphere), ("plane", plane), ("blobs", blobs)):
    x, y = mk(), mk()
    # call by call: the grid-sizing feedback refines the grid from the second call on
    seq = []
    for call in range(8):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); pcu.chamfer_distance(x, y); b.record(); torch.cuda.synchronize()
        seq.append("%.3f" % a.elapsed_time(b))
    ms = timeit(lambda: pcu.chamfer_distance(x, y), flush=False)[0]
    print("%-8s calls %s  steady %.3f ms -> %.3e qpts/s  refinement %s" % (name, " ".join(seq), ms, 2 * n / ms * 1e3, pcu._pcu_internal._grid_refinement()), flush=True)
