"""Scratch timing of the device-resident paths (CUDA events, torch current stream)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from timing import timeit
import pcu_b200 as pcu

g = torch.Generator(device="cuda").manual_seed(0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
x = torch.rand((n, 3), generator=g, device="cuda"); y = torch.rand((n, 3), generator=g, device="cuda")
for occ in (1.0, 2.0, 3.0, 4.0, 6.0):
    pcu._pcu_internal._set_defaults(cell_occupancy=occ)
    med, mn = timeit(lambda: pcu.chamfer_distance(x, y), flush=False)
    print("chamfer n=%d occ=%.1f: median %.3f ms  min %.3f ms -> %.3e qpts/s" % (n, occ, med, mn, 2 * n / med * 1e3), flush=True)
pcu._pcu_internal._set_defaults(cell_occupancy=0.0)
med, mn = timeit(lambda: pcu.k_nearest_neighbors(x, y, 1), flush=False)
print("knn k=1: median %.3f ms min %.3f -> %.3e q/s" % (med, mn, n / med * 1e3), flush=True)
for occ in (4.0, 8.0, 12.0, 16.0):
    pcu._pcu_internal._set_defaults(cell_occupancy=occ)
    med, mn = timeit(lambda: pcu.k_nearest_neighbors(x, y, 16), warm=2, it=5, flush=False)
    print("knn k=16 occ=%.0f: median %.3f ms min %.3f -> %.3e q/s" % (occ, med, mn, n / med * 1e3), flush=True)
pcu._pcu_internal._set_defaults(cell_occupancy=0.0)
xb = torch.rand((64, 65536, 3), generator=g, device="cuda"); yb = torch.rand((64, 65536, 3), generator=g, device="cuda")
med, mn = timeit(lambda: pcu.batched_chamfer_distance(xb, yb), warm=2, it=5, flush=False)
print("batched 64x65536: median %.3f ms -> %.3e qpts/s" % (med, 64 * 2 * 65536 / med * 1e3), flush=True)
v = pcu.batched_chamfer_distance(xb, yb)
print("batched check", float(v[3]), float(pcu.chamfer_distance(xb[3], yb[3])))
