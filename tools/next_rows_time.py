"""Device-resident timings of the 8(f) rows (CUDA events around the public API, CUDA tensors in):
python tools/next_rows_time.py [n]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from timing import timeit
import pcu_b200 as pcu

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
g = torch.Generator(device="cuda").manual_seed(0)


def timed(label, fn, reps=5):
    print("%-58s %9.3f ms" % (label, timeit(fn, warm=1, it=reps, flush=False)[1]), flush=True)


x = torch.rand((n, 3), generator=g, device="cuda")
sph = torch.nn.functional.normalize(torch.randn((n, 3), generator=g, device="cuda"), dim=1)
timed("normals knn k=12, %d uniform points" % n, lambda: pcu.estimate_point_cloud_normals_knn(x, 12))
timed("normals knn k=12, %d points on a sphere" % n, lambda: pcu.estimate_point_cloud_normals_knn(sph, 12))
r_vol = float((12.0 / (4.19 * n)) ** (2.0 / 3.0))           # squared reach holding ~12 points of the uniform cloud
r_sph = float(12.0 * 4.0 / n)                               # ... of the sphere: pi r^2 n / (4 pi) = 12
timed("normals ball (~12 neighbours), uniform", lambda: pcu.estimate_point_cloud_normals_ball(x, r_vol))
timed("normals ball (~12 neighbours), sphere", lambda: pcu.estimate_point_cloud_normals_ball(sph, r_sph))
timed("normals ball (~100 neighbours), sphere, rbf", lambda: pcu.estimate_point_cloud_normals_ball(sph, 100 * 4.0 / n, weight_function="rbf"))
timed("voxel down-sampling, 100^3 voxels", lambda: pcu.downsample_point_cloud_on_voxel_grid(0.01, x))
dup = torch.cat([x, x[: n // 4]])
timed("deduplicate_point_cloud fp32, %d rows (20 %% duplicates)" % dup.shape[0], lambda: pcu.deduplicate_point_cloud(dup, 1e-11))
timed("deduplicate_point_cloud fp64", lambda: pcu.deduplicate_point_cloud(dup.double(), 1e-11))
# N3 Morton codes (numpy in / numpy out through the host entry points: H2D + kernel + D2H) and on-device kernel time
I = pcu._pcu_internal
pts_i = np.random.default_rng(0).integers(-(1 << 20), 1 << 20, (10_000_000, 3)).astype(np.int32)
import time
def wall(label, fn, reps=3):
    fn(); best = 1e30
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); best = min(best, (time.perf_counter() - t0) * 1e3)
    print("%-58s %9.3f ms (wall, host arrays)" % (label, best), flush=True)
codes = pcu.morton_encode(pts_i)
wall("morton_encode 10^7 points (120 MB in, 80 MB out)", lambda: pcu.morton_encode(pts_i))
wall("morton_decode 10^7 codes", lambda: pcu.morton_decode(codes))
sc = np.sort(codes)
wall("morton_knn k=15, 10^6 queries in 10^7 sorted codes", lambda: pcu.morton_knn(sc, codes[:1_000_000], 15))
# N4 dense metrics on device tensors
a = torch.rand((4, 2048, 3), generator=g, device="cuda", dtype=torch.float32); b = torch.rand((4, 2048, 3), generator=g, device="cuda", dtype=torch.float32)
timed("pairwise_distances 4 x 2048 x 2048 (fp32)", lambda: pcu.pairwise_distances(a, b))
M = pcu.pairwise_distances(a, b)
wa = torch.full((4, 2048), 1.0 / 2048, device="cuda"); wb = torch.full((4, 2048), 1.0 / 2048, device="cuda")
timed("sinkhorn 4 x 2048 x 2048, eps 1e-2, 100 iterations (no early stop)", lambda: pcu.sinkhorn(wa, wb, M, eps=1e-2, max_iters=100, stop_thresh=0.0))
p64 = a[0].double(); q64 = b[0].double()     # like the reference, EMD wants float64 points (its weights are np.ones(n) / n)
timed("earth_movers_distance 2048 vs 2048 (fp64), 100 iterations", lambda: pcu.earth_movers_distance(p64, q64, eps=1e-2, max_iters=100, stop_thresh=0.0))
