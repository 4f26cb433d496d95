"""voronoi_centroids_unit_cube, lloyd_3d and lloyd_2d: time per call (warm-up, L2 flushed before every timed call,
median and minimum of 10; host clock around the call, which ends by synchronising the device).

  uniform 1e5 / 1e6   voronoi_centroids_unit_cube of uniform seeds (CUDA tensor in and out)
  cluster 1e6         90 % of the seeds in a ball of radius 1e-3, the rest uniform in the cube: the cells of the sparse
                      seeds next to the ball take the last resort, some of them in several rounds
  graded 1e6          every coordinate u^3, u uniform: the density grows without bound toward the corner (0, 0, 0)
  lloyd_3d / lloyd_2d 10^6 points with the defaults (10 Lloyd steps, at most 10 Newton steps)
The cells each pass handled are printed beside every time.  The reference's time cannot be taken: geogram is not
part of it as checked out.  `python tools/lloyd_time.py [repeats [cluster repeats]]`; the card's name and power limit are printed first."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import time
import numpy as np
import torch
from timing import card
import pcu_b200 as pcu

flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush_buf.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return np.median(ts) * 1e3, min(ts) * 1e3


print(card())
rng = np.random.default_rng(0)


def ball(n, r):
    d = rng.normal(size=(n, 3))
    d *= (r * rng.random(n) ** (1 / 3) / np.linalg.norm(d, axis=1))[:, None]
    return 0.5 + d


cases = {
    "centroids uniform 1e5": rng.random((100_000, 3)),
    "centroids uniform 1e6": rng.random((1_000_000, 3)),
    "centroids graded 1e6": rng.random((1_000_000, 3)) ** 3,
}
for name, x in cases.items():
    xt = torch.from_numpy(x).cuda()
    med, lo = timed(lambda: pcu.voronoi_centroids_unit_cube(xt), reps)
    print("%-24s median %9.2f ms  min %9.2f ms  cells per pass %s" % (name, med, lo, pcu._lloyd.last_pass_counts), flush=True)
for name, fn in (("lloyd_2d 1e6", pcu.lloyd_2d), ("lloyd_3d 1e6", pcu.lloyd_3d)):
    np.random.seed(0)
    med, lo = timed(lambda: fn(1_000_000), reps)
    print("%-24s median %9.2f ms  min %9.2f ms  cells per pass %s  Newton steps %d" % (
        name, med, lo, pcu._lloyd.last_pass_counts, len(pcu._lloyd.last_newton_energies) - 1), flush=True)
x = torch.from_numpy(np.concatenate([ball(900_000, 1e-3), rng.random((100_000, 3))])).cuda()
med, lo = timed(lambda: pcu.voronoi_centroids_unit_cube(x), int(sys.argv[2]) if len(sys.argv) > 2 else reps)
print("%-24s median %9.2f ms  min %9.2f ms  cells per pass %s" % ("centroids cluster 1e6", med, lo, pcu._lloyd.last_pass_counts),
      flush=True)
