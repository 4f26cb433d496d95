"""estimate_point_cloud_areas: time per call on a noisy sphere of 10^6 points (uniform directions, radius 1 + 1e-3 x
standard normal, radial normals), k = 8, 16 and 32, float32 and float64, with k_nearest_neighbors(p, p, k) on the same
cloud for comparison (device-resident inputs, int64 neighbour rows as k_nearest_neighbors returns them, warm-up, L2
flushed before every timed call, CUDA events around the public call).

"bytes/row": what the algorithm must move per row -- the index row (8 k), the gathered points and normals (2 x 3 k x
sizeof(T)) and the area (sizeof(T)); "at 3.35 TB/s" is the time those bytes alone would take at the H100's HBM3
data-sheet bandwidth.  The gathers are random, so the kernel is not expected to reach it.
`python tools/point_areas_time.py`; the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import numpy as np
import torch
from timing import card, timeit
import pcu_b200 as pcu

M = 10 ** 6


def cloud(dtype):
    rng = np.random.default_rng(0)
    u = rng.standard_normal((M, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = u * (1.0 + 1e-3 * rng.standard_normal((M, 1)))
    return torch.from_numpy(p.astype(dtype)).cuda(), torch.from_numpy(u.astype(dtype)).cuda()


def main():
    print("card:", card())
    print("%-8s %3s %12s %12s %10s %14s %12s %12s" % ("dtype", "k", "areas ms", "(min)", "bytes/row", "at 3.35 TB/s", "knn ms", "sum(a)"))
    for dtype in (np.float32, np.float64):
        p, n = cloud(dtype)
        for k in (8, 16, 32):
            _, i = pcu.k_nearest_neighbors(p, p, k)
            med, lo = timeit(lambda: pcu.estimate_point_cloud_areas(p, i, n), warm=3, it=20)
            kmed, _ = timeit(lambda: pcu.k_nearest_neighbors(p, p, k), warm=2, it=10)
            row = 8 * k + 2 * 3 * k * np.dtype(dtype).itemsize + np.dtype(dtype).itemsize
            total = float(pcu.estimate_point_cloud_areas(p, i, n).double().sum())
            print("%-8s %3d %12.3f %12.3f %10d %11.3f ms %12.3f %12.6f" % (np.dtype(dtype).name, k, med, lo, row, row * M / 3.35e12 * 1e3,
                                                                          kmed, total))


if __name__ == "__main__":
    main()
