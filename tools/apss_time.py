"""pointcloud_apss_curvature and project_points_onto_apss: time per call on a noisy sphere of 10^6 points (uniform
directions, radius 1 + 1e-3 x standard normal, radial normals), r = 3 and 6 mean spacings, float32 and float64
(device-resident inputs, warm-up, L2 flushed before every timed call, CUDA events around the public call).

Rows: the curvature of every point; the projection of 10^6 queries (the points moved by up to r / 4 per axis) in a
spatially coherent order (sorted by the Morton code of their cell of size r) and in a random permutation of the same
queries, which puts a number on the cost of incoherent queries; and estimate_point_cloud_normals_ball on the same ball
(ball_radius = r^2, constant weights) as the yardstick: it walks each ball once.  "ball" is the mean ball population,
counted on 2 000 points on the host.
`python tools/apss_time.py`; the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import numpy as np
import torch
from scipy.spatial import cKDTree
from timing import card, timeit
import pcu_b200 as pcu

M = 10 ** 6


def cloud():
    rng = np.random.default_rng(0)
    u = rng.standard_normal((M, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = u * (1.0 + 1e-3 * rng.standard_normal((M, 1)))
    return p, u


def morton_order(q, cell):
    """The queries' order along the Morton curve of a grid of cells of size `cell`."""
    c = np.floor((q - q.min(0)) / cell).astype(np.uint64)
    key = np.zeros(len(q), np.uint64)
    for b in range(21):
        for a in range(3):
            key |= ((c[:, a] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + a)
    return np.argsort(key, kind="stable")


def main():
    print("card:", card())
    p, u = cloud()
    h = np.sqrt(4 * np.pi / M)
    tree = cKDTree(p)
    print("%-8s %6s %6s %14s %14s %14s %14s %10s" % ("dtype", "r/h", "ball", "curvature ms", "coherent ms", "random ms",
                                                      "normals ms", "nan"))
    for k in (3, 6):
        r = k * h
        ball = np.mean([len(c) for c in tree.query_ball_point(p[:2000], r)])
        rng = np.random.default_rng(1)
        q = p + rng.uniform(-0.25, 0.25, p.shape) * r
        q = q[morton_order(q, r)]
        perm = rng.permutation(M)
        for dtype in (np.float32, np.float64):
            pt, nt = torch.from_numpy(p.astype(dtype)).cuda(), torch.from_numpy(u.astype(dtype)).cuda()
            qc = torch.from_numpy(q.astype(dtype)).cuda()
            qr = qc[torch.from_numpy(perm).cuda()].contiguous()
            cm, cl = timeit(lambda: pcu.pointcloud_apss_curvature(pt, nt, r), warm=2, it=10)
            pm, pl = timeit(lambda: pcu.project_points_onto_apss(pt, nt, qc, r), warm=2, it=10)
            rm, rl = timeit(lambda: pcu.project_points_onto_apss(pt, nt, qr, r), warm=2, it=10)
            nm, nl = timeit(lambda: pcu.estimate_point_cloud_normals_ball(pt, r * r), warm=2, it=10)
            nan = int(torch.isnan(pcu.pointcloud_apss_curvature(pt, nt, r)).sum())
            print("%-8s %6d %6.0f %7.2f (%5.2f) %7.2f (%5.2f) %7.2f (%5.2f) %7.2f (%5.2f) %10d"
                  % (np.dtype(dtype).name, k, ball, cm, cl, pm, pl, rm, rl, nm, nl, nan))


if __name__ == "__main__":
    main()
