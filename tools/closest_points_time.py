"""closest_points_on_mesh: time per call (CUDA events, device-resident inputs, warm-up, L2 flushed before every timed call).

  mesh     jittered icosphere of 1 310 720 faces (subdivision 8, as in tools/mesh_sampling_time.py), int32 faces,
           fp32 and fp64 vertices
  build    the call with one query: the tree build plus one traversal
  call     10^6 near-surface queries (points on random faces plus noise of 1e-3) and 10^6 queries uniform in the box
           twice the mesh's, each in input (random) order and pre-sorted by the Morton code of their positions, the
           second showing what traversal in Morton order would gain before the cost of sorting the queries

`python tools/closest_points_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch
from meshes import icosphere
from timing import card, timeit
import pcu_b200 as pcu

I = pcu._pcu_internal


def morton_order(p):
    """Rows of p sorted by the Morton code of their positions quantised to 21 bits per axis over their box."""
    lo, hi = p.min(0), p.max(0)
    q = np.minimum(((p - lo) / np.maximum(hi - lo, 1e-30) * 2 ** 21).astype(np.int64), 2 ** 21 - 1)
    code = np.zeros(len(p), dtype=np.uint64)
    for bit in range(21):
        for k in range(3):
            code |= ((q[:, k] >> bit) & 1).astype(np.uint64) << np.uint64(3 * bit + k)
    return np.argsort(code, kind="stable")


print(card(), flush=True)
sub = int(sys.argv[1]) if len(sys.argv) > 1 else 8
v64, f = icosphere(sub, 0.2 * 2.0 ** -sub, 1)
f = f.astype(np.int32)
rng = np.random.default_rng(4)
n = 10 ** 6
fi = rng.integers(0, len(f), n)
r = rng.random((n, 2))
s = np.sqrt(r[:, :1])
bc = np.concatenate([1 - s, s * (1 - r[:, 1:]), s * r[:, 1:]], 1)
near = (v64[f[fi]] * bc[:, :, None]).sum(1) + 1e-3 * rng.standard_normal((n, 3))
lo, hi = v64.min(0), v64.max(0)
box = (lo + hi) / 2 + (rng.random((n, 3)) - 0.5) * 2 * (hi - lo)
ft = torch.from_numpy(f).cuda()
stream = torch.cuda.current_stream().cuda_stream
print("mesh: %d vertices, %d faces; %d queries per set" % (len(v64), len(f), n), flush=True)
for dt in (torch.float32, torch.float64):
    vt = torch.from_numpy(v64).to(dt).cuda()
    is64 = dt == torch.float64
    d = torch.empty(n, dtype=dt, device="cuda")
    fidx = torch.empty(n, dtype=torch.int32, device="cuda")
    out_bc = torch.empty((n, 3), dtype=dt, device="cuda")
    bad = torch.empty(1, dtype=torch.int64, device="cuda")

    def call(pt):
        return lambda: I._closest_points_on_mesh_device(is64, pt.data_ptr(), pt.shape[0], vt.data_ptr(), len(v64), ft.data_ptr(),
                                                        len(f), 0, d.data_ptr(), fidx.data_ptr(), out_bc.data_ptr(),
                                                        bad.data_ptr(), 0, stream)
    one = torch.from_numpy(near[:1]).to(dt).cuda()
    med, mn = timeit(call(one))
    print("%s build (one query): median %.3f ms min %.3f ms" % (str(dt)[6:], med, mn), flush=True)
    for name, pts in (("near-surface", near), ("uniform-box", box)):
        for order, rows in (("input order", np.arange(n)), ("Morton-sorted", morton_order(pts))):
            pt = torch.from_numpy(pts[rows]).to(dt).cuda()
            med, mn = timeit(call(pt))
            print("%s %s %s: call median %.3f ms min %.3f ms  (%.1f M queries/s at the median)"
                  % (str(dt)[6:], name, order, med, mn, n / (med * 1e-3) / 1e6), flush=True)
