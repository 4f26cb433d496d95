"""point_cloud_fast_winding_number: time per call (CUDA events, device-resident inputs, warm-up, L2 flushed before every
timed call).

  cloud     about 10^6 oriented points on the jittered subdivision-8 icosphere of tools/winding_number_time.py: one
            sample_mesh_random point per sample, the face's unit normal, area = surface area / #samples
  build     the call with one query: the point tree, the centre, radius and moment passes, one walk
  walk      10^6 near-surface and 10^6 uniform-box queries: the call minus the build

`python tools/point_winding_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch
from meshes import icosphere
from timing import card, timeit
import pcu_b200 as pcu

I = pcu._pcu_internal


print(card(), flush=True)
sub = int(sys.argv[1]) if len(sys.argv) > 1 else 8
v64, f = icosphere(sub, 0.2 * 2.0 ** -sub, 1)
f = f.astype(np.int32)
m = 10 ** 6
fi, bc = pcu.sample_mesh_random(v64, f, m, random_seed=7)
fi = fi.astype(np.int64)
x = (v64[f[fi]] * bc[:, :, None]).sum(1)
cr = np.cross(v64[f[:, 1]] - v64[f[:, 0]], v64[f[:, 2]] - v64[f[:, 0]])
nrm = (cr / np.linalg.norm(cr, axis=1, keepdims=True))[fi]
area = np.full(len(x), 0.5 * np.linalg.norm(cr, axis=1).sum() / len(x))
rng = np.random.default_rng(4)
n = 10 ** 6
qf = rng.integers(0, len(f), n)
r = rng.random((n, 2))
s = np.sqrt(r[:, :1])
qbc = np.concatenate([1 - s, s * (1 - r[:, 1:]), s * r[:, 1:]], 1)
near = (v64[f[qf]] * qbc[:, :, None]).sum(1) + 1e-3 * rng.standard_normal((n, 3))
lo, hi = v64.min(0), v64.max(0)
box = (lo + hi) / 2 + (rng.random((n, 3)) - 0.5) * 2 * (hi - lo)
stream = torch.cuda.current_stream().cuda_stream
print("cloud: %d oriented points on a %d-face icosphere; %d queries per set" % (len(x), len(f), n), flush=True)
for dt in (torch.float32, torch.float64):
    pt, nt, at = (torch.from_numpy(y).to(dt).cuda() for y in (x, nrm, area))
    is64 = dt == torch.float64
    name = str(dt)[6:]
    out = torch.empty(n, dtype=dt, device="cuda")

    def winding(qt):
        return lambda: I._point_cloud_fast_winding_number_device(is64, pt.data_ptr(), nt.data_ptr(), at.data_ptr(), len(x),
                                                                 qt.data_ptr(), qt.shape[0], 2.0, out.data_ptr(), 0, stream)
    one = torch.from_numpy(near[:1]).to(dt).cuda()
    build, build_min = timeit(winding(one))
    print("%s build + moments (one query): median %.3f ms min %.3f ms" % (name, build, build_min), flush=True)
    for label, pts in (("near-surface", near), ("uniform-box", box)):
        qt = torch.from_numpy(pts).to(dt).cuda()
        wmed, wmin = timeit(winding(qt))
        print("%s %s: call %.3f ms (min %.3f), walk %.3f ms, %.1f M queries/s"
              % (name, label, wmed, wmin, wmed - build, n / ((wmed - build) * 1e-3) / 1e6), flush=True)
