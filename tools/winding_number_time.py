"""triangle_soup_fast_winding_number / signed_distance_to_mesh: time per call (CUDA events, device-resident inputs,
warm-up, L2 flushed before every timed call), on the mesh and query sets of tools/closest_points_time.py.

  mesh      jittered icosphere of 1 310 720 faces (subdivision 8), int32 faces, fp32 and fp64 vertices
  build     the winding-number call with one query: the tree build, the moment and radius passes, one walk
  walk      10^6 near-surface and 10^6 uniform-box queries: the winding-number call minus the build
  signed    signed_distance_to_mesh on the same queries, and closest_points_on_mesh beside it (what the sign costs)

`python tools/winding_number_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
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
    name = str(dt)[6:]
    out = torch.empty(n, dtype=dt, device="cuda")
    fidx = torch.empty(n, dtype=torch.int32, device="cuda")
    out_bc = torch.empty((n, 3), dtype=dt, device="cuda")
    bad = torch.empty(1, dtype=torch.int64, device="cuda")

    def winding(pt):
        return lambda: I._fast_winding_number_device(is64, vt.data_ptr(), len(v64), ft.data_ptr(), len(f), 0, pt.data_ptr(),
                                                      pt.shape[0], 2.0, out.data_ptr(), bad.data_ptr(), 0, stream)

    def signed(pt):
        return lambda: I._signed_distance_to_mesh_device(is64, pt.data_ptr(), pt.shape[0], vt.data_ptr(), len(v64), ft.data_ptr(),
                                                         len(f), 0, -float("inf"), float("inf"), out.data_ptr(), fidx.data_ptr(),
                                                         out_bc.data_ptr(), bad.data_ptr(), 0, stream)

    def closest(pt):
        return lambda: I._closest_points_on_mesh_device(is64, pt.data_ptr(), pt.shape[0], vt.data_ptr(), len(v64), ft.data_ptr(),
                                                        len(f), 0, out.data_ptr(), fidx.data_ptr(), out_bc.data_ptr(),
                                                        bad.data_ptr(), 0, stream)
    one = torch.from_numpy(near[:1]).to(dt).cuda()
    build, build_min = timeit(winding(one))
    cbuild, _ = timeit(closest(one))
    print("%s build + moments (one query): median %.3f ms min %.3f ms  (closest-point build alone: %.3f ms)"
          % (name, build, build_min, cbuild), flush=True)
    for label, pts in (("near-surface", near), ("uniform-box", box)):
        pt = torch.from_numpy(pts).to(dt).cuda()
        wmed, wmin = timeit(winding(pt))
        smed, smin = timeit(signed(pt))
        cmed, cmin = timeit(closest(pt))
        print("%s %s: winding call %.3f ms (walk %.3f ms, %.1f M queries/s); signed distance %.3f ms; closest points %.3f ms;"
              " the sign costs %.3f ms" % (name, label, wmed, wmed - build, n / ((wmed - build) * 1e-3) / 1e6, smed, cmed,
                                           smed - cmed), flush=True)
