"""ray_mesh_intersection and RayMeshIntersector: time per call (CUDA events, device-resident inputs, warm-up, L2 flushed
before every timed call).

  mesh     jittered icosphere of 1 310 720 faces (subdivision 8, as in tools/closest_points_time.py), int32 faces,
           fp32 and fp64 vertices
  rays     10^6 coherent camera rays (a pinhole grid from outside the sphere, in scan-line order) and 10^6 incoherent
           rays (random origins around the sphere aimed at random points inside it)
  one-shot the function: tree build plus cast; the build alone is the call with one ray
  prepared RayMeshIntersector.intersect_rays: the cast alone

`python tools/ray_mesh_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first.
There is no CPU arm: the reference casts with Embree, which is not built here."""
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
side = 1000
n = side * side
u = np.linspace(-0.45, 0.45, side)
px = np.stack(np.meshgrid(u, u, indexing="ij"), -1).reshape(-1, 2)
cam_o = np.broadcast_to(np.array([0.0, 0.0, -3.0]), (n, 3)).copy()
cam_d = np.concatenate([px, np.ones((n, 1))], 1)
rnd_o = 3.0 * rng.standard_normal((n, 3))
rnd_d = 0.5 * rng.standard_normal((n, 3)) - rnd_o
ft = torch.from_numpy(f).cuda()
stream = torch.cuda.current_stream().cuda_stream
print("mesh: %d vertices, %d faces; %d rays per set" % (len(v64), len(f), n), flush=True)
for dt in (torch.float32, torch.float64):
    vt = torch.from_numpy(v64).to(dt).cuda()
    is64 = dt == torch.float64
    fidx = torch.empty(n, dtype=torch.int32, device="cuda")
    out_bc = torch.empty((n, 3), dtype=dt, device="cuda")
    out_t = torch.empty(n, dtype=dt, device="cuda")
    bad = torch.empty(1, dtype=torch.int64, device="cuda")
    inf = float("inf")

    def call(ot, d_):
        return lambda: I._ray_mesh_intersection_device(is64, vt.data_ptr(), len(v64), ft.data_ptr(), len(f), 0, ot.data_ptr(), 3,
                                                       d_.data_ptr(), d_.shape[0], 0.0, inf, fidx.data_ptr(), out_bc.data_ptr(),
                                                       out_t.data_ptr(), bad.data_ptr(), 0, stream)
    one_o, one_d = (torch.from_numpy(x[:1]).to(dt).cuda() for x in (cam_o, cam_d))
    med, mn = timeit(call(one_o, one_d))
    print("%s build (one ray): median %.3f ms min %.3f ms" % (str(dt)[6:], med, mn), flush=True)
    isect = pcu.RayMeshIntersector(vt, ft)
    for name, o, d in (("camera", cam_o, cam_d), ("random", rnd_o, rnd_d)):
        ot, d_ = (torch.from_numpy(x).to(dt).cuda() for x in (o, d))
        med, mn = timeit(call(ot, d_))
        hits = float((fidx >= 0).float().mean())
        print("%s %s one-shot: median %.3f ms min %.3f ms (%.1f M rays/s; %.0f %% hit)"
              % (str(dt)[6:], name, med, mn, n / (med * 1e-3) / 1e6, 100 * hits), flush=True)
        med, mn = timeit(lambda: isect.intersect_rays(ot, d_))
        print("%s %s prepared: median %.3f ms min %.3f ms (%.1f M rays/s)"
              % (str(dt)[6:], name, med, mn, n / (med * 1e-3) / 1e6), flush=True)
    isect.close()
