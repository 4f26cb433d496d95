"""ray_surfel_intersection and RaySurfelIntersector against the materialized route: time per call (CUDA events,
device-resident inputs, warm-up, L2 flushed before every timed call) and device memory of the prepared trees.

  surfels    10^6 points from sample_mesh_random on the jittered subdivision-8 icosphere of tools/ray_mesh_time.py,
             with their faces' normals and r = 1.5 x the mean spacing sqrt(area / 10^6), so that neighbours overlap;
             subdivs = 7; fp32 and fp64
  rays       the 10^6 camera rays and 10^6 random rays of tools/ray_mesh_time.py
  one-shot   ray_surfel_intersection: surfel tree build plus cast; the build alone is the call with one ray
  prepared   RaySurfelIntersector.intersect_rays: the cast alone
  material.  pointcloud_surfel_geometry, then RayMeshIntersector on its (v, f) and its intersect_rays (fp32 only: its
             fp32 vertices are the fans the surfel cast tests, so both routes give the same pid and t)
  memory     device memory taken by each prepared tree (cudaMemGetInfo before and after the constructor)

`python tools/ray_surfel_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch
from meshes import icosphere
from timing import card, timeit
import pcu_b200 as pcu

I = pcu._pcu_internal
SUBDIVS = 7


def held(make):
    """(object, device bytes it holds): cudaMemGetInfo around its construction."""
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    obj = make()
    torch.cuda.synchronize()
    return obj, before - torch.cuda.mem_get_info()[0]


print(card(), flush=True)
sub = int(sys.argv[1]) if len(sys.argv) > 1 else 8
v64, f = icosphere(sub, 0.2 * 2.0 ** -sub, 1)
f = f.astype(np.int32)
m = 10 ** 6
fid, bc = pcu.sample_mesh_random(v64, f, m, 7)
p64 = pcu.interpolate_barycentric_coords(f, fid, bc, v64)
e1, e2 = v64[f[:, 1]] - v64[f[:, 0]], v64[f[:, 2]] - v64[f[:, 0]]
fn = np.cross(e1, e2)
area = 0.5 * np.linalg.norm(fn, axis=1).sum()
n64 = (fn / np.linalg.norm(fn, axis=1, keepdims=True))[fid]
r = 1.5 * float(np.sqrt(area / m))
rng = np.random.default_rng(4)
side = 1000
nr = side * side
u = np.linspace(-0.45, 0.45, side)
px = np.stack(np.meshgrid(u, u, indexing="ij"), -1).reshape(-1, 2)
cam_o = np.broadcast_to(np.array([0.0, 0.0, -3.0]), (nr, 3)).copy()
cam_d = np.concatenate([px, np.ones((nr, 1))], 1)
rnd_o = 3.0 * rng.standard_normal((nr, 3))
rnd_d = 0.5 * rng.standard_normal((nr, 3)) - rnd_o
stream = torch.cuda.current_stream().cuda_stream
print("surfels: %d points from %d faces, r = %.3g (1.5 x mean spacing), subdivs = %d; %d rays per set"
      % (m, len(f), r, SUBDIVS, nr), flush=True)
for dt in (torch.float32, torch.float64):
    name = str(dt)[6:]
    pt, nt = (torch.from_numpy(x).to(dt).cuda() for x in (p64, n64))
    rt = torch.full((m,), r, dtype=dt, device="cuda")
    is64 = dt == torch.float64
    pid = torch.empty(nr, dtype=torch.int32, device="cuda")
    out_t = torch.empty(nr, dtype=dt, device="cuda")
    inf = float("inf")

    def call(ot, d_):
        return lambda: I._ray_surfel_intersection_device(is64, pt.data_ptr(), nt.data_ptr(), rt.data_ptr(), m, SUBDIVS, ot.data_ptr(),
                                                         3, d_.data_ptr(), d_.shape[0], 0.0, inf, pid.data_ptr(), out_t.data_ptr(),
                                                         0, stream)
    one_o, one_d = (torch.from_numpy(x[:1]).to(dt).cuda() for x in (cam_o, cam_d))
    med, mn = timeit(call(one_o, one_d))
    print("%s surfel build (one ray): median %.3f ms min %.3f ms" % (name, med, mn), flush=True)
    isect, nbytes = held(lambda: pcu.RaySurfelIntersector(pt, nt, rt, SUBDIVS))
    print("%s RaySurfelIntersector holds %.1f MB" % (name, nbytes / 1e6), flush=True)
    mesh = None
    if not is64:
        med, mn = timeit(lambda: pcu.pointcloud_surfel_geometry(pt, nt, rt, SUBDIVS))
        print("%s materialized: pointcloud_surfel_geometry median %.3f ms min %.3f ms" % (name, med, mn), flush=True)
        gv, gf = pcu.pointcloud_surfel_geometry(pt, nt, rt, SUBDIVS)
        med, mn = timeit(lambda: pcu.RayMeshIntersector(gv, gf).close(), warm=1, it=5)
        print("%s materialized: RayMeshIntersector build median %.3f ms min %.3f ms (geometry arrays %.1f MB)"
              % (name, med, mn, (gv.numel() * gv.element_size() + gf.numel() * gf.element_size()) / 1e6), flush=True)
        mesh, nbytes = held(lambda: pcu.RayMeshIntersector(gv, gf))
        print("%s materialized: RayMeshIntersector holds %.1f MB" % (name, nbytes / 1e6), flush=True)
    for setname, o, d in (("camera", cam_o, cam_d), ("random", rnd_o, rnd_d)):
        ot, d_ = (torch.from_numpy(x).to(dt).cuda() for x in (o, d))
        med, mn = timeit(call(ot, d_))
        hits = float((pid >= 0).float().mean())
        print("%s %s one-shot: median %.3f ms min %.3f ms (%.1f M rays/s; %.0f %% hit)"
              % (name, setname, med, mn, nr / (med * 1e-3) / 1e6, 100 * hits), flush=True)
        med, mn = timeit(lambda: isect.intersect_rays(ot, d_))
        print("%s %s prepared: median %.3f ms min %.3f ms (%.1f M rays/s)"
              % (name, setname, med, mn, nr / (med * 1e-3) / 1e6), flush=True)
        if mesh is not None:
            med, mn = timeit(lambda: mesh.intersect_rays(ot, d_))
            got, ref = isect.intersect_rays(ot, d_), mesh.intersect_rays(ot, d_)
            agree = torch.equal(got[0], torch.where(ref[0] >= 0, ref[0] // SUBDIVS, ref[0])) and torch.equal(got[1], ref[2])
            print("%s %s materialized cast: median %.3f ms min %.3f ms (%.1f M rays/s; same pid and t: %s)"
                  % (name, setname, med, mn, nr / (med * 1e-3) / 1e6, agree), flush=True)
    isect.close()
    if mesh is not None:
        mesh.close()
