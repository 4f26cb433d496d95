"""Sparse voxel grids and voxel cube meshes: time per call and per phase (device-resident inputs, warm-up, L2 flushed
before every timed call).

  points   10^7 fp32 points on the unit sphere's surface -> sparse_voxel_grid_from_pointcloud at voxel size 1/512
  dilate   that shell grid dilated 1 and 3 times (dilate_sparse_voxel_grid, int32)
  erode    a solid ball of about 4 * 10^6 voxels (radius 98.5) eroded once (erode_sparse_voxel_grid, int32)
  hex      the once-dilated shell -> sparse_voxel_grid_to_hex_mesh (fp32 and fp64 vertices)
  cubes    voxel_grid_geometry of 10^6 voxels (int32)
  pipeline 10^6 points on a sphere -> grid -> dilate(2) -> hex mesh -> exact SDF at the vertices (torch) ->
           marching_cubes_sparse_voxel_grid, end to end
  numpy    the host restatement of the points -> grid step (quantise, Morton-encode through the oracle, np.unique) on
           the same 10^7 points, for context

Each call is timed end to end with a host clock around the synchronised call (median of 10 and minimum).  The phases
come from a torch.profiler pass of their own, summed kernel times by kernel-name prefix.  `python
tools/sparse_voxel_time.py`; the card's name and power limit are printed first."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import time
import numpy as np
import torch
from timing import card
import pcu_b200 as pcu

flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2


def timeit(fn, warm=2, it=10):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(it):
        flush_buf.add_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), float(np.min(ts))


GROUPS = [("codes", ("svg_point_codes", "svb_codes", "svg_corners")), ("sort", ("sort_",)),
          ("neighbours", ("svg_dilate_flag", "svg_erode_flag")), ("runs/compaction", ("mc_heads", "keep_count", "keep_offsets",
                                                                                   "svg_dilate_write", "svg_keep_voxels")),
          ("emit", ("svg_decode", "svg_rank", "vg_geometry", "Memcpy"))]


def phases(fn):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    out = {g: 0.0 for g, _ in GROUPS}
    out["other"] = 0.0
    for e in prof.key_averages():
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        for g, keys in GROUPS:
            if any(k in e.key for k in keys):
                out[g] += us
                break
        else:
            out["other"] += us
    return " ".join("%s %.3f" % (k, v / 1e3) for k, v in out.items() if v > 0)


def report(name, fn, sizes):
    med, mn = timeit(fn)
    print("%s: %s; call median %.3f ms min %.3f ms; phases (kernel ms) %s" % (name, sizes, med, mn, phases(fn)), flush=True)


def sphere(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = torch.randn((n, 3), device="cuda", generator=g, dtype=torch.float64)
    return d / d.norm(dim=1, keepdim=True)


print(card(), flush=True)

s = 1.0 / 512
pts = sphere(10 ** 7, 0).float()
grid, p2v = pcu.sparse_voxel_grid_from_pointcloud(pts, s)
report("points -> grid", lambda: pcu.sparse_voxel_grid_from_pointcloud(pts, s), "%d points -> %d voxels" % (len(pts), len(grid)))

d1 = pcu.dilate_sparse_voxel_grid(grid, 1)
report("dilate x1", lambda: pcu.dilate_sparse_voxel_grid(grid, 1), "%d -> %d voxels" % (len(grid), len(d1)))
d3 = pcu.dilate_sparse_voxel_grid(grid, 3)
report("dilate x3", lambda: pcu.dilate_sparse_voxel_grid(grid, 3), "%d -> %d voxels" % (len(grid), len(d3)))
del d3

a = torch.arange(-100, 101, device="cuda", dtype=torch.int32)
z, y, x = torch.meshgrid(a, a, a, indexing="ij")
cube = torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], 1)
ball = cube[(cube.double() ** 2).sum(1) <= 98.5 ** 2].contiguous()
del cube, x, y, z
e1 = pcu.erode_sparse_voxel_grid(ball)
report("erode ball", lambda: pcu.erode_sparse_voxel_grid(ball), "%d -> %d voxels" % (len(ball), len(e1)))

for dt in (np.float32, np.float64):
    hv, hc = pcu.sparse_voxel_grid_to_hex_mesh(d1, s, dtype=dt)
    report("hex mesh %s" % np.dtype(dt).name, lambda: pcu.sparse_voxel_grid_to_hex_mesh(d1, s, dtype=dt),
           "%d voxels -> %d vertices" % (len(d1), len(hv)))
    del hv, hc

ijk = torch.randint(-500, 500, (10 ** 6, 3), device="cuda", dtype=torch.int32)
report("voxel_grid_geometry", lambda: pcu.voxel_grid_geometry(ijk, 0.01), "%d voxels" % len(ijk))


def pipeline(p, sv):
    g, _ = pcu.sparse_voxel_grid_from_pointcloud(p, sv)
    band = pcu.dilate_sparse_voxel_grid(g, 2)
    v, c = pcu.sparse_voxel_grid_to_hex_mesh(band, sv)
    sdf = v.norm(dim=1) - 1.0
    return pcu.marching_cubes_sparse_voxel_grid(sdf, v, c, 0.0)


pp = sphere(10 ** 6, 1)
mv, mf = pipeline(pp, 1.0 / 256)
report("pipeline points -> surface", lambda: pipeline(pp, 1.0 / 256), "%d points -> %d vertices, %d faces" % (len(pp), len(mv), len(mf)))

from oracle import oracle as O
hp = pts.cpu().numpy()
def host():
    r = (hp.astype(np.float64) / s)
    t = np.trunc(r)
    r = np.where(np.abs(r - t) >= 0.5, t + np.sign(r), t).astype(np.int64)
    codes = O.morton_encode(r)
    u, inv = np.unique(codes, return_inverse=True)
    return O.morton_decode(u), inv
t0 = time.perf_counter(); host(); print("numpy restatement of points -> grid on the host: %.1f ms" % (1e3 * (time.perf_counter() - t0)), flush=True)
