"""voxelize_triangle_mesh and flood_fill_3d: time per call and per phase (device-resident inputs, warm-up, L2 flushed
before every timed call).

  sphere mesh   a UV sphere of 10^6 faces (r = 1), voxelized at 256^3 and 1024^3 grid extents (voxel size 2 / 256 and
                2 / 1024), fp32 and fp64 vertices, int32 faces
  tilted cube   12 triangles of a cube 512 voxels on a side, rotated: about 10^8 candidates per face
  flood fill    the surface voxels of a sphere (r = 0.45 n) in an n^3 grid, the exterior flooded from a corner: n = 256
                and 512, int32 and float32
  serpentine    a one-voxel corridor of about 10^6 voxels through a 161^3 grid, flooded from one end (int32)

The calls are timed end to end with a host clock (voxelize_triangle_mesh synchronises twice to size its buffers and
its output; flood_fill_3d does not synchronise, the timer does).  The phases come from a torch.profiler pass of their
own, summed kernel times: voxelization bounds + scan (vx_bounds, vx_tiles), count (vx_test_kernel<T, false>), emit
(vx_test_kernel<T, true>), sort + unique (the radix sort, mc_heads, keep_count, keep_offsets) and decode (vx_decode);
flood fill tile (ff_tile), cross (ff_cross) and out (ff_out).  "bytes": for the voxelization the accepted codes (8
bytes per accepted (face, voxel) pair), for the flood fill the grid read plus the output written; "at 3.35 TB/s" is
the time those bytes alone would take at the H100's HBM3 data-sheet bandwidth.  `python tools/voxelize_time.py`; the
card's name and power limit are printed first."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import math
import time
import numpy as np
import torch
from timing import card
import pcu_b200 as pcu

flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2


def sphere_mesh(n_lat, n_lon):
    """A closed UV sphere (r = 1) built in torch: n_lon (2 n_lat - 2) faces."""
    th = torch.linspace(0, math.pi, n_lat + 1, dtype=torch.float64)[1:-1]
    ph = torch.arange(n_lon, dtype=torch.float64) * (2 * math.pi / n_lon)
    ring = torch.stack([torch.outer(th.sin(), ph.cos()), torch.outer(th.sin(), ph.sin()),
                        th.cos()[:, None].expand(-1, n_lon)], -1).reshape(-1, 3)
    v = torch.cat([torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float64), ring, torch.tensor([[0.0, 0.0, -1.0]], dtype=torch.float64)])
    j = torch.arange(n_lon)
    jn = (j + 1) % n_lon
    faces = [torch.stack([torch.zeros_like(j), 1 + j, 1 + jn], 1)]
    i = torch.arange(n_lat - 2)[:, None]
    a, b = 1 + i * n_lon + j, 1 + i * n_lon + jn
    c, d = a + n_lon, b + n_lon
    faces += [torch.stack([a, c, d], -1).reshape(-1, 3), torch.stack([a, d, b], -1).reshape(-1, 3)]
    base = 1 + (n_lat - 2) * n_lon
    faces.append(torch.stack([base + j, torch.full_like(j, len(v) - 1), base + jn], 1))
    return v.cuda(), torch.cat(faces).int().cuda()


def tilted_cube(k):
    c = torch.tensor([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=torch.float64) - 0.5
    f = torch.tensor([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                      [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=torch.int32)
    ax, ay = 0.5, 0.3
    rx = torch.tensor([[1, 0, 0], [0, math.cos(ax), -math.sin(ax)], [0, math.sin(ax), math.cos(ax)]], dtype=torch.float64)
    ry = torch.tensor([[math.cos(ay), 0, math.sin(ay)], [0, 1, 0], [-math.sin(ay), 0, math.cos(ay)]], dtype=torch.float64)
    return ((c @ rx.T @ ry.T) * k + 0.123).cuda(), f.cuda()


def shell_grid(n, dt):
    ax = torch.arange(n, device="cuda", dtype=torch.float64) - (n - 1) / 2
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    r = torch.sqrt(x * x + y * y + z * z)
    return ((r - 0.45 * n).abs() <= 0.87).to(dt)


def serpentine(X):
    g = torch.ones((2 * X + 1,) * 3, dtype=torch.int32)
    xs, ys, zs = torch.meshgrid(torch.arange(X), torch.arange(X), torch.arange(X), indexing="ij")
    ys = torch.where(xs % 2 == 1, X - 1 - ys, ys)
    row = xs * X + torch.arange(X)[None, :, None]
    zs = torch.where(row % 2 == 1, X - 1 - zs, zs)
    cells = torch.stack([xs, ys, zs], -1).reshape(-1, 3) * 2 + 1
    g[tuple(cells.T)] = 0
    mid = (cells[1:] + cells[:-1]) // 2
    g[tuple(mid.T)] = 0
    return g.cuda(), tuple(int(t) for t in cells[0])


def timeit(fn, warm=3, it=10):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(it):
        flush_buf.add_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), float(np.min(ts))


VX_PHASES = [("bounds+scan", ("vx_bounds", "vx_tiles")), ("count", ("vx_test_kernel<float, false>", "vx_test_kernel<double, false>")),
             ("emit", ("vx_test_kernel<float, true>", "vx_test_kernel<double, true>")),
             ("sort+unique", ("sort_", "mc_heads", "keep_count", "keep_offsets")), ("decode", ("vx_decode",))]
FF_PHASES = [("tile", ("ff_tile",)), ("cross", ("ff_cross",)), ("out", ("ff_out",))]


def phases(fn, table):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    out = {k: 0.0 for k, _ in table}
    for e in prof.key_averages():
        name, us = e.key, e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        for k, keys in table:
            if any(s in name for s in keys):
                out[k] += us
                break
    return " ".join("%s %.3f" % (k, v / 1e3) for k, v in out.items())


def accepted_pairs(v, f, size):
    """The accepted (face, voxel) count, from the prepare call's second count."""
    from pcu_b200 import _pcu_internal as I
    stream = torch.cuda.current_stream().cuda_stream
    h, n, acc = I._voxelize_prepare_device(v.dtype == torch.float64, v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], 0,
                                           [size] * 3, [0.0] * 3, v.device.index or 0, stream)
    I._voxelize_destroy(h)
    return n, acc


print(card(), flush=True)
v64, f = sphere_mesh(708, 708)
cube_v, cube_f = tilted_cube(512)
vx_runs = [("sphere 1.0e6 faces 256^3 fp32", v64.float(), f, 2.0 / 256), ("sphere 1.0e6 faces 256^3 fp64", v64, f, 2.0 / 256),
           ("sphere 1.0e6 faces 1024^3 fp32", v64.float(), f, 2.0 / 1024), ("sphere 1.0e6 faces 1024^3 fp64", v64, f, 2.0 / 1024),
           ("tilted cube 512 fp64", cube_v, cube_f, 1.0)]
for name, v, ff, size in vx_runs:
    call = lambda: pcu.voxelize_triangle_mesh(v, ff, size, (0.0, 0.0, 0.0))
    n, acc = accepted_pairs(v, ff, size)
    med, mn = timeit(call, warm=2, it=5 if "cube" in name else 10)
    nbytes = 8 * acc
    print("%s: %d faces -> %d accepted pairs, %d voxels; call median %.3f ms min %.3f ms; phases (kernel ms) %s; "
          "accepted-code bytes %.1f MB = %.3f ms at 3.35 TB/s"
          % (name, ff.shape[0], acc, n, med, mn, phases(call, VX_PHASES), nbytes / 1e6, nbytes / 3.35e12 * 1e3), flush=True)
for n in (256, 512):
    for dt in (torch.int32, torch.float32):
        g = shell_grid(n, dt)
        call = lambda: pcu.flood_fill_3d(g, (0, 0, 0), 2)
        med, mn = timeit(call)
        nbytes = 2 * g.numel() * g.element_size()
        print("flood fill shell %d^3 %s: call median %.3f ms min %.3f ms; phases (kernel ms) %s; bytes %.1f MB = %.3f ms "
              "at 3.35 TB/s" % (n, str(dt).replace("torch.", ""), med, mn, phases(call, FF_PHASES), nbytes / 1e6,
                                nbytes / 3.35e12 * 1e3), flush=True)
        del g
g, a = serpentine(80)
call = lambda: pcu.flood_fill_3d(g, a, 7)
med, mn = timeit(call)
nbytes = 2 * g.numel() * g.element_size()
print("serpentine %d voxels in 161^3 int32: call median %.3f ms min %.3f ms; phases (kernel ms) %s; bytes %.1f MB = %.3f ms "
      "at 3.35 TB/s" % (int((g == 0).sum()), med, mn, phases(call, FF_PHASES), nbytes / 1e6, nbytes / 3.35e12 * 1e3), flush=True)
