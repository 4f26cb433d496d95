"""marching_cubes_sparse_voxel_grid: time per call and per phase (device-resident inputs, warm-up, L2 flushed before
every timed call).

  sphere  dense SDF of a sphere (r = 0.8) on a 256^3 lattice of [-1, 1]^3 (255^3 cubes): int32 cubes / fp32 scalars and
          coordinates, and int64 / fp64
  torus   narrow band of a torus SDF (R = 0.6, r = 0.25) on a 1024^3 lattice: the cubes whose 8 corners all lie within
          1.5 spacings of the surface, built in torch; int32 / fp32

The call is timed end to end with a host clock (it synchronises twice to size its buffers and outputs).  The phases
come from a torch.profiler pass of their own: classify + scan (mc_classify, mc_tiles), sort / owners (mc_slots, the
radix sort, mc_heads, mc_runs, mc_owner and their compactions) and emit (mc_emit), summed kernel times.  "bytes" is
cube_indices plus the outputs; "at 3.35 TB/s" is the time those bytes alone would take at the H100's HBM3 data-sheet
bandwidth.  `python tools/marching_cubes_time.py`; the card's name and power limit are printed first."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import time
import numpy as np
import torch
from timing import card
import pcu_b200 as pcu

flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2
OFF = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]


def lattice_coords(k, dt):
    ax = torch.linspace(-1, 1, k, device="cuda", dtype=torch.float64)
    z, y, x = torch.meshgrid(ax, ax, ax, indexing="ij")
    return torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], 1).to(dt)


def cubes_of(base, k, it):
    """(m, 8) corner indices of the cubes whose corner 0 has lattice index `base` (x fastest)."""
    off = torch.tensor([dx + k * dy + k * k * dz for dx, dy, dz in OFF], device="cuda", dtype=torch.int64)
    return (base[:, None] + off[None, :]).to(it)


def sphere(k, dt, it):
    gc = lattice_coords(k, dt)
    s = gc.double().norm(dim=1).sub(0.8).to(dt)
    idx = torch.arange(k ** 3, device="cuda", dtype=torch.int64).reshape(k, k, k)
    return s, gc, cubes_of(idx[:-1, :-1, :-1].reshape(-1), k, it)


def torus_band(k):
    """Only the band's corners are stored: the grid vertices are the band cubes' corners, renumbered."""
    h = 2.0 / (k - 1)
    ax = torch.linspace(-1, 1, k, device="cuda", dtype=torch.float64)
    keep = []
    for z0 in range(0, k - 1, 64):                        # slabs of z, to bound the temporaries
        z = ax[z0:min(z0 + 65, k)]
        zz, yy, xx = torch.meshgrid(z, ax, ax, indexing="ij")
        q = torch.sqrt(xx * xx + yy * yy) - 0.6
        d = (torch.sqrt(q * q + zz * zz) - 0.25).abs() <= 1.5 * h
        c = d[:-1, :-1, :-1] & d[1:, :-1, :-1] & d[:-1, 1:, :-1] & d[:-1, :-1, 1:] & d[1:, 1:, :-1] & d[1:, :-1, 1:] \
            & d[:-1, 1:, 1:] & d[1:, 1:, 1:]
        iz, iy, ix = torch.nonzero(c, as_tuple=True)
        keep.append(ix + k * iy + k * k * (iz + z0))
    cubes = cubes_of(torch.cat(keep), k, torch.int64)
    verts, inv = torch.unique(cubes.reshape(-1), return_inverse=True)
    x, y, z = ax[verts % k], ax[(verts // k) % k], ax[verts // (k * k)]
    gc = torch.stack([x, y, z], 1).float()
    q = torch.sqrt(x * x + y * y) - 0.6
    s = (torch.sqrt(q * q + z * z) - 0.25).float()
    return s, gc, inv.reshape(-1, 8).int()


def timeit(fn, warm=3, it=10):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(it):
        flush_buf.add_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), float(np.min(ts))


def phases(fn):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    out = {"classify+scan": 0.0, "sort/owners": 0.0, "emit": 0.0}
    for e in prof.key_averages():
        name, us = e.key, e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if "mc_classify" in name or "mc_tiles" in name:
            out["classify+scan"] += us
        elif "mc_emit" in name:
            out["emit"] += us
        elif any(k in name for k in ("mc_slots", "sort_", "mc_heads", "mc_runs", "mc_owner", "keep_count", "keep_offsets")):
            out["sort/owners"] += us
    return {k: v / 1e3 for k, v in out.items()}


print(card(), flush=True)
runs = [("sphere 256^3 int32/fp32", lambda: sphere(256, torch.float32, torch.int32)),
        ("sphere 256^3 int64/fp64", lambda: sphere(256, torch.float64, torch.int64)),
        ("torus band 1024^3 int32/fp32", lambda: torus_band(1024))]
for name, make in runs:
    s, gc, ci = make()
    torch.cuda.synchronize()
    call = lambda: pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.0)
    v, f = call()
    med, mn = timeit(call)
    ph = phases(call)
    nbytes = ci.numel() * ci.element_size() + v.numel() * v.element_size() + f.numel() * f.element_size()
    print("%s: %d cubes, %d grid vertices -> #v %d, #f %d; call median %.3f ms min %.3f ms; phases (kernel ms) %s; "
          "bytes %.1f MB = %.3f ms at 3.35 TB/s"
          % (name, ci.shape[0], gc.shape[0], v.shape[0], f.shape[0], med, mn,
             " ".join("%s %.3f" % kv for kv in ph.items()), nbytes / 1e6, nbytes / 3.35e12 * 1e3), flush=True)
    del s, gc, ci, v, f
    torch.cuda.empty_cache()
