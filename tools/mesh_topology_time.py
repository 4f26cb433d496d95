"""connected_components, remove_mesh_vertices and remove_unreferenced_mesh_vertices: time per call and per phase
(device-resident inputs, warm-up, L2 flushed before every timed call).

  sphere          the subdivision-8 icosphere, 1 310 720 faces, vertices numbered by subdivision
  permuted        the same sphere with its vertex order randomly permuted
  disjoint        10^6 disjoint triangles, corners randomly numbered
  strip           a triangle strip of 10^6 faces numbered along the strip: (i, i + 1, i + 2)
  marching cubes  marching cubes of a smoothed noise field on a 160^3 lattice: thousands of components
  removals        remove_mesh_vertices (mask z > -0.3) and remove_unreferenced_mesh_vertices (half the faces) on the sphere

The calls are timed with CUDA events around the public call (each synchronises the host: connected_components twice,
the removals once).  The phases come from a torch.profiler pass of their own, summed kernel times: validate, init +
hook, flatten, number (keep_count, keep_offsets, cc_rank), label (cc_label, cc_face) and emit; for the removals mark
(rur_mark / the mask's keep_count, keep_offsets), vertices (rmv_vertex / rur_vertex) and faces.  "bytes": f read plus
the outputs written; "at 3.35 TB/s" is the time those bytes alone would take at the H100's HBM3 data-sheet bandwidth.
scipy.sparse.csgraph.connected_components on the host is printed for context.  `python tools/mesh_topology_time.py`;
the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import time
import numpy as np
import scipy.sparse
import scipy.sparse.csgraph
import torch
from meshes import icosphere
from timing import card, timeit
import pcu_b200 as pcu


def noisy_mc(k=160, seed=5):
    g = torch.randn((k, k, k), generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    for ax in range(3):
        g = (g + g.roll(1, ax) + g.roll(-1, ax)) / 3.0
    ax_ = torch.linspace(-1, 1, k, dtype=torch.float64)
    z, y, x = torch.meshgrid(ax_, ax_, ax_, indexing="ij")
    gc = torch.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    idx = torch.arange(k ** 3).reshape(k, k, k)[:-1, :-1, :-1].ravel()
    off = torch.tensor([0, 1, 1 + k, k, k * k, 1 + k * k, 1 + k + k * k, k + k * k])
    return pcu.marching_cubes_sparse_voxel_grid((g.ravel() - 0.4).cuda(), gc.cuda(), (idx[:, None] + off).cuda(), 0.0)


CC_PHASES = [("validate", ("cc_validate",)), ("hook", ("cc_init", "cc_hook")), ("flatten", ("cc_flatten",)),
             ("number", ("keep_count", "keep_offsets", "cc_rank")), ("label", ("cc_label", "cc_face")), ("emit", ("cc_emit",))]
RM_PHASES = [("mark", ("rur_mark", "keep_count", "keep_offsets")), ("vertices", ("rmv_vertex", "rur_vertex")),
             ("faces", ("rmv_face", "rur_face"))]


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


def scipy_ms(f):
    F = f.cpu().numpy().astype(np.int64)
    n = int(F.max()) + 1
    t0 = time.perf_counter()
    g = scipy.sparse.coo_matrix((np.ones(2 * len(F), np.int8), (F[:, :2].ravel(), F[:, 1:].ravel())), shape=(n, n))
    k, _ = scipy.sparse.csgraph.connected_components(g, directed=False)
    return 1e3 * (time.perf_counter() - t0), k


print(card(), flush=True)
v, f = icosphere(8)
perm = np.random.default_rng(2).permutation(len(v))
inv = np.empty_like(perm)
inv[perm] = np.arange(len(v))
m = 10 ** 6
i = np.arange(m)
mcv, mcf = noisy_mc()
vt = torch.from_numpy(v).float().cuda()
cases = [("sphere", vt, torch.from_numpy(f).int().cuda()),
         ("permuted sphere", vt, torch.from_numpy(inv[f]).int().cuda()),
         ("disjoint triangles", torch.zeros((3 * m, 3), device="cuda"),
          torch.from_numpy(np.random.default_rng(4).permutation(3 * m).reshape(m, 3)).int().cuda()),
         ("numbered strip", torch.zeros((m + 2, 3), device="cuda"), torch.from_numpy(np.stack([i, i + 1, i + 2], 1)).int().cuda()),
         ("marching cubes", mcv, mcf)]
for name, cv_, cf_ in cases:
    call = lambda: pcu.connected_components(cv_, cf_)
    out = call()
    n, k = out[0].numel(), out[1].numel()
    med, mn = timeit(call)
    nbytes = cf_.numel() * cf_.element_size() + (n + 2 * k + cf_.shape[0]) * cf_.element_size()
    sp, ks = scipy_ms(cf_)
    assert ks == k
    print("connected_components %s: %d faces, %d vertices, %d components; call median %.3f ms min %.3f ms; phases (kernel ms) %s; "
          "bytes %.1f MB = %.3f ms at 3.35 TB/s; scipy on the host %.1f ms"
          % (name, cf_.shape[0], n, k, med, mn, phases(call, CC_PHASES), nbytes / 1e6, nbytes / 3.35e12 * 1e3, sp), flush=True)
ft = torch.from_numpy(f).int().cuda()
mask = vt[:, 2] > -0.3
call = lambda: pcu.remove_mesh_vertices(vt, ft, mask)
v2, f2 = call()
med, mn = timeit(call)
nbytes = ft.numel() * 4 + mask.numel() + vt.numel() * 4 + v2.numel() * 4 + f2.numel() * 4
print("remove_mesh_vertices sphere fp32 / int32: %d -> %d vertices, %d -> %d faces; call median %.3f ms min %.3f ms; phases (kernel ms) %s; "
      "bytes %.1f MB = %.3f ms at 3.35 TB/s" % (len(vt), len(v2), len(ft), len(f2), med, mn, phases(call, RM_PHASES), nbytes / 1e6,
                                                nbytes / 3.35e12 * 1e3), flush=True)
fh = ft[torch.rand(len(ft), generator=torch.Generator().manual_seed(0)) < 0.5].contiguous()
call = lambda: pcu.remove_unreferenced_mesh_vertices(vt, fh)
out = call()
med, mn = timeit(call)
nbytes = 2 * fh.numel() * 4 + vt.numel() * 4 + out[0].numel() * 4 + (out[2].numel() + out[3].numel()) * 4
print("remove_unreferenced_mesh_vertices sphere fp32 / int32, half the faces: %d -> %d vertices, %d faces; call median %.3f ms "
      "min %.3f ms; phases (kernel ms) %s; bytes %.1f MB = %.3f ms at 3.35 TB/s"
      % (len(vt), len(out[0]), len(fh), med, mn, phases(call, RM_PHASES), nbytes / 1e6, nbytes / 3.35e12 * 1e3), flush=True)
