"""mesh_principal_curvatures: time per call and per phase on the subdivision-8 icosphere (1 310 720 faces) with 1 %
normal noise, float32 and float64, in the one-ring mode and in the ball mode at r = 3 and 6 mean edge lengths
(device-resident inputs, warm-up, L2 flushed before every timed call).

The calls are timed with CUDA events around the public call (it synchronises the host once).  The phases come from a
torch.profiler pass of their own, summed kernel times: face (mg_face), incidence (mg_corner, the sort, mg_rows),
normals (mg_vertex_normal), then curv_face and curv_vertex (one-ring) or binning (the grid build and cell_order) and
ball (curv_ball).  "neighbours": the mean number of other vertices in a ball, counted on the host.  "bytes": the
inputs read, the outputs written and the fp64 scratch each pass writes and reads once (one-ring: unit normals, corner
weights, halfcot, dblA, the frames and forms, the corner CSR and the vertex normals); "at 3.35 TB/s" is the time those
bytes alone would take at the H100's HBM3 data-sheet bandwidth.  The numpy restatement of tests/test_mesh_curvature.py
is timed on the host for context (the ball mode on 2000 vertices, scaled to all of them).
`python tools/curvature_time.py`; the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import time
import numpy as np
import torch
from scipy.spatial import cKDTree
from meshes import noisy_icosphere
from timing import card, timeit
import pcu_b200 as pcu
import test_mesh_curvature as restatement

PHASES = [("face", ("mg_face",)), ("incidence", ("mg_corner", "sort_", "mg_rows")), ("normals", ("mg_vertex_normal",)),
          ("curv_face", ("curv_face",)), ("curv_vertex", ("curv_vertex",)), ("ball", ("curv_ball",))]


def phases(fn):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    tot = {name: 0.0 for name, _ in PHASES}
    other = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
        if t <= 0 or "Memset" in e.key or "Memcpy" in e.key:
            continue
        for name, keys in PHASES:
            if any(k in e.key for k in keys):
                tot[name] += t
                break
        else:
            other += t
    return "  ".join("%s %.3f" % (k, v) for k, v in tot.items() if v) + ("  binning %.3f" % other if other else "")


def main():
    print("card:", card())
    v64, f = noisy_icosphere(8, 0, 0.01)
    nv, m = len(v64), len(f)
    el = float(np.linalg.norm(v64[f[:, 0]] - v64[f[:, 1]], axis=1).mean())
    print("icosphere: %d vertices, %d faces, mean edge %.5f" % (nv, m, el))
    ft = torch.from_numpy(f).cuda()
    tree = cKDTree(v64)
    for dt in (torch.float32, torch.float64):
        vt = torch.from_numpy(v64).to(dt).cuda()
        es = vt.element_size()
        inp = vt.numel() * es + ft.numel() * 8
        out = 8 * nv * es
        common = 2 * (3 * m * 8 * 2) + 3 * m * 8 * 2 + (nv + 1 + 3 * m) * 4 * 2 + 3 * nv * 8 * 2   # unit, weights, sorted CSR, normals
        for label, r in (("one-ring", -1.0), ("ball 3 edges", 3 * el), ("ball 6 edges", 6 * el)):
            fn = lambda r=r: pcu.mesh_principal_curvatures(vt, ft, r)
            med, mn = timeit(fn, warm=2, it=7)
            if r < 0:
                extra = (m * 8 + 3 * m * 8) * 2 + 6 * m * 8 * 2 + 3 * m * 8   # dblA, halfcot, frames + forms, corner areas
                nb = ""
            else:
                extra = nv * (4 * es) * 3   # binned points written, sorted, read
                sample = np.random.default_rng(0).choice(nv, 20000, replace=False)
                nb = "  neighbours %.1f" % (np.mean(tree.query_ball_point(v64[sample], r, return_length=True)) - 1)
            nbytes = inp + out + common + extra
            print("%-8s %-14s median %8.3f ms  min %8.3f ms  bytes %6.1f MB (%.3f ms at 3.35 TB/s)%s  phases: %s"
                  % (str(dt).replace("torch.", ""), label, med, mn, nbytes / 1e6, nbytes / 3.35e9, nb, phases(fn)))
    t0 = time.perf_counter()
    restatement.curvatures(v64, f)
    print("numpy restatement, one-ring: %.2f s" % (time.perf_counter() - t0))
    rows = np.random.default_rng(1).choice(nv, 2000, replace=False)
    for k in (3, 6):
        t0 = time.perf_counter()
        restatement.curvatures(v64, f, k * el, rows)
        print("numpy restatement, ball %d edges: %.1f s for all vertices (2000 timed)" % (k, (time.perf_counter() - t0) * nv / len(rows)))


if __name__ == "__main__":
    main()
