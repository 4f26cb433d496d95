"""mesh_face_areas, estimate_mesh_face_normals, estimate_mesh_vertex_normals and laplacian_smooth_mesh: time per call
and per phase on the subdivision-8 icosphere (1 310 720 faces) with 1 % normal noise, float32 and float64
(device-resident inputs, warm-up, L2 flushed before every timed call).

The calls are timed with CUDA events around the public call (every call synchronises the host at least once).  The
phases come from a torch.profiler pass of their own, summed kernel times: face (mg_face), incidence (mg_corner, the
sort, mg_rows), vertex (mg_vertex_normal); for the smoothing load (lap_load), assembly (lap_edge, the sorts, heads,
keep_count / keep_offsets, lap_entries, mg_rows, lap_diag, and the incidence in cotan mode), mass (face pass + lap_mass),
cg (lap_cg_*), rescale (face pass + lap_rescale) and store.  Smoothing runs both modes at num_iters = 4 and prints the
CG iterations of every step.  "bytes": the inputs read plus the outputs written, and for the smoothing the CSR of L
(int32 columns, fp64 values, row pointers, diagonal) once; "at 3.35 TB/s" is the time those bytes alone would take at
the H100's HBM3 data-sheet bandwidth.  scipy's host solve (spsolve of the same system, one step) is printed for
context.  `python tools/mesh_geometry_time.py`; the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import time
import numpy as np
import torch
from meshes import noisy_icosphere
from timing import card, timeit
import pcu_b200 as pcu
from pcu_b200 import _mesh_geometry


NORMAL_PHASES = [("face", ("mg_face",)), ("incidence", ("mg_corner", "sort_", "mg_rows")), ("vertex", ("mg_vertex_normal",))]
SMOOTH_PHASES = [("load", ("lap_load",)), ("assembly", ("lap_edge", "sort_", "mc_heads", "keep_", "lap_entries", "mg_rows",
                                                         "lap_diag", "mg_corner")),
                 ("face passes", ("mg_face",)), ("mass", ("lap_mass",)), ("cg", ("lap_cg_",)), ("rescale", ("lap_rescale",)),
                 ("store", ("lap_store",))]


def phases(fn, table):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    tot = {name: 0.0 for name, _ in table}
    other = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
        if t <= 0 or not any(k in e.key for k in ("kernel", "pcu", "sort", "keep", "lap_", "mg_", "mc_")):
            continue
        for name, keys in table:
            if any(k in e.key for k in keys):
                tot[name] += t
                break
        else:
            other += t
    return "  ".join("%s %.3f" % (k, v) for k, v in tot.items()) + ("  other %.3f" % other if other else "")


def main():
    print("card:", card())
    v64, f = noisy_icosphere(8, 0, 0.01)
    nv, m = len(v64), len(f)
    print("icosphere: %d vertices, %d faces" % (nv, m))
    ft = torch.from_numpy(f).cuda()
    for dt in (torch.float32, torch.float64):
        vt = torch.from_numpy(v64).to(dt).cuda()
        es = vt.element_size()
        inp = vt.numel() * es + ft.numel() * 8
        rows = [("mesh_face_areas", lambda: pcu.mesh_face_areas(vt, ft), inp + m * es, [("face", ("mg_face",))]),
                ("face normals", lambda: pcu.estimate_mesh_face_normals(vt, ft), inp + 3 * m * es, [("face", ("mg_face",))])]
        for w in ("uniform", "area", "angle"):
            rows.append(("vertex normals %s" % w, lambda w=w: pcu.estimate_mesh_vertex_normals(vt, ft, w), inp + 3 * nv * es, NORMAL_PHASES))
        for name, fn, nbytes, table in rows:
            med, mn = timeit(fn, warm=2, it=7)
            print("%-8s %-24s median %8.3f ms  min %8.3f ms  bytes %6.1f MB (%.3f ms at 3.35 TB/s)  phases: %s"
                  % (str(dt).replace("torch.", ""), name, med, mn, nbytes / 1e6, nbytes / 3.35e9, phases(fn, table)))
        csr = 6 * m * (4 + 8) + (nv + 1) * 4 + nv * 8   # upper bound: 6 entries per face before the runs are merged
        for cotan in (False, True):
            fn = lambda: _mesh_geometry._smooth(vt, ft, 4, 0.1, cotan, None)
            iters = fn()[1]
            med, mn = timeit(fn, warm=1, it=5)
            nbytes = inp + csr + 3 * nv * es
            print("%-8s %-24s median %8.3f ms  min %8.3f ms  bytes %6.1f MB (%.3f ms at 3.35 TB/s)  CG iterations per step %s  phases: %s"
                  % (str(dt).replace("torch.", ""), "smooth cotan=%d x4" % cotan, med, mn, nbytes / 1e6, nbytes / 3.35e9, iters,
                     phases(fn, SMOOTH_PHASES)))
    try:
        import scipy.sparse as sp
        import scipy.sparse.linalg as spl
        from test_laplacian_smooth_mesh import cot_laplacian
        t0 = time.perf_counter()
        off, diag = cot_laplacian(v64, f)
        S = (sp.eye(nv) - 0.1 * (off + sp.diags(diag))).tocsc()
        t1 = time.perf_counter()
        spl.spsolve(S, v64)
        t2 = time.perf_counter()
        print("scipy host: assembly %.1f ms, spsolve of one step %.1f ms" % (1e3 * (t1 - t0), 1e3 * (t2 - t1)))
    except ImportError as e:
        print("scipy host: not measured (%s)" % e)


if __name__ == "__main__":
    main()
