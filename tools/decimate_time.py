"""decimate_triangle_mesh: time per call and per phase on a 1.3 * 10^6-face icosphere (r = 1, fp64 vertices, int64
faces, device-resident) at targets of 1/4, 1/20 and 1/100 of its faces.

The calls are timed end to end with a host clock (the call synchronises once per round and once for its output
counts, so it ends synchronised), median of 5 after a warm-up call.  The phases come from a torch.profiler pass of
their own, summed kernel times: adjacency (dc_records, dc_heads, dc_runs, and the first half of the record sort's
kernels), validity (dc_valid), ranking (dc_keys and the other half of the sort), selection (dc_stamp, dc_select),
collapse (dc_apply, dc_faces, dc_live), emit (the input check, dc_mark, dc_vrank, dc_fout, dc_emit) and the shared
compaction scans (keep_count, keep_offsets) on their own.  The two sorts of a round launch the same kernels, so their
time is reported together as "sorts".  `python tools/decimate_time.py [out.json]`; the card's name and power limit are
printed first."""
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402
from meshes import icosphere  # noqa: E402
from timing import card  # noqa: E402
import pcu_b200 as pcu  # noqa: E402

PHASES = [("adjacency", ("dc_records", "dc_heads", "dc_runs", "dc_accept")),
          ("validity", ("dc_valid",)),
          ("ranking", ("dc_keys",)),
          ("sorts", ("sort_",)),
          ("selection", ("dc_stamp", "dc_select")),
          ("collapse", ("dc_apply", "dc_faces_kernel", "dc_live")),
          ("compaction scans", ("keep_count", "keep_offsets")),
          ("emit", ("dc_faces_in", "dc_verts_in", "dc_mark", "dc_vrank", "dc_fout", "dc_emit"))]


def phase_of(name):
    for phase, keys in PHASES:
        if any(k in name for k in keys):
            return phase
    return "other"


def main():
    print(card())
    v, f = icosphere(8)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    rows = []
    for frac in (4, 20, 100):
        target = len(f) // frac
        vo, fo, _, _ = pcu.decimate_triangle_mesh(vt, ft, target)               # warm-up
        torch.cuda.synchronize()
        times = []
        for _ in range(5):
            t0 = time.perf_counter()
            pcu.decimate_triangle_mesh(vt, ft, target)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            pcu.decimate_triangle_mesh(vt, ft, target)
            torch.cuda.synchronize()
        phases, rounds = {}, 0
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            p = phase_of(e.name)
            phases[p] = phases.get(p, 0.0) + e.device_time / 1e3
            rounds += "dc_apply" in e.name
        row = {"target": target, "faces_in": len(f), "v_out": len(vo), "f_out": len(fo), "rounds": rounds,
               "call_ms": 1e3 * statistics.median(times), "call_ms_min": 1e3 * min(times),
               "phases_ms": {k: round(x, 3) for k, x in sorted(phases.items())}}
        rows.append(row)
        print(json.dumps(row))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
