"""make_mesh_watertight: time per call and per phase on a 1.3 * 10^6-face icosphere (r = 1, fp64 vertices, int64
faces, device-resident) at resolutions 2 * 10^4, 10^5 and 10^6.

The calls are timed end to end with a host clock (the call synchronises once per phase and once per flip pass, so it
ends synchronised), median of 5 after a warm-up call.  The phases come from a torch.profiler pass of their own, summed
kernel times: depth search (wt_bounds, vx_bounds, vx_tiles, vx_test_kernel<T, 0>), occupancy (vx_test_kernel<T, 2>),
exterior (ff_tile, ff_cross, wt_exterior), surface (wt_count, mc_tiles, wt_verts, wt_faces), tree (the closest-point
tree's build) and projection (mq_query, wt_propose, wt_flip, wt_commit).  The flip passes per round are counted from
the profile.  `python tools/watertight_time.py [out.json]`; the card's name and power limit are printed first."""
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

PHASES = [("depth search", ("wt_bounds", "vx_bounds", "vx_tiles", "vx_test_kernel<double, 0>")),
          ("occupancy", ("vx_test_kernel<double, 2>",)),
          ("exterior", ("ff_tile", "ff_cross", "wt_exterior")),
          ("surface", ("wt_count", "mc_tiles", "wt_verts", "wt_faces")),
          ("projection", ("mq_query", "wt_propose", "wt_flip", "wt_commit", "wt_start")),
          ("tree", ("mq_", "radix", "sort", "digit", "scan"))]


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
    for res in (20_000, 100_000, 1_000_000):
        vw, fw = pcu.make_mesh_watertight(vt, ft, res)                  # warm-up
        torch.cuda.synchronize()
        times = []
        for _ in range(5):
            t0 = time.perf_counter()
            pcu.make_mesh_watertight(vt, ft, res)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            pcu.make_mesh_watertight(vt, ft, res)
            torch.cuda.synchronize()
        phases, flips = {}, 0
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            p = phase_of(e.name)
            phases[p] = phases.get(p, 0.0) + e.device_time / 1e3
            flips += "wt_flip" in e.name
        side = float((vw.max(0).values - vw.min(0).values).max())
        row = {"resolution": res, "faces_in": len(f), "vw": len(vw), "fw": len(fw), "call_ms": 1e3 * statistics.median(times),
               "call_ms_min": 1e3 * min(times), "phases_ms": {k: round(x, 3) for k, x in sorted(phases.items())},
               "flip_passes": flips, "extent": side}
        rows.append(row)
        print(json.dumps(row))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
