"""adjacency_list and pointcloud_sphere_geometry: time per call.

adjacency_list runs on the subdivision-8 icosphere (1.31 * 10^6 faces, int64, device-resident): with return_csr=True
(median of 5 after a warm-up; the call synchronises to read its sizes, so a host clock around it ends synchronised),
then with Python lists (median of 3), then the numpy restatement on the host for context (one sort-based unique over
the directed edges).  The CSR call's kernels come from a torch.profiler pass of their own, summed per phase: validate
(cc_validate), edges (lap_edge), sort (the record sort's kernels), runs (mc_heads and the compaction scans), csr
(adj_entries, mg_rows) and emit (adj_emit).

pointcloud_sphere_geometry runs on 10^6 points at 8 x 8 and 10^5 points at 16 x 32, fp32 and fp64, CUDA tensors: the
call from CUDA events (median of 10 after a warm-up), the kernel from a profiler pass, and the bytes the kernel must
move (the vertices and faces written, the points and radii read) against 3.35 TB/s, the H100 SXM's data-sheet HBM3
bandwidth.

`python tools/adjacency_time.py [out.json]`; the card's name and power limit are printed first."""
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
from timing import card, timeit  # noqa: E402
import pcu_b200 as pcu  # noqa: E402

PEAK_BYTES = 3.35e12
PHASES = [("validate", ("cc_validate",)), ("edges", ("lap_edge",)), ("sort", ("sort_",)),
          ("runs", ("mc_heads", "keep_count", "keep_offsets")), ("csr", ("adj_entries", "mg_rows")), ("emit", ("adj_emit",))]


def host_csr(f):
    """The numpy restatement: offsets and neighbours from one unique over the directed edges."""
    n = int(f.max()) + 1
    src, dst = f.ravel(), f[:, [1, 2, 0]].ravel()
    key = np.unique(np.concatenate([src * n + dst, dst * n + src]))
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(key // n, minlength=n))
    return offsets, key % n


def host_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return 1e3 * statistics.median(times), 1e3 * min(times)


def kernel_ms(fn, classify):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = classify(e.name)
        if k is not None:
            out[k] = out.get(k, 0.0) + e.device_time / 1e3
    return {k: round(x, 4) for k, x in sorted(out.items())}


def phase_of(name):
    for phase, keys in PHASES:
        if any(k in name for k in keys):
            return phase
    return "other"


def adjacency_rows():
    _, f = icosphere(8)
    ft = torch.from_numpy(f).cuda()
    o, nb = pcu.adjacency_list(ft, return_csr=True)
    wo, wnb = host_csr(f)
    assert np.array_equal(o.cpu().numpy(), wo) and np.array_equal(nb.cpu().numpy(), wnb)
    csr_med, csr_min = host_time(lambda: pcu.adjacency_list(ft, return_csr=True), 5)
    lists_med, lists_min = host_time(lambda: pcu.adjacency_list(ft), 3)
    t0 = time.perf_counter()
    host_csr(f)
    host_ms = 1e3 * (time.perf_counter() - t0)
    phases = kernel_ms(lambda: pcu.adjacency_list(ft, return_csr=True), phase_of)
    row = {"what": "adjacency_list", "faces": len(f), "lists": len(wo) - 1, "entries": len(wnb),
           "csr_ms": round(csr_med, 3), "csr_ms_min": round(csr_min, 3), "lists_ms": round(lists_med, 3),
           "lists_ms_min": round(lists_min, 3), "numpy_host_ms": round(host_ms, 3), "csr_kernels_ms": phases,
           "csr_kernels_total_ms": round(sum(phases.values()), 4)}
    print(json.dumps(row), flush=True)
    return row


def sphere_rows():
    rows = []
    rng = np.random.default_rng(0)
    for n, stacks, slices in ((1_000_000, 8, 8), (100_000, 16, 32)):
        for dt in (torch.float32, torch.float64):
            p = torch.from_numpy(rng.standard_normal((n, 3))).to(device="cuda", dtype=dt)
            r = torch.from_numpy(0.01 + 0.01 * rng.random(n)).to(device="cuda", dtype=dt)
            call = lambda: pcu.pointcloud_sphere_geometry(p, r, stacks, slices)   # noqa: E731
            call_ms, call_ms_min = timeit(call, warm=1, flush=False)
            kern = kernel_ms(call, lambda name: "kernel" if "sp_geometry" in name else None).get("kernel", float("nan"))
            V, F, size = (stacks + 1) * (slices + 1), 2 * (stacks - 1) * slices, p.element_size()
            moved = n * (V * 3 * size + F * 12 + 4 * size)
            row = {"what": "pointcloud_sphere_geometry", "points": n, "stacks": stacks, "slices": slices,
                   "dtype": str(dt).replace("torch.", ""), "vertices": n * V, "faces": n * F, "bytes": moved,
                   "call_ms": round(call_ms, 4), "call_ms_min": round(call_ms_min, 4), "kernel_ms": kern,
                   "kernel_TBps": round(moved / (kern * 1e-3) / 1e12, 3), "share_of_3.35TBps": round(moved / (kern * 1e-3) / PEAK_BYTES, 3)}
            print(json.dumps(row), flush=True)
            rows.append(row)
            del p, r
            torch.cuda.empty_cache()
    return rows


def main():
    print(card(), flush=True)
    rows = [adjacency_rows()] + sphere_rows()
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
