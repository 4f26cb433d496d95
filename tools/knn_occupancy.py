"""k > 1: search / far-pass / replay times over cell occupancies, and the kd build's timeline.
python tools/knn_occupancy.py [n_queries] [m]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pcu_b200 as pcu
I = pcu._pcu_internal
n = int(sys.argv[1]) if len(sys.argv) > 1 else 2000000
m = int(sys.argv[2]) if len(sys.argv) > 2 else 1000000
dev = 0
stream = torch.cuda.current_stream().cuda_stream
g = torch.Generator(device="cuda").manual_seed(0)
d = torch.rand((m, 3), generator=g, device="cuda")
q = torch.rand((n, 3), generator=g, device="cuda")
for k, occs in ((16, (0, 4, 5, 6, 7, 8, 10, 12)), (8, (0, 2, 3, 4, 5, 6)), (4, (0, 1.5, 2, 3, 4)), (32, (0, 8, 12, 16, 20, 24))):
    dists = torch.empty((n, k), dtype=torch.float32, device="cuda")
    corrs = torch.empty((n, k), dtype=torch.int64, device="cuda")
    tied = torch.zeros(1, dtype=torch.int64, device="cuda")
    for occ in occs:
        I._set_defaults(cell_occupancy=float(occ), disable_tie_replay=1)
        I._set_profiling(dev, stream, True)
        acc = {}
        reps = 3
        for r in range(reps + 2):
            I._knn_device(False, q.data_ptr(), n, d.data_ptr(), m, k, False, dists.data_ptr(), corrs.data_ptr(), tied.data_ptr(), 10, dev, stream)
            torch.cuda.synchronize()
            if r >= 2:
                for key, val in I._last_profile(dev, stream).items():
                    acc[key] = acc.get(key, 0.0) + val / reps
        I._set_profiling(dev, stream, False)
        build = sum(acc.get(s, 0) for s in ("bbox+grid", "slab_count", "partition", "cell_sort"))
        print("k=%2d occupancy %5s: build %.3f  search %.3f  far %.3f ms   (per 10^6 queries: %.3f ms)" %
              (k, occ if occ else "dflt", build, acc.get("search", 0), acc.get("search_far", 0),
               (acc.get("search", 0) + acc.get("search_far", 0)) * 1e6 / n), flush=True)
    del dists, corrs
I._set_defaults()
# the kd build's timeline (full tree over the m dataset points: lattice queries force ties -> replay)
k = 16
lat = torch.stack(torch.meshgrid(*[torch.arange(40, device="cuda", dtype=torch.float32)] * 3, indexing="ij"), -1).reshape(-1, 3) / 40
dists = torch.empty((lat.shape[0], k), dtype=torch.float32, device="cuda")
corrs = torch.empty((lat.shape[0], k), dtype=torch.int64, device="cuda")
tied = torch.zeros(1, dtype=torch.int64, device="cuda")
for mode in (2, 0):
    I._set_defaults(disable_tie_replay=mode)
    for r in range(3):
        I._knn_device(False, lat.data_ptr(), lat.shape[0], d.data_ptr(), m, k, False, dists.data_ptr(), corrs.data_ptr(), tied.data_ptr(), 10, dev, stream)
        torch.cuda.synchronize()
    # dataset = a lattice too, so that ties really occur
    I._knn_device(False, q.data_ptr(), 100000, lat.data_ptr(), lat.shape[0], k, False, dists.data_ptr(), corrs.data_ptr(), tied.data_ptr(), 10, dev, stream)
    torch.cuda.synchronize()
    t = I._debug_kd_times(dev, stream)
    print("mode %d (lattice dataset %d pts, tied %d): set-up %.1f us, grid-wide levels %d: %s us, grid-wide total %.1f us, single-CTA subtrees %d: %.1f us" %
          (mode, lat.shape[0], int(tied.item()), (t[1] - t[0]) / 1e3, t[32], [round((t[2 + l] - (t[1 + l] if l else t[1])) / 1e3, 1) for l in range(min(int(t[32]), 28))],
           (t[30] - t[0]) / 1e3, t[33], (t[31] - t[30]) / 1e3), flush=True)
# the same on the uniform 10^6-point dataset with queries that tie: duplicate a few dataset points
dd = d.clone(); dd[:5000] = dd[5000:10000]
dists = torch.empty((n, k), dtype=torch.float32, device="cuda"); corrs = torch.empty((n, k), dtype=torch.int64, device="cuda")
for mode in (2, 0):
    I._set_defaults(disable_tie_replay=mode)
    for r in range(2):
        I._knn_device(False, q.data_ptr(), n, dd.data_ptr(), m, k, False, dists.data_ptr(), corrs.data_ptr(), tied.data_ptr(), 10, dev, stream)
        torch.cuda.synchronize()
    t = I._debug_kd_times(dev, stream)
    print("mode %d (uniform dataset %d pts, tied %d): set-up %.1f us, grid-wide levels %d: %s us, grid-wide total %.1f us, single-CTA subtrees %d: %.1f us" %
          (mode, m, int(tied.item()), (t[1] - t[0]) / 1e3, t[32], [round((t[2 + l] - (t[1 + l] if l else t[1])) / 1e3, 1) for l in range(min(int(t[32]), 28))],
           (t[30] - t[0]) / 1e3, t[33], (t[31] - t[30]) / 1e3), flush=True)
I._set_defaults()
