"""orient_mesh_faces: time per call and per phase (device-resident inputs, warm-up, L2 flushed before every timed call,
median and minimum of 10).

  sphere           the subdivision-8 icosphere, 1 310 720 faces, half of them reversed, vertices numbered by subdivision
  permuted sphere  the same with its vertex order randomly permuted
  disjoint         10^6 disjoint triangles, corners randomly numbered (every face its own patch)
  moebius          a Moebius strip of 10^5 faces: one collapsed patch, answered by the one-thread replay
  welded           the subdivision-6 icosphere with its cap z > 0.8 removed and a degenerate face (a, b, b) welded onto
                   every boundary edge (a, b): 74 084 faces in one collapsed patch (irregular pairs), replayed
Each case runs with int32 faces, the sphere also with int64 (two key words per half-edge record, so twice the sort
passes over records of twice the size).  The call never synchronises the host; the timed window is CUDA events around
it.  The phases come from a torch.profiler pass of their own, summed kernel times: records, sort, runs (classification,
neighbour slots, unions), number (flatten, keep_count, keep_offsets, cc_rank), emit and replay.  "bytes": f read plus
the outputs written; "at 3.35 TB/s" is the time those bytes alone would take at the H100's HBM3 data-sheet bandwidth.
A host-side parity BFS with scipy (pair edges by a sort, components of the doubled face graph) on the same input is
printed for context; it does not replay collapsed patches.  `python tools/orient_time.py`; the card's name and power
limit are printed first.  Results are fp-independent: integer inputs, integer outputs."""
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


def moebius(n):
    i = np.arange(n)
    t, b = 2 * i, 2 * i + 1
    tn, bn = np.where(i + 1 < n, t + 2, 1), np.where(i + 1 < n, b + 2, 0)
    f = np.empty((2 * n, 3), np.int64)
    f[0::2] = np.stack([t, b, tn], 1)
    f[1::2] = np.stack([b, bn, tn], 1)
    return f


def reverse_half(f, seed=1):
    f = f.copy()
    r = np.random.default_rng(seed).random(len(f)) < 0.5
    f[r] = f[r][:, ::-1]
    return f


PHASES = [("records", ("om_records",)), ("sort", ("sort_",)), ("runs", ("om_runs",)),
          ("number", ("om_flatten", "keep_count", "keep_offsets", "cc_rank")), ("emit", ("om_emit",)), ("replay", ("om_replay",))]


def phases(fn):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    out = {k: 0.0 for k, _ in PHASES}
    for e in prof.key_averages():
        name, us = e.key, e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        for k, keys in PHASES:
            if any(s in name for s in keys):
                out[k] += us
                break
    return " ".join("%s %.3f" % (k, v / 1e3) for k, v in out.items())


def scipy_ms(F):
    """Host parity BFS: pair edges found by a sort, then the components of the doubled face graph."""
    t0 = time.perf_counter()
    m = len(F)
    frm = np.concatenate([F[:, 1], F[:, 2], F[:, 0]])
    to = np.concatenate([F[:, 2], F[:, 0], F[:, 1]])
    key = np.minimum(frm, to) * (1 << 32) + np.maximum(frm, to)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    start = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    length = np.diff(np.r_[start, len(ks)])
    two = start[length == 2]
    h0, h1 = order[two], order[two + 1]
    f0, f1 = h0 % m, h1 % m
    same = frm[h0] == frm[h1]
    a = np.concatenate([2 * f0, 2 * f0 + 1])
    b = np.concatenate([np.where(same, 2 * f1 + 1, 2 * f1), np.where(same, 2 * f1, 2 * f1 + 1)])
    g = scipy.sparse.coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(2 * m, 2 * m))
    scipy.sparse.csgraph.connected_components(g, directed=False)
    return 1e3 * (time.perf_counter() - t0)


print(card(), flush=True)
_, f = icosphere(8)
hf = reverse_half(f)
perm = np.random.default_rng(2).permutation(int(f.max()) + 1)
vs, ws = icosphere(6)
ws = ws[~(vs[ws][:, :, 2] > 0.8).all(1)]
e = np.concatenate([ws[:, [1, 2]], ws[:, [2, 0]], ws[:, [0, 1]]])
key = np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1])
u, cnt = np.unique(key, return_counts=True)
b = e[np.isin(key, u[cnt == 1])]
welded = np.concatenate([ws, np.stack([b[:, 0], b[:, 1], b[:, 1]], 1)])
m = 10 ** 6
cases = [("sphere int32", hf.astype(np.int32)), ("sphere int64", hf), ("permuted sphere int32", perm[hf].astype(np.int32)),
         ("disjoint int32", np.random.default_rng(4).permutation(3 * m).reshape(m, 3).astype(np.int32)),
         ("moebius int32", reverse_half(moebius(50000)).astype(np.int32)),
         ("welded int32", reverse_half(welded).astype(np.int32))]
for name, F in cases:
    ft = torch.from_numpy(F).cuda()
    call = lambda: pcu.orient_mesh_faces(ft)
    ff, comp = call()
    patches = int(comp.max()) + 1
    med, mn = timeit(call)
    nbytes = (2 * ft.numel() + len(F)) * ft.element_size()
    print("orient_mesh_faces %s: %d faces, %d patches; call median %.3f ms min %.3f ms; phases (kernel ms) %s; "
          "bytes %.1f MB = %.3f ms at 3.35 TB/s; scipy parity BFS on the host %.1f ms"
          % (name, len(F), patches, med, mn, phases(call), nbytes / 1e6, nbytes / 3.35e12 * 1e3, scipy_ms(F.astype(np.int64))), flush=True)
