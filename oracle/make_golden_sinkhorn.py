"""Generates tests/golden/sinkhorn_ref.npz (d = 3) and tests/golden/sinkhorn_wide_ref.npz (d = 8 .. 130) by running
the REFERENCE's own numpy code (/root/reference/point_cloud_utils/_sinkhorn.py, loaded by path: the package __init__
needs the compiled module).

    python oracle/make_golden_sinkhorn.py
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("ref_sinkhorn", "/root/reference/point_cloud_utils/_sinkhorn.py")
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

rng = np.random.default_rng(77)
out = {}
cases = []
for tag, dtype, nb, n, m, eps in (("f64_single", np.float64, 0, 100, 100, 1e-3), ("f32_single", np.float32, 0, 64, 96, 1e-2),
                                  ("f64_batch", np.float64, 3, 50, 70, 5e-3), ("f32_batch", np.float32, 2, 128, 128, 2e-2)):
    shape_a = (n, 3) if nb == 0 else (nb, n, 3)
    shape_b = (m, 3) if nb == 0 else (nb, m, 3)
    a = rng.random(shape_a).astype(dtype)
    b = rng.random(shape_b).astype(dtype)
    M = ref.pairwise_distances(a, b)
    wa = rng.random(shape_a[:-1]).astype(dtype) + dtype(0.5)
    wb = rng.random(shape_b[:-1]).astype(dtype) + dtype(0.5)
    wa /= wa.sum(-1, keepdims=True)
    wb /= wb.sum(-1, keepdims=True)
    P = ref.sinkhorn(wa, wb, M, eps)
    out.update({tag + "_a": a, tag + "_b": b, tag + "_M": M, tag + "_wa": wa, tag + "_wb": wb, tag + "_P": P,
                tag + "_eps": np.float64(eps)})
    for p in (1, np.inf, -np.inf, 0, 3):
        out[tag + "_M_p%s" % str(p).replace("-", "neg")] = ref.pairwise_distances(a, b, p)
    cases.append(tag)
p = rng.random((80, 3)); q = rng.random((60, 3))          # test_examples.py:289-310 shapes, float64
emd, P = ref.earth_movers_distance(p, q, eps=1e-3)
out.update(emd_p=p, emd_q=q, emd_value=np.float64(emd), emd_P=P)
out["cases"] = np.array(cases)
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "sinkhorn_ref.npz"), **out)
print("written", len(out), "arrays; emd", emd)

# Wide points: numpy sums d >= 8 terms pairwise (eight partial sums, split above 128 terms), so these pin that order.
rng = np.random.default_rng(78)
out = {}
cases = []
for d in (8, 16, 33, 130):
    for dtype in (np.float32, np.float64):
        for nb in (0, 2):
            tag = "d%d_%s_%s" % (d, np.dtype(dtype).name, "single" if nb == 0 else "batch")
            n, m = (24, 20) if nb == 0 else (12, 16)
            shape_a = (n, d) if nb == 0 else (nb, n, d)
            shape_b = (m, d) if nb == 0 else (nb, m, d)
            a = (rng.standard_normal(shape_a) * 3).astype(dtype)
            b = (rng.standard_normal(shape_b) * 3).astype(dtype)
            M = ref.pairwise_distances(a, b)
            wa = rng.random(shape_a[:-1]).astype(dtype) + dtype(0.5)
            wb = rng.random(shape_b[:-1]).astype(dtype) + dtype(0.5)
            wa /= wa.sum(-1, keepdims=True)
            wb /= wb.sum(-1, keepdims=True)
            eps = 0.05 * float(M.mean())
            out.update({tag + "_a": a, tag + "_b": b, tag + "_wa": wa, tag + "_wb": wb, tag + "_eps": np.float64(eps),
                        tag + "_P": ref.sinkhorn(wa, wb, M, eps)})
            for p in (2, 1, np.inf, -np.inf, 0, 3):
                out[tag + "_M_p%s" % str(p).replace("-", "neg")] = ref.pairwise_distances(a, b, p)
            cases.append(tag)
p = rng.random((50, 16)); q = rng.random((40, 16))
emd, P = ref.earth_movers_distance(p, q, eps=1e-2)
out.update(emd_p=p, emd_q=q, emd_eps=np.float64(1e-2), emd_value=np.float64(emd), emd_P=P)
out["cases"] = np.array(cases)
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "sinkhorn_wide_ref.npz"), **out)
print("written", len(out), "arrays; emd", emd)
