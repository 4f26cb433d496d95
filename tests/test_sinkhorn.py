"""Dense metrics (SURVEY.md 8f, N4; /root/reference/point_cloud_utils/_sinkhorn.py:4-156): pairwise_distances,
sinkhorn, earth_movers_distance.  The golden vectors were produced by the reference's own numpy code
(oracle/make_golden_sinkhorn.py).  CPU: the restatement reproduces them bit for bit.  GPU: the kernels agree with
them within the stated tolerances -- pairwise p = 2 / 1 / inf / -inf / 0 exactly (same rounded operations, summed in
numpy's pairwise order, which for these d = 3 goldens is a plain sequential sum), general p to a relative 5e-7 /
1e-15 (pow is evaluated in fp64 on the device, in the array's precision by numpy); the Sinkhorn plan to 2e-3 relative
in float32 and 1e-9 in float64 (the potentials enter the plan divided by eps, which amplifies the rounding of the two
reductions -- numpy sums pairwise in the array's precision, the kernels accumulate in fp64 -- by 1 / eps).
tests/test_dense_metrics.py covers d >= 8, non-finite inputs, edge shapes and the iteration count."""
import numpy as np
import pytest

from conftest import load_golden


def _cases():
    g = load_golden("sinkhorn_ref")
    return g, [str(c) for c in g["cases"]]


def test_restatement_matches_the_reference(oracle):
    from oracle import sinkhorn_oracle as S
    g, cases = _cases()
    for tag in cases:
        a, b = g[tag + "_a"], g[tag + "_b"]
        M = S.pairwise_distances(a, b)
        assert M.dtype == a.dtype and np.array_equal(M, g[tag + "_M"])
        for p, key in ((1, "1"), (np.inf, "inf"), (-np.inf, "neginf"), (0, "0"), (3, "3")):
            assert np.array_equal(S.pairwise_distances(a, b, p), g[tag + "_M_p" + key])
        P = S.sinkhorn(g[tag + "_wa"], g[tag + "_wb"], M, float(g[tag + "_eps"]))
        assert P.shape == g[tag + "_P"].shape and np.array_equal(P, g[tag + "_P"])
    emd, P = S.earth_movers_distance(g["emd_p"], g["emd_q"], eps=1e-3)
    assert emd == float(g["emd_value"]) and np.array_equal(P, g["emd_P"])


def test_shape_and_dtype_rules(pcu):
    a = np.random.rand(5, 3)
    with pytest.raises(ValueError):
        pcu.pairwise_distances(a[0], a)                       # 1-D input
    with pytest.raises(ValueError):
        pcu.sinkhorn(np.ones(5) / 5, np.ones(5) / 5, np.zeros((5, 5), np.float32), 1e-3)      # dtype mismatch (:88-90)
    with pytest.raises(ValueError):
        pcu.sinkhorn(np.ones(4) / 4, np.ones(5) / 5, np.zeros((5, 5)), 1e-3)                  # a does not match M (:91-93)
    with pytest.raises(ValueError):
        pcu.sinkhorn(np.ones((2, 5)) / 5, np.ones(5) / 5, np.zeros((5, 5)), 1e-3)             # 2-D weights with a 2-D M (:66-68)
    with pytest.raises(ValueError):
        pcu.earth_movers_distance(a.astype(np.float32), a.astype(np.float32))                 # float64 weights vs float32 M, as in the reference


@pytest.mark.gpu
def test_kernels_match_the_reference_goldens(pcu):
    g, cases = _cases()
    for tag in cases:
        a, b = g[tag + "_a"], g[tag + "_b"]
        f32 = a.dtype == np.float32
        M = pcu.pairwise_distances(a, b)
        assert M.dtype == a.dtype and M.shape == g[tag + "_M"].shape
        assert np.array_equal(M, g[tag + "_M"])
        for p, key in ((1, "1"), (np.inf, "inf"), (-np.inf, "neginf"), (0, "0")):
            assert np.array_equal(pcu.pairwise_distances(a, b, p), g[tag + "_M_p" + key]), (tag, p)
        assert np.allclose(pcu.pairwise_distances(a, b, 3), g[tag + "_M_p3"], rtol=5e-7 if f32 else 1e-15, atol=0)
        P = pcu.sinkhorn(g[tag + "_wa"], g[tag + "_wb"], g[tag + "_M"], float(g[tag + "_eps"]))
        ref = g[tag + "_P"]
        assert P.dtype == ref.dtype and P.shape == ref.shape
        scale = np.abs(ref).max()
        assert np.abs(P - ref).max() <= (2e-3 if f32 else 1e-9) * scale, (tag, float(np.abs(P - ref).max() / scale))
        # the last half-iteration fixed v: the column marginals of the plan are the weights b (the row marginals are not
        # there yet at these eps after 100 iterations -- in the reference just the same)
        wb = np.atleast_2d(g[tag + "_wb"])
        P3 = P if P.ndim == 3 else P[None]
        assert np.abs(P3.sum(1) - wb).sum(1).max() < 1e-2
    emd, P = pcu.earth_movers_distance(g["emd_p"], g["emd_q"], eps=1e-3)
    assert abs(float(emd) - float(g["emd_value"])) <= 1e-9 * float(g["emd_value"])
    assert np.abs(P - g["emd_P"]).max() <= 1e-9 * np.abs(g["emd_P"]).max()


@pytest.mark.gpu
def test_cuda_tensors_and_the_reference_test_shapes(pcu):
    """tests/test_examples.py:289-335: 100 x 100 and batched (3, 100, 100) problems, eps = 1e-3; CUDA tensors stay on the device."""
    import torch
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(4)
    a, b = rng.random((3, 100, 3)), rng.random((3, 100, 3))
    M = pcu.pairwise_distances(a, b)
    assert np.array_equal(M, S.pairwise_distances(a, b))
    w = np.ones((3, 100)) / 100
    P = pcu.sinkhorn(w, w, M, eps=1e-3)
    ref = S.sinkhorn(w, w, M, 1e-3)
    assert np.abs(P - ref).max() <= 1e-9 * np.abs(ref).max()
    at, bt = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    Mt = pcu.pairwise_distances(at, bt)
    assert Mt.is_cuda and torch.equal(Mt.cpu(), torch.from_numpy(M))
    wt = torch.from_numpy(w).cuda()
    Pt = pcu.sinkhorn(wt, wt, Mt, eps=1e-3)
    assert Pt.is_cuda and np.array_equal(Pt.cpu().numpy(), P)
    emd, Pe = pcu.earth_movers_distance(at[0], bt[0], eps=1e-3)
    ref_emd, ref_P = S.earth_movers_distance(a[0], b[0], eps=1e-3)
    assert emd.is_cuda and abs(float(emd) - ref_emd) <= 1e-9 * ref_emd
