"""Dense metrics (csrc/sinkhorn.cuh) at the shapes and inputs where their kernels can go wrong: points with d >= 8
(numpy's pairwise summation order), grid tails in m, more than 65535 rows or batches, NaN / inf coordinates, zero
weights, infinite costs and the iteration count of Sinkhorn's device-side stopping test.

The oracle is oracle/sinkhorn_oracle.py, pure numpy and pinned bit for bit to the reference by the fixtures
tests/golden/sinkhorn_ref.npz (d = 3) and tests/golden/sinkhorn_wide_ref.npz (d = 8 .. 130), both written by
oracle/make_golden_sinkhorn.py from the reference's own file.

What is exact and what is bounded:
- pairwise_distances for p = 2, 1, inf, -inf and 0 equals numpy bit for bit, NaN where numpy gives NaN.
- pairwise_distances for other p is within _general_p_ulps(d, p, dtype) ulp of numpy (derived there: numpy calls
  pow in the array's precision, the kernel in fp64).
- The Sinkhorn plan is within 1e-9 of its largest entry in float64 and within _plan_rel_f32 (derived there)
  entry by entry in float32; the iteration count equals the reference's."""
import math

import numpy as np
import pytest

from conftest import load_golden

D_EXACT = (1, 2, 3, 7, 8, 9, 15, 16, 17, 64, 127, 128, 129, 130, 257, 1000)
M_TAILS = (1, 255, 256, 257, 1000)
EXACT_P = (2, 1, np.inf, -np.inf, 0)
DTYPES = (np.float32, np.float64)


def _dtype_id(dt):
    return np.dtype(dt).name


# ---- numpy's summation order -------------------------------------------------------------------------------------

def _np_sum(t):
    """add.reduce over the last axis in numpy's pairwise order: below 8 terms a sequential sum from 0; up to 128
    terms eight strided partial sums combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest one by one;
    above 128 terms split at n/2 - (n/2) % 8 and recurse."""
    n = t.shape[-1]
    if n < 8:
        s = np.zeros(t.shape[:-1], t.dtype)
        for c in range(n):
            s = s + t[..., c]
        return s
    if n <= 128:
        r = [t[..., k].copy() for k in range(8)]
        c = 8
        while c < n - n % 8:
            for k in range(8):
                r[k] = r[k] + t[..., c + k]
            c += 8
        s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for c in range(c, n):
            s = s + t[..., c]
        return s
    h = n // 2 - (n // 2) % 8
    return _np_sum(t[..., :h]) + _np_sum(t[..., h:])


def _sum_depth(n):
    """Most roundings any one term goes through in _np_sum's order (each addition rounds once)."""
    if n < 8:
        return n
    if n <= 128:
        return (n // 8 - 1) + 3 + n % 8
    h = n // 2 - (n // 2) % 8
    return 1 + max(_sum_depth(h), _sum_depth(n - h))


@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_pairwise_summation_order_is_numpys(dtype):
    """The order the kernel follows (np_pairwise_sum in sinkhorn.cuh) is the one np.linalg.norm uses, bit for bit.
    A sequential sum differs from it for d >= 8; fails loudly if a future numpy changes its order."""
    rng = np.random.default_rng(11)
    for d in (3, 8, 9, 15, 16, 17, 33, 127, 128, 129, 130, 300, 1000):
        x = (rng.standard_normal((300, d)) * rng.random((300, 1)) * 10).astype(dtype)
        assert np.array_equal(np.sqrt(_np_sum(x * x)), np.linalg.norm(x, axis=-1, ord=2)), d
        assert np.array_equal(_np_sum(np.abs(x)), np.linalg.norm(x, axis=-1, ord=1)), d
        if d >= 8:      # the order matters there: a plain running sum is not numpy's
            seq = np.cumsum(np.abs(x), axis=-1)[..., -1]
            assert not np.array_equal(seq, np.linalg.norm(x, axis=-1, ord=1)), d


def test_restatement_matches_the_wide_reference():
    """The oracle reproduces the reference's own results for d = 8 .. 130 bit for bit."""
    from oracle import sinkhorn_oracle as S
    g = load_golden("sinkhorn_wide_ref")
    for tag in (str(c) for c in g["cases"]):
        a, b = g[tag + "_a"], g[tag + "_b"]
        for p, key in ((2, "2"), (1, "1"), (np.inf, "inf"), (-np.inf, "neginf"), (0, "0"), (3, "3")):
            M = S.pairwise_distances(a, b, p)
            assert M.dtype == a.dtype and np.array_equal(M, g[tag + "_M_p" + key]), (tag, p)
        P = S.sinkhorn(g[tag + "_wa"], g[tag + "_wb"], g[tag + "_M_p2"], float(g[tag + "_eps"]))
        assert P.shape == g[tag + "_P"].shape and np.array_equal(P, g[tag + "_P"]), tag
    emd, P = S.earth_movers_distance(g["emd_p"], g["emd_q"], eps=float(g["emd_eps"]))
    assert emd == float(g["emd_value"]) and np.array_equal(P, g["emd_P"])


# ---- error bounds ------------------------------------------------------------------------------------------------

def _general_p_ulps(d, p, dtype):
    """Bound, in ulp of numpy's result, on |kernel - numpy| for a general p over d coordinates.

    Both sides form the same |x| and sum the terms t = |x|^p in the same order (depth h = _sum_depth(d)); they
    differ in how each pow is evaluated.  Relative to the exact values, with u the unit roundoff (2^-24, 2^-53):
    - terms: numpy calls libm pow in the array's precision (glibc: < 1 ulp, i.e. 2u); the kernel calls CUDA's fp64
      pow (2 ulp of fp64) and rounds to the dtype, i.e. u in float32 (the fp64 error is below 2^-50 u) and 4u in
      float64.  So tau = 3u (float32) or 6u (float64) between the two.
    - the sums: h roundings each, of non-negative terms, so each sum is within h u of its exact value: 2 h u apart.
    - the result S^q, q = 1 / p rounded to the dtype on both sides, scales a relative error of S by |q|, and adds
      the two final pows (numpy 2u, kernel u in float32; 2u and 4u in float64): phi = 3u or 6u.
    A relative difference r is at most r / u ulp of the result.  One ulp more absorbs the second-order terms."""
    q = abs(float(dtype(1) / dtype(p)))
    tau = phi = 3 if dtype == np.float32 else 6
    return math.ceil(q * (tau + 2 * _sum_depth(d)) + phi) + 1


def _assert_within_ulps(got, ref, ulps):
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)])
    err = np.abs(got[fin] - ref[fin])
    lim = ulps * np.spacing(np.abs(ref[fin]))
    assert (err <= lim).all(), float((err / np.spacing(np.abs(ref[fin]))).max())


# ---- pairwise_distances ------------------------------------------------------------------------------------------

def _clouds(rng, shape_a, shape_b, dtype):
    scale = 10.0 ** rng.integers(-3, 4)          # differences over several binades of exponent
    return ((rng.standard_normal(shape_a) * scale).astype(dtype), (rng.standard_normal(shape_b) * scale).astype(dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("p", EXACT_P, ids=lambda p: "p%s" % p)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_pairwise_exact_norms(pcu, dtype, p):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(21)
    for d in D_EXACT:
        for m in M_TAILS:
            for shape_a, shape_b in (((5, d), (m, d)), ((2, 3, d), (2, m, d))):
                a, b = _clouds(rng, shape_a, shape_b, dtype)
                got, ref = pcu.pairwise_distances(a, b, p), S.pairwise_distances(a, b, p)
                assert got.dtype == ref.dtype and got.shape == ref.shape, (d, m, shape_a)
                assert np.array_equal(got, ref), (d, m, shape_a, int((got != ref).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("p", (3, 0.5, -2), ids=lambda p: "p%s" % p)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_pairwise_general_p(pcu, dtype, p):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(22)
    for d in (1, 3, 8, 17, 128, 129, 257, 1000):
        for shape_a, shape_b in (((5, d), (257, d)), ((2, 3, d), (2, 40, d))):
            a, b = _clouds(rng, shape_a, shape_b, dtype)
            _assert_within_ulps(pcu.pairwise_distances(a, b, p), S.pairwise_distances(a, b, p), _general_p_ulps(d, p, dtype))


def _with_non_finite(rng, dtype, d):
    """Two batches; chosen rows of both clouds carry NaN, +inf or -inf in some coordinates, including rows where
    the same coordinate is inf in both (inf - inf = NaN) and an inf that meets a NaN."""
    a = rng.standard_normal((2, 7, d)).astype(dtype)
    b = rng.standard_normal((2, 6, d)).astype(dtype)
    a[0, 1, 0] = np.nan
    a[0, 2, d - 1] = np.inf
    a[0, 3, d // 2] = -np.inf
    a[1, 4, 0] = np.inf
    a[1, 4, d - 1] = -np.inf
    a[1, 5, :] = np.nan
    b[0, 1, d - 1] = np.inf              # meets a[0, 2]: inf - inf
    b[0, 2, d // 2] = np.nan
    b[1, 0, 0] = np.inf                  # meets a[1, 4]: inf - inf; others: -inf
    b[1, 3, d - 1] = -np.inf
    a[1, 6] = b[1, 2]                    # an all-zero difference
    return a, b


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_pairwise_non_finite_coordinates(pcu, dtype):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(23)
    for d in (3, 9, 130):
        a, b = _with_non_finite(rng, dtype, d)
        for p in EXACT_P:
            ref = S.pairwise_distances(a, b, p)
            got = pcu.pairwise_distances(a, b, p)
            assert np.array_equal(got, ref, equal_nan=True), (d, p)
            num = ~np.isnan(ref)        # the sign of a NaN is not part of the result; that of a zero is
            assert np.array_equal(np.signbit(got[num]), np.signbit(ref[num])), (d, p)
        for p in (3, 0.5, -2):
            _assert_within_ulps(pcu.pairwise_distances(a, b, p), S.pairwise_distances(a, b, p), _general_p_ulps(d, p, dtype))
    # the inf norms do not skip a NaN (numpy's max / min propagate it)
    row = np.array([[1.0, np.nan, 2.0]], dtype)
    zero = np.zeros((1, 3), dtype)
    assert np.isnan(pcu.pairwise_distances(row, zero, np.inf)) and np.isnan(pcu.pairwise_distances(row, zero, -np.inf))


@pytest.mark.gpu
def test_pairwise_more_than_65535_rows_and_batches(pcu):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(24)
    a, b = rng.random((70000, 3)), rng.random((4, 3))
    for p in (2, 1):
        assert np.array_equal(pcu.pairwise_distances(a, b, p), S.pairwise_distances(a, b, p))
    a, b = rng.random((70000, 2, 3)).astype(np.float32), rng.random((70000, 2, 3)).astype(np.float32)
    got = pcu.pairwise_distances(a, b)
    assert got.shape == (70000, 2, 2) and np.array_equal(got, S.pairwise_distances(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_pairwise_cuda_inputs_give_the_same_bits(pcu, dtype):
    import torch
    rng = np.random.default_rng(25)
    a, b = _clouds(rng, (2, 40, 33), (2, 300, 33), dtype)
    for p in (None, 1, 3):
        want = pcu.pairwise_distances(a, b, p)
        got = pcu.pairwise_distances(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), p)
        assert got.is_cuda and np.array_equal(got.cpu().numpy(), want), p


# ---- sinkhorn and earth_movers_distance --------------------------------------------------------------------------

def _problem(rng, nb, n, m, dtype, d=3):
    """Random points in the unit cube, their 2-norm costs and random positive weights summing to 1."""
    from oracle import sinkhorn_oracle as S
    shape = (lambda k: (k, d)) if nb == 0 else (lambda k: (nb, k, d))
    M = S.pairwise_distances(rng.random(shape(n)).astype(dtype), rng.random(shape(m)).astype(dtype))
    M = M.reshape((n, m) if nb == 0 else (nb, n, m))     # the oracle squeezes a 1-row or 1-column result
    wa = rng.random((n,) if nb == 0 else (nb, n)).astype(dtype) + dtype(0.5)
    wb = rng.random((m,) if nb == 0 else (nb, m)).astype(dtype) + dtype(0.5)
    return wa / wa.sum(-1, keepdims=True), wb / wb.sum(-1, keepdims=True), M


def _plan_rel_f32(iters, eps, M, wa, wb):
    """Bound on |P_kernel - P_numpy| / P_numpy for float32 after `iters` iterations, both runs on the same inputs.

    One half-iteration sets pot = eps * (log w - lse((-M + pot_in) / eps)).  log-sum-exp is 1-Lipschitz in the max
    norm, so a difference of the incoming potentials passes through unchanged, and each half-iteration adds its own
    rounding difference: the two reductions (numpy sums h = _sum_depth(C) terms in float32, h u; the kernel in fp64,
    rounded once, u), the log, exp and the element-wise steps (a few u, on terms of size up to B / eps with B the
    size of the potentials), times eps.  Per half-iteration at most eps (h + 3) u + 3 u B; after 2 * iters of them
    the potentials differ by at most 2 iters times that.  The plan exp((-M + u + v) / eps) turns an absolute
    difference of u + v into that difference / eps, relative, plus the rounding of its own three operations and
    exp: 4u on each side.  B bounds |u| and |v|: the first u lies in eps log a + [min M - eps log m, min M] and the
    iteration keeps the potentials within max M + eps |log w| + eps log(n m) of zero; twice that is taken."""
    u = 2.0 ** -24
    h = _sum_depth(max(M.shape[-1], M.shape[-2]))
    B = 2 * (np.abs(M).max() + eps * (abs(np.log(min(wa.min(), wb.min()))) + np.log(M.shape[-1] * M.shape[-2])))
    per_half = eps * (h + 3) * u + 3 * u * B
    return 2 * (2 * iters * per_half) / eps + 8 * u


def _sinkhorn_iters(pcu, wa, wb, M, eps, max_iters, stop_thresh):
    """The plan and the iteration count the device ran, read through the out_iters argument."""
    import torch
    from pcu_b200 import _pcu_internal
    ta, tb, tM = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (wa, wb, M))
    if tM.dim() == 2:
        ta, tb, tM = ta[None], tb[None], tM[None]
    nb, n, m = tM.shape
    P = torch.empty_like(tM)
    iters = torch.full((1,), -1, dtype=torch.int32, device=tM.device)
    _pcu_internal._sinkhorn_device(tM.dtype == torch.float64, ta.data_ptr(), tb.data_ptr(), tM.data_ptr(), nb, n, m,
                                   float(eps), int(max_iters), float(stop_thresh), P.data_ptr(), 0, iters.data_ptr(),
                                   tM.device.index or 0, torch.cuda.current_stream(tM.device).cuda_stream)
    torch.cuda.synchronize()
    return P.cpu().numpy().reshape(np.shape(M)), int(iters.item())


def _oracle_loop(wa, wb, M, eps, max_iters, stop_thresh):
    """The oracle's Sinkhorn loop (oracle/sinkhorn_oracle.py: the same numpy operations) on a 3-D problem without its
    np.squeeze, so one-row and one-column problems, which the reference's squeeze rejects, can be checked too.
    Returns the (nb, n, m) plan, the iteration count and, after each iteration, the L1 changes of u and of v per
    batch; the loop stops when the largest of each is below stop_thresh.  test_oracle_loop_is_the_oracle pins it to sinkhorn_oracle.sinkhorn."""
    from oracle import sinkhorn_oracle as S
    M3, a, b = (M if M.ndim == 3 else M[None]), np.atleast_2d(wa), np.atleast_2d(wb)
    u, v, errs = np.zeros_like(a), np.zeros_like(b), []
    for _ in range(max_iters):
        u0, v0 = u, v
        u = eps * (np.log(a) - S._lse((-M3 + np.expand_dims(v, 1)) / eps))
        v = eps * (np.log(b) - S._lse((-np.transpose(M3, (0, 2, 1)) + np.expand_dims(u, 1)) / eps))
        errs.append((np.sum(np.abs(u0 - u), axis=1), np.sum(np.abs(v0 - v), axis=1)))
        if errs[-1][0].max() < stop_thresh and errs[-1][1].max() < stop_thresh:
            break
    return np.exp((-M3 + np.expand_dims(u, 2) + np.expand_dims(v, 1)) / eps), len(errs), errs


def _iteration_errors(wa, wb, M, eps, max_iters):
    """The per-batch changes after each of max_iters iterations (none stops the loop)."""
    return _oracle_loop(wa, wb, M, eps, max_iters, -np.inf)[2]


@pytest.mark.parametrize("zero", (None, "a", "b"))
def test_oracle_loop_is_the_oracle(zero):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(61)
    for nb in (0, 3):
        wa, wb, M = _problem(rng, nb, 12, 9, np.float64)
        if zero is not None:
            (wa if zero == "a" else wb)[..., 4] = 0.0
        for stop in (0.0, 1e-3):
            ref, want = S.sinkhorn(wa, wb, M, 0.3, max_iters=40, stop_thresh=stop, return_iters=True)
            P, got, _ = _oracle_loop(wa, wb, M, 0.3, 40, stop)
            assert got == want and np.array_equal(P.reshape(ref.shape), ref), (nb, stop)


def _assert_plan_f64(P, ref, tag):
    assert P.dtype == ref.dtype and P.shape == ref.shape, tag
    assert np.abs(P - ref).max() <= 1e-9 * np.abs(ref).max(), (tag, float(np.abs(P - ref).max() / np.abs(ref).max()))


def _assert_column_marginals(P, wb):
    P3 = P if P.ndim == 3 else P.reshape((1,) + np.shape(P)[-2:])
    assert np.abs(P3.sum(1) - np.reshape(wb, (P3.shape[0], -1))).sum(1).max() < 1e-2


# (nb, n, m, max_iters).  nb = 0 is a 2-D problem.  The 2048 x 2048 float64 case is the largest oracle run of this
# file (20 iterations: a few seconds of numpy).
SINKHORN_SHAPES = ((0, 1, 7, 100), (0, 7, 1, 100), (0, 33, 257, 100), (0, 300, 1000, 50), (0, 1000, 300, 50),
                   (0, 2048, 2048, 20), (1, 33, 257, 100), (3, 33, 40, 100), (300, 9, 12, 100))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
@pytest.mark.parametrize("nb,n,m,max_iters", SINKHORN_SHAPES, ids=lambda v: str(v))
def test_sinkhorn_shapes(pcu, nb, n, m, max_iters, dtype):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(31 + n + m + nb)
    wa, wb, M = _problem(rng, nb, n, m, dtype)
    eps = 0.05
    # stop_thresh = 0: both sides run all max_iters, so the bound below counts the same iterations on each
    if min(n, m) == 1:
        # np.squeeze leaves a 1-D M, which the reference rejects, and so does sinkhorn(); the device entry takes it
        for f in (pcu.sinkhorn, S.sinkhorn):
            with pytest.raises(ValueError):
                f(wa, wb, M, eps)
        P, _ = _sinkhorn_iters(pcu, wa, wb, M, eps, max_iters, 0.0)
        ref = _oracle_loop(wa, wb, M, eps, max_iters, 0.0)[0].reshape(M.shape)
    else:
        P = pcu.sinkhorn(wa, wb, M, eps, max_iters=max_iters, stop_thresh=0.0)
        ref = S.sinkhorn(wa, wb, M, eps, max_iters=max_iters, stop_thresh=0.0)
    assert P.dtype == ref.dtype and P.shape == ref.shape
    if dtype == np.float64:
        _assert_plan_f64(P, ref, (nb, n, m))
    else:
        rel = _plan_rel_f32(max_iters, eps, M, wa, wb)
        tiny = np.finfo(np.float32).smallest_subnormal
        assert (np.abs(P.astype(np.float64) - ref) <= rel * ref.astype(np.float64) + 2 * tiny).all(), \
            float((np.abs(P.astype(np.float64) - ref) / np.maximum(ref, tiny)).max())
    _assert_column_marginals(P, wb)


def _assert_margins(errs, count, stop_thresh):
    """Every iteration run either passed the test by a factor of 2 (only the last may) or failed it by a factor of 2:
    the device's fp64 atomics sum in no fixed order, so a case near stop_thresh would be a bad case, not a flake."""
    for k, (eu, ev) in enumerate(errs[:count]):
        e = max(eu.max(), ev.max())
        if k == count - 1 and e < stop_thresh:
            assert e < stop_thresh / 2, (k, e, stop_thresh)
        else:
            assert e > 2 * stop_thresh or not np.isfinite(e) or stop_thresh == 0, (k, e, stop_thresh)


@pytest.mark.gpu
@pytest.mark.parametrize("max_iters", (0, 1, 5, 100))
@pytest.mark.parametrize("stop_thresh", (0.0, 1e-3, 1e9))
def test_sinkhorn_iteration_count(pcu, max_iters, stop_thresh):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(41)
    wa, wb, M = _problem(rng, 0, 30, 45, np.float64)
    eps = 0.34                          # stops after 6 iterations, clear of stop_thresh on both sides
    ref, want = S.sinkhorn(wa, wb, M, eps, max_iters=max_iters, stop_thresh=stop_thresh, return_iters=True)
    _assert_margins(_iteration_errors(wa, wb, M, eps, max_iters), want, stop_thresh)
    if stop_thresh == 1e-3 and max_iters == 100:
        assert 5 < want < 100           # the case stops early, on the test
    P, got = _sinkhorn_iters(pcu, wa, wb, M, eps, max_iters, stop_thresh)
    assert got == want
    _assert_plan_f64(P, ref, (max_iters, stop_thresh))


@pytest.mark.gpu
def test_sinkhorn_iteration_count_when_one_batch_converges_first(pcu):
    """Batch 0 has a constant cost (its potentials settle after one iteration); batches 1 and 2 take many more.  The
    stopping test takes the largest change over the batch, so the count is the slow batches'."""
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(42)
    wa, wb, M = _problem(rng, 3, 20, 25, np.float64)
    M[0] = 0.7
    eps = 0.34                          # stops after 7 iterations, clear of stop_thresh on both sides
    ref, want = S.sinkhorn(wa, wb, M, eps, max_iters=100, stop_thresh=1e-3, return_iters=True)
    errs = _iteration_errors(wa, wb, M, eps, 100)
    _assert_margins(errs, want, 1e-3)
    first = _iteration_errors(wa[:1], wb[:1], M[:1], eps, 100)
    assert max(e.max() for e in first[2]) < 1e-3 / 2 and want > 5
    P, got = _sinkhorn_iters(pcu, wa, wb, M, eps, 100, 1e-3)
    assert got == want
    _assert_plan_f64(P, ref, "one batch first")


@pytest.mark.gpu
@pytest.mark.parametrize("where", ("a", "b"))
@pytest.mark.parametrize("nb", (0, 3))
def test_sinkhorn_zero_weights(pcu, where, nb):
    """A zero weight makes its potential -inf; from the second iteration on its change is -inf - -inf = NaN, which
    never counts as converged (numpy: NaN < stop_thresh is false), so all max_iters run.  The plan has a zero row
    (weight of a) or column (weight of b) there."""
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(51)
    wa, wb, M = _problem(rng, nb, 40, 50, np.float64)
    w = wa if where == "a" else wb
    w[(7,) if nb == 0 else (1, 7)] = 0.0
    w /= w.sum(-1, keepdims=True)       # balanced again: the other changes settle, only the NaN keeps the loop going
    eps = 0.34
    ref, want = S.sinkhorn(wa, wb, M, eps, max_iters=100, stop_thresh=1e-3, return_iters=True)
    assert want == 100
    # a maximum that skipped the NaN would have stopped well inside max_iters
    skip_nan = [np.nanmax(np.concatenate(it)) for it in _iteration_errors(wa, wb, M, eps, 100)]
    assert min(k for k, e in enumerate(skip_nan) if e < 1e-3 / 2) < 50
    P, got = _sinkhorn_iters(pcu, wa, wb, M, eps, 100, 1e-3)
    assert got == want
    zero = ref == 0
    assert zero.any() and np.array_equal(P == 0, zero)
    _assert_plan_f64(P, ref, (where, nb))
    assert np.array_equal(pcu.sinkhorn(wa, wb, M, eps), P)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dtype_id)
def test_sinkhorn_infinite_costs(pcu, dtype):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(52)
    wa, wb, M = _problem(rng, 2, 30, 40, dtype)
    mask = rng.random(M.shape) < 0.3
    mask[:, :, 0] = False                # every row and column keeps a finite cost
    mask[:, 0, :] = False
    M[mask] = np.inf
    eps, iters = 0.05, 100
    P = pcu.sinkhorn(wa, wb, M, eps, max_iters=iters, stop_thresh=0.0)
    ref = S.sinkhorn(wa, wb, M, eps, max_iters=iters, stop_thresh=0.0)
    assert (P[mask] == 0).all() and (ref[mask] == 0).all()
    if dtype == np.float64:
        _assert_plan_f64(P, ref, "inf costs")
    else:
        Mf = np.where(mask, 0, M)        # B of the bound counts the finite costs
        rel = _plan_rel_f32(iters, eps, Mf, wa, wb)
        assert (np.abs(P.astype(np.float64) - ref) <= rel * ref + 2 * np.finfo(np.float32).smallest_subnormal).all()


@pytest.mark.gpu
def test_sinkhorn_more_than_65535_rows_and_batches(pcu):
    from oracle import sinkhorn_oracle as S
    rng = np.random.default_rng(53)
    for nb, n, m in ((0, 70000, 4), (70000, 2, 3)):
        wa, wb, M = _problem(rng, nb, n, m, np.float64)
        P = pcu.sinkhorn(wa, wb, M, 0.1, max_iters=10, stop_thresh=0.0)
        _assert_plan_f64(P, S.sinkhorn(wa, wb, M, 0.1, max_iters=10, stop_thresh=0.0), (nb, n, m))


@pytest.mark.gpu
def test_earth_movers_distance_16d(pcu):
    import torch
    from oracle import sinkhorn_oracle as S
    g = load_golden("sinkhorn_wide_ref")
    p, q, eps = g["emd_p"], g["emd_q"], float(g["emd_eps"])
    ref, ref_P = S.earth_movers_distance(p, q, eps=eps)
    assert ref == float(g["emd_value"])
    emd, P = pcu.earth_movers_distance(p, q, eps=eps)
    assert abs(float(emd) - ref) <= 1e-9 * ref
    _assert_plan_f64(P, ref_P, "emd")
    emd_t, P_t = pcu.earth_movers_distance(torch.from_numpy(p).cuda(), torch.from_numpy(q).cuda(), eps=eps)
    assert emd_t.is_cuda and abs(float(emd_t) - ref) <= 1e-9 * ref
    assert np.array_equal(P_t.cpu().numpy(), P)


@pytest.mark.gpu
def test_kernels_match_the_wide_reference_goldens(pcu):
    g = load_golden("sinkhorn_wide_ref")
    for tag in (str(c) for c in g["cases"]):
        a, b = g[tag + "_a"], g[tag + "_b"]
        for p, key in ((2, "2"), (1, "1"), (np.inf, "inf"), (-np.inf, "neginf"), (0, "0")):
            assert np.array_equal(pcu.pairwise_distances(a, b, p), g[tag + "_M_p" + key]), (tag, p)
        d = a.shape[-1]
        _assert_within_ulps(pcu.pairwise_distances(a, b, 3), g[tag + "_M_p3"], _general_p_ulps(d, 3, a.dtype.type))
        if a.dtype == np.float64:
            P = pcu.sinkhorn(g[tag + "_wa"], g[tag + "_wb"], g[tag + "_M_p2"], float(g[tag + "_eps"]))
            _assert_plan_f64(P, g[tag + "_P"], tag)
