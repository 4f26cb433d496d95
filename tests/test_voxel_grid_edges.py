"""Voxel-grid down-sampling at the inputs where its kernels go wrong (SURVEY.md 8f, N2; the reference:
point_cloud_utils/__init__.py:123-200, src/sample_point_cloud.cpp:163-244 and :336-367).

Integer part, exact.  `oracle.voxel_indices` restates the reference's index arithmetic, including its conversion of a
quotient that does not fit an int (outside [-2^31, 2^31), +-inf, NaN: INT_MIN, as x86-64 converts).  Against it: the
number of rows, the point count of every row and the row order -- rows come in the order of each voxel's first point.
The order is pinned through the means: row r must hold the mean of the r-th voxel.

Means, against the exact mean of each voxel's members.  The exact sum of a voxel is formed here without rounding loss
(error-free TwoSum for small voxels, math.fsum plus its residual for large ones) and divided with a correction step,
so E, the value the outputs are compared with, is the exact mean rounded to fp64 (to within a hair over 1/2 ulp).
For a voxel of m < 2^20 points and u = 2^-53:
* The kernel sums the m values in fp64 in whatever order its atomics land: the sum is within (m - 1) u sum|x| (1 + mu)
  of the exact one, and the division by m adds u |mean|.  So the fp64 mean q is within m u mean|x| (1 + mu) of the
  exact mean.
* float64 outputs are q: |got - E| <= (m + 1) u mean|x| + 1/2 ulp_f64(E); the extra u mean|x| covers the (1 + mu)
  factor, the 1/2 ulp the rounding of E.
* float32 outputs (float32 clouds, float32 attributes; their members are float32 values) are q rounded once to float32.
  Where the members of a column share one sign, mean|x| = |mean| and |q - mean| <= (m + 1) u |mean| < 2^-32 |mean|,
  far below ulp_f32(mean) >= 2^-24 |mean|; the rounding to float32 adds 1/2 ulp_f32:
  |got - E| <= 1 ulp_f32(E).  Where they have both signs, the fp64 cancellation term (m + 1) u mean|x| is added.
A float32 accumulator, a point dropped or counted twice, or a point filed under the wrong voxel misses these bounds by
orders of magnitude: `test_means_against_the_exact_mean` holds a voxel of 1.0 and thousands of values between 2^-40 and
2^-11, whose float32 running sum loses about 4e-6 of the total, dozens of float32 ulps.
A column that holds +-inf or NaN has the mean np.sum gives (inf, or NaN) -- the same in any summation order.

fp64 atomics make a float64 mean depend, in its last bit, on the order they land in, so no test here compares two
calls bit for bit."""
import math

import numpy as np
import pytest

INT_MIN = -2 ** 31
U = 2.0 ** -53
DTYPE_PAIRS = [(np.float32, np.float32), (np.float32, np.float64), (np.float64, np.float32), (np.float64, np.float64)]


def _mod():
    from importlib import import_module
    return import_module("point-cloud-utils_b200")


# ---- the reference side ---------------------------------------------------------------------------------------------
def _groups(oracle, points, vs, lo):
    """Voxel of every point as a row number (voxels in the order of their first point) and the count of every voxel."""
    idx = oracle.voxel_indices(points, vs, lo)
    _, first, inverse, counts = np.unique(idx, axis=0, return_index=True, return_inverse=True, return_counts=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return rank[inverse.reshape(-1)], counts[order]


def _two_prod(a, b):
    """a * b = p + e exactly (Dekker's product; |a|, |b| far from overflow)."""
    p = a * b
    def split(v):
        t = 134217729.0 * v                  # 2^27 + 1
        h = t - (t - v)
        return h, v - h
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _exact_means(x, group, counts):
    """x (n, c) float64.  Per voxel and column: E (exact mean rounded to fp64), mean|x|, members of both signs,
    all members finite.  Columns with a non-finite member get np.sum's mean instead of E."""
    g, c = len(counts), x.shape[1]
    order = np.argsort(group, kind="stable")
    xs = x[order]
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    m = counts.astype(np.float64)[:, None]
    with np.errstate(invalid="ignore"):
        plain = np.add.reduceat(xs, starts, axis=0)
    finite = np.logical_and.reduceat(np.isfinite(xs), starts, axis=0)
    mean_abs = np.add.reduceat(np.where(np.isfinite(xs), np.abs(xs), 0.0), starts, axis=0) / m
    mixed = (np.minimum.reduceat(xs, starts, axis=0) < 0) & (np.maximum.reduceat(xs, starts, axis=0) > 0)
    xf = np.where(np.isfinite(xs), xs, 0.0)
    hi, lo = np.zeros((g, c)), np.zeros((g, c))
    small = counts <= 64
    for k in range(int(min(64, counts.max()))):        # TwoSum over the k-th member of every small voxel at once
        rows = np.nonzero(small & (counts > k))[0]
        a, b = hi[rows], xf[starts[rows] + k]
        s = a + b
        bb = s - a
        hi[rows], lo[rows] = s, lo[rows] + ((a - (s - bb)) + (b - bb))
    for r in np.nonzero(~small)[0]:                       # large voxels: fsum, and fsum of what it left over
        seg = xf[starts[r]:starts[r] + counts[r]]
        for j in range(c):
            col = seg[:, j].tolist()
            hi[r, j] = math.fsum(col)
            lo[r, j] = math.fsum(col + [-hi[r, j]])
    q = hi / m                                            # (hi + lo) / m, with one correction step
    p, e = _two_prod(q, m)
    exact = q + (((hi - p) - e) + lo) / m
    exact = np.where(finite, exact, plain / m)
    return exact, mean_abs, mixed, finite


def _ulp32(e):
    """ulp of the largest float32 <= |e|."""
    a = np.abs(e)
    f = a.astype(np.float32)
    f = np.where(f.astype(np.float64) > a, np.nextafter(f, np.float32(0)), f)
    return np.spacing(f).astype(np.float64)


def _check_means(got, x, group, counts, keep, what):
    got = np.asarray(got)
    exact, mean_abs, mixed, finite = (a[keep] for a in _exact_means(x.reshape(len(x), -1).astype(np.float64), group, counts))
    m = counts[keep].astype(np.float64)[:, None]
    g = got.reshape(len(got), int(np.prod(got.shape[1:]))).astype(np.float64)
    assert g.shape == exact.shape, what
    if got.dtype == np.float32:
        bound = _ulp32(exact) + np.where(mixed, (m + 1) * U * mean_abs, 0.0)
    else:
        bound = (m + 1) * U * mean_abs + 0.5 * np.spacing(np.abs(exact))
    err = np.where(finite, np.abs(g - exact), 0.0)
    bad = np.nonzero(err > bound)
    assert bad[0].size == 0, "%s: %d means off, e.g. row %d col %d: got %r exact %r bound %r count %d" % (
        what, bad[0].size, bad[0][0], bad[1][0], g[bad][0], exact[bad][0], bound[bad][0], m[bad[0][0], 0])
    assert np.array_equal(g[~finite], exact[~finite], equal_nan=True), what


# ---- one call, checked --------------------------------------------------------------------------------------------
def _numpy(a):
    return a if isinstance(a, np.ndarray) else a.detach().cpu().numpy()


def _check(pcu, oracle, points, attrs=(), size=0.1, min_bound=None, max_bound=None, min_pts=1):
    """Down-sample through the public function, fetch the per-row counts, and hold both to the oracle: the integer
    part exactly, every mean within the bounds of the module docstring.  Returns (voxel of every point, counts)."""
    tensor = not isinstance(points, np.ndarray)
    pts = _numpy(points)
    vs = np.array([size] * 3, dtype=np.float64) if np.isscalar(size) else np.array(size, dtype=np.float64)
    lo = pts.min(axis=0) - vs * 0.5 if min_bound is None else np.array(min_bound, dtype=np.float64)
    hi = pts.max(axis=0) + vs * 0.5 if max_bound is None else np.array(max_bound, dtype=np.float64)
    out = pcu.downsample_point_cloud_on_voxel_grid(size, points, *attrs, min_bound=min_bound, max_bound=max_bound,
                                                   min_points_per_voxel=min_pts)
    out = out if isinstance(out, tuple) else (out,)
    assert len(out) == 1 + len(attrs)
    counts_arg = (np.zeros([0, 0]) if not tensor else None)
    _, _, got_counts = _mod()._voxel_internal(points, counts_arg, vs, lo, hi, min_pts, None, return_counts=True)
    group, counts = _groups(oracle, pts, vs, lo)
    keep = counts >= min_pts
    rows = int(keep.sum())
    for o, a in zip(out, (points,) + tuple(attrs)):
        assert (not isinstance(o, np.ndarray)) == tensor and (not tensor or o.is_cuda)
        assert o.dtype == a.dtype and tuple(o.shape) == (rows,) + tuple(a.shape[1:]), (o.dtype, tuple(o.shape), rows)
    assert (not isinstance(got_counts, np.ndarray)) == tensor
    assert np.array_equal(_numpy(got_counts), counts[keep]), "counts / row order differ from the oracle"
    _check_means(_numpy(out[0]), pts, group, counts, keep, "points")
    for i, a in enumerate(attrs):
        _check_means(_numpy(out[1 + i]), _numpy(a), group, counts, keep, "attribute %d" % i)
    return group, counts


# ---- the conversion rule of the oracle (no GPU) -----------------------------------------------------------------------
def _special_quotients(dtype):
    """(quotient, index the reference gives it) around the ends of the int range, for a voxel size of 1 at 0."""
    if dtype == np.float32:                 # float32 neighbours of 2^31: 2^31 - 128 below, 2^31 + 256 above
        return [(0.5, 0), (2.0 ** 31 - 128, 2 ** 31 - 128), (2147483647.0, INT_MIN), (2.0 ** 31, INT_MIN),
                (2.0 ** 31 + 256, INT_MIN), (3e9, INT_MIN), (-(2.0 ** 31) + 128, -(2 ** 31) + 128),
                (-(2.0 ** 31), INT_MIN), (-(2.0 ** 31) - 256, INT_MIN), (-3e9, INT_MIN),
                (np.inf, INT_MIN), (-np.inf, INT_MIN), (np.nan, INT_MIN)]
    return [(0.5, 0), (2.0 ** 31 - 0.5, 2 ** 31 - 1), (2.0 ** 31, INT_MIN), (2.0 ** 31 + 0.5, INT_MIN), (3e9, INT_MIN),
            (-(2.0 ** 31) + 0.5, INT_MIN), (-(2.0 ** 31), INT_MIN), (-(2.0 ** 31) - 0.5, INT_MIN), (-3e9, INT_MIN),
            (np.inf, INT_MIN), (-np.inf, INT_MIN), (np.nan, INT_MIN)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_oracle_gives_int_min_where_the_quotient_does_not_fit(oracle, dtype):
    import warnings
    q, want = zip(*_special_quotients(dtype))
    x = np.array(q, dtype=dtype)
    for a in range(3):
        pts = np.full((len(x), 3), 0.25, dtype=dtype)
        pts[:, a] = x
        with warnings.catch_warnings():
            warnings.simplefilter("error")                  # explicit rule, no cast of invalid values
            idx = oracle.voxel_indices(pts, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0))
        assert idx.dtype == np.int32
        assert idx[:, a].tolist() == list(want)
        assert not idx[:, [b for b in range(3) if b != a]].any()
    # finite points outside explicit bounds: quotient 5e9 and -5e9 both land in INT_MIN, so they share a voxel
    pts = np.array([[0.5e-9, 0.5e-9, 0.5e-9], [5.0, 0.5e-9, 0.5e-9], [-5.0, 0.5e-9, 0.5e-9], [np.nan, 0.5e-9, 0.5e-9]], dtype)
    v, cnt = oracle.downsample_point_cloud_on_voxel_grid(1e-9, pts, min_bound=(0, 0, 0), max_bound=(1, 1, 1), return_counts=True)
    assert cnt.tolist() == [1, 3] and np.array_equal(v[0], pts[0]) and np.isnan(v[1, 0])


def test_oracle_default_bounds_with_non_finite_coordinates(oracle):
    rng = np.random.default_rng(5)
    p = rng.random((500, 3))
    for bad in (np.inf, -np.inf):
        q = p.copy()
        q[17, 1] = bad
        with pytest.raises(ValueError, match="too small"):
            oracle.downsample_point_cloud_on_voxel_grid(0.1, q)
    q = p.copy()
    q[17, 1] = np.nan                                       # the default bound of y is NaN: every y index is INT_MIN
    idx = oracle.voxel_indices(q, (0.1, 0.1, 0.1), np.min(q, axis=0) - 0.05)
    assert (idx[:, 1] == INT_MIN).all()
    _, cnt = oracle.downsample_point_cloud_on_voxel_grid(0.1, q, return_counts=True)
    assert len(cnt) == len(np.unique(idx[:, [0, 2]], axis=0))


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _binade_voxel(rng, dtype, k):
    """k - 1 values between 2^-40 and 2^-11 (random mantissas) and one 1.0 in the middle: a float32 running sum drops
    everything below 2^-24 of it."""
    v = (2.0 ** -rng.integers(12, 41, size=k) * (1.0 + rng.random(k))).astype(dtype)
    v[k // 2] = 1.0
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_means_against_the_exact_mean(pcu, oracle, dtype, adtype):
    rng = np.random.default_rng(31)
    k = 4096
    binade = np.stack([_binade_voxel(rng, dtype, k) for _ in range(3)], axis=1)       # the voxel [0, 2)^3
    bulk = (rng.random((60000, 3)) * 6.0 + 2.0).astype(dtype)                           # [2, 8)^3
    neg = (-rng.random((20000, 3)) * 8.0).astype(dtype)                                 # [-8, 0)^3, one sign per voxel
    pts = np.concatenate([binade, bulk, neg])
    n = len(pts)
    attr = np.empty((n, 3), dtype=adtype)
    attr[:, 0] = np.concatenate([_binade_voxel(rng, adtype, k), rng.random(n - k)])       # binades in one voxel again
    attr[:, 1] = rng.standard_normal(n)                                                   # both signs in every voxel
    attr[:, 2] = rng.random(n) * 1e3 + 1e6
    perm = rng.permutation(n)
    pts, attr = pts[perm], attr[perm]
    bounds = dict(min_bound=(-8.0, -8.0, -8.0), max_bound=(8.0, 8.0, 8.0))
    group, counts = _check(pcu, oracle, pts, (attr,), size=2.0, **bounds)
    assert counts.max() >= k
    _check(pcu, oracle, pts, (attr,), size=0.37, **bounds)                               # non-power-of-two size
    _check(pcu, oracle, pts, (attr[:, 0],), size=0.05)                                   # many small voxels


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 262143, 262144, 262145, 600000])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_integer_part_across_sizes(pcu, oracle, n, dtype):
    """Partial last blocks, one block, and 1023 / 1024 / 1025+ blocks of 256 rows (one or two scan rounds)."""
    rng = np.random.default_rng(n)
    pts = rng.random((n, 3)).astype(dtype)
    pts[-1] = 1.5                                          # the last row is a voxel of its own, so it is emitted
    a32 = rng.random((n, 2, 3)).astype(np.float32)
    a64 = rng.standard_normal(n)
    size = (3.0 / n) ** (1.0 / 3.0)                        # about 3 points per voxel
    _check(pcu, oracle, pts, (a32, a64), size=size)
    if n >= 256:
        _check(pcu, oracle, pts, (a64,), size=size, min_pts=3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_one_voxel_and_one_point_per_voxel(pcu, oracle, dtype, adtype):
    rng = np.random.default_rng(7)
    n = 262145
    pts = rng.random((n, 3)).astype(dtype) + 1.0
    attr = rng.random((n, 4)).astype(adtype)
    _, counts = _check(pcu, oracle, pts, (attr,), size=10.0)
    assert counts.tolist() == [n]
    lattice = np.stack(np.meshgrid(np.arange(73), np.arange(61), np.arange(59), indexing="ij"), -1).reshape(-1, 3)
    pts = (lattice[rng.permutation(len(lattice))] + 0.5).astype(dtype)                  # voxel centres, size 1
    attr = rng.random((len(pts), 4)).astype(adtype)
    _, counts = _check(pcu, oracle, pts, (attr,), size=1.0)
    assert len(counts) == len(pts) and (counts == 1).all()


def _voxel_hash(v):
    """voxel_hash of voxel.cuh on uint32."""
    u = v.astype(np.int64).astype(np.uint32)
    h = (u[:, 0] * np.uint32(73856093)) ^ (u[:, 1] * np.uint32(19349663)) ^ (u[:, 2] * np.uint32(83492791))
    h ^= h >> np.uint32(15)
    h *= np.uint32(0x2C1B3C6D)
    h ^= h >> np.uint32(12)
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("n,slots", [(32, 64), (128, 256)])
@pytest.mark.parametrize("dtype,adtype", [(np.float32, np.float64), (np.float64, np.float32)])
def test_probing_wraps_past_the_end_of_the_table(pcu, oracle, n, slots, dtype, adtype):
    """The table has 64 slots up to 32 points, 256 up to 128.  Voxels whose hash lands on the last slots and on the
    first ones make linear probing run past the end and start over at slot 0."""
    rng = np.random.default_rng(slots)
    cells = np.stack(np.meshgrid(*[np.arange(16)] * 3, indexing="ij"), -1).reshape(-1, 3)
    h = _voxel_hash(cells) % np.uint32(slots)
    chosen = np.concatenate([cells[h == slots - 1][:6], cells[h == slots - 2][:2], cells[h == 0][:3], cells[h == 1][:2]])
    per = n // len(chosen)
    pts = np.repeat(chosen, per, axis=0) + rng.choice([0.25, 0.5, 0.75], size=(per * len(chosen), 3))
    filler = cells[rng.choice(len(cells), n - len(pts), replace=False)] + 0.5              # the rest of the n points
    pts = np.concatenate([pts, filler])[rng.permutation(n)].astype(dtype)
    assert len(pts) == n
    attr = rng.standard_normal((n, 40)).astype(adtype)
    bounds = dict(min_bound=(0.0, 0.0, 0.0), max_bound=(16.0, 16.0, 16.0))
    _, counts = _check(pcu, oracle, pts, (attr,), size=1.0, **bounds)
    assert (counts >= per).sum() >= len(chosen)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_anisotropic_large_coordinates_and_faces(pcu, oracle, dtype, adtype):
    rng = np.random.default_rng(3)
    n = 100000
    pts = (rng.random((n, 3)) * [2.0, 1.0, 0.5] - 0.3).astype(dtype)
    attr = rng.random((n, 1)).astype(adtype)
    _check(pcu, oracle, pts, (attr,), size=(0.05, 0.3, 0.011))
    _check(pcu, oracle, pts, (attr,), size=(1e-3, 1.0, 10.0))
    # around 1e6 p - min_bound rounds (float32 spacing there is 1/16)
    far = (1e6 + rng.random((n, 3)) * [10.0, 3.0, 1.0]).astype(dtype)
    _check(pcu, oracle, far, (attr,), size=0.1)
    _check(pcu, oracle, far, (attr,), size=(0.25, 0.07, 0.5), min_bound=(999999.9, 1e6, 1e6 - 0.3), max_bound=(1e6 + 20, 1e6 + 5, 1e6 + 2))
    # points on voxel faces: p - min_bound an exact multiple of the size (quotient an integer), and k * 0.1, whose
    # quotient by 0.1 rounds to either side of k
    k = rng.integers(0, 40, size=(n, 3))
    faces = (k * 0.25).astype(dtype)
    _check(pcu, oracle, faces, (attr,), size=0.25, min_bound=(0.0, 0.0, 0.0), max_bound=(10.0, 10.0, 10.0))
    _check(pcu, oracle, faces + dtype(0.5), (attr,), size=(0.25, 0.5, 0.125), min_bound=(0.5, 0.5, 0.5), max_bound=(11.0, 11.0, 11.0))
    tenth = (k * dtype(0.1)).astype(dtype)
    _, counts = _check(pcu, oracle, tenth, (attr,), size=0.1, min_bound=(0.0, 0.0, 0.0), max_bound=(4.0, 4.0, 4.0))
    assert len(counts) >= 40 ** 3 // 2


@pytest.mark.gpu
@pytest.mark.parametrize("tensor", [False, True])
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_min_points_attribute_shapes_and_zero_rows(pcu, oracle, tensor, dtype, adtype):
    import torch
    rng = np.random.default_rng(9)
    n = 20000
    pts = rng.random((n, 3)).astype(dtype)
    attrs = [rng.random(n).astype(adtype), rng.random((n, 1)).astype(adtype), rng.standard_normal((n, 2, 3)).astype(adtype),
             rng.random((n, 40)).astype(adtype)]
    if tensor:
        pts, attrs = torch.from_numpy(pts).cuda(), [torch.from_numpy(a).cuda() for a in attrs]
    _, counts = _check(pcu, oracle, pts, attrs, size=0.07, min_pts=0)
    assert counts.max() >= 3
    _check(pcu, oracle, pts, attrs, size=0.07, min_pts=1)
    _check(pcu, oracle, pts, attrs, size=0.07, min_pts=int(np.median(counts)))
    _check(pcu, oracle, pts, attrs, size=0.07, min_pts=int(counts.max()) + 1)          # no rows at all
    out = pcu.downsample_point_cloud_on_voxel_grid(0.07, pts, *attrs, min_points_per_voxel=int(counts.max()) + 1)
    assert tuple(out[0].shape) == (0, 3)
    assert [tuple(o.shape) for o in out[1:]] == [(0,), (0, 1), (0, 2, 3), (0, 40)]
    alone = pcu.downsample_point_cloud_on_voxel_grid(0.07, pts, min_points_per_voxel=int(counts.max()) + 1)
    assert tuple(alone.shape) == (0, 3) and alone.dtype == pts.dtype


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_out_of_range_and_non_finite_coordinates(pcu, oracle, dtype, adtype):
    """Explicit bounds [0, 1)^3 with size 1 and points far outside them, on each axis: where the quotient does not fit
    an int the reference files the point under INT_MIN on that axis -- 2^31 and -2^31 - 1 alike, NaN too, which must
    not land in the occupied layer at index 0."""
    rng = np.random.default_rng(13)
    ordinary = rng.random((3000, 3)) * 4.0                                               # cells 0..3, index 0 included
    rows = [ordinary]
    for a in range(3):
        others = [b for b in range(3) if b != a]
        for q, want in _special_quotients(dtype):
            # finite values beside cell 0 / cell 1 of the other axes, inf with cell 2 and NaN with cell 3, so that the
            # finite out-of-range voxels keep finite means
            cell = 3 if np.isnan(q) else 2 if np.isinf(q) else rng.integers(0, 2)
            r = np.empty((5, 3))
            r[:, a] = q
            r[:, others] = cell + rng.random((5, 2))
            rows.append(r)
    pts = np.concatenate(rows)
    pts = pts[rng.permutation(len(pts))].astype(dtype)
    attr = rng.random((len(pts), 2)).astype(adtype)
    bounds = dict(min_bound=(0.0, 0.0, 0.0), max_bound=(1.0, 1.0, 1.0))
    group, counts = _check(pcu, oracle, pts, (attr,), size=1.0, **bounds)
    idx = oracle.voxel_indices(pts, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0))
    assert (idx[np.isnan(pts)] == INT_MIN).all() and (idx[np.isinf(pts)] == INT_MIN).all()
    # finite coordinates only, a tiny size: +-5 give quotients of +-5e9, one voxel in the reference
    tiny = (rng.random((2000, 3)) * 4e-9).astype(dtype)
    far = np.array([[5.0, 1e-9, 1e-9], [-5.0, 1e-9, 1e-9], [1e-9, 5.0, 1e-9], [1e-9, -3.0, 1e-9], [1e-9, 1e-9, 7.0]], dtype)
    pts = np.concatenate([tiny[:1000], far, tiny[1000:]])
    attr = rng.random((len(pts), 3)).astype(adtype)
    _, counts = _check(pcu, oracle, pts, (attr,), size=1e-9, **bounds)
    assert 2 in counts.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_default_bounds_with_non_finite_coordinates(pcu, oracle, dtype):
    rng = np.random.default_rng(17)
    p = rng.random((5000, 3)).astype(dtype)
    for a in range(3):
        for bad in (np.inf, -np.inf):
            q = p.copy()
            q[1234, a] = bad
            with pytest.raises(ValueError, match="too small"):
                pcu.downsample_point_cloud_on_voxel_grid(0.1, q)
            with pytest.raises(ValueError, match="too small"):
                oracle.downsample_point_cloud_on_voxel_grid(0.1, q)
        # NaN on one axis: that axis's default bounds are NaN, every point has index INT_MIN there, the other two
        # axes still split the cloud
        q = p.copy()
        q[1234, a] = np.nan
        attr = rng.random((len(q), 2)).astype(dtype)
        group, counts = _check(pcu, oracle, q, (attr,), size=0.1)
        lo = np.min(q, axis=0) - 0.05
        idx = oracle.voxel_indices(q, (0.1, 0.1, 0.1), lo)
        assert (idx[:, a] == INT_MIN).all()
        assert len(counts) == len(np.unique(idx[:, [b for b in range(3) if b != a]], axis=0)) > 1


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,adtype", DTYPE_PAIRS)
def test_tensor_numpy_and_offset_views_agree(pcu, oracle, dtype, adtype):
    import torch
    rng = np.random.default_rng(19)
    n = 70001
    pts = rng.random((n, 3)).astype(dtype)
    attr = rng.random((n, 5)).astype(adtype)
    _, c_np = _check(pcu, oracle, pts, (attr,), size=0.03)
    _, c_t = _check(pcu, oracle, torch.from_numpy(pts).cuda(), (torch.from_numpy(attr).cuda(),), size=0.03)
    # storage offsets of one element: 4 or 8 bytes past a 16-byte boundary
    tdt, adt = torch.from_numpy(pts).dtype, torch.from_numpy(attr).dtype
    big = torch.zeros(3 * n + 7, dtype=tdt, device="cuda")
    view = big.view(-1)[1:3 * n + 1].view(n, 3)
    view.copy_(torch.from_numpy(pts))
    abig = torch.zeros(5 * n + 3, dtype=adt, device="cuda")
    aview = abig[1:5 * n + 1].view(n, 5)
    aview.copy_(torch.from_numpy(attr))
    assert view.storage_offset() == 1 and view.is_contiguous() and view.data_ptr() % 16 != 0
    _, c_v = _check(pcu, oracle, view, (aview,), size=0.03)
    assert np.array_equal(c_np, c_t) and np.array_equal(c_np, c_v)
