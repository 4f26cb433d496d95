"""Nearest-neighbour search where the rounded squared distance ((dx^2 + dy^2) + dz^2) reaches the top or the
bottom of the floating-point range.

nanoflann admits a candidate only when its distance is strictly below the list's current worst, which starts at
the largest finite value (KNNResultSet::init), not at +inf.  So a point whose rounded d^2 equals FLT_MAX / DBL_MAX
exactly, or overflows to +inf, is never a neighbour; a row with fewer than k admissible points is padded with
-1 / -1.0.  The grid sweeps, the pyramid descent and the fused metric sweeps must follow the same rule.

Families (seeded; every reference answer is computed by the oracle at test time):
  max_*       points whose d^2 to every query is exactly the largest finite value: alone, mixed with a few nearer
              points, and spread so that the boundary points are met by the main, far and very-far passes (filler
              points at +inf distance stretch the grid along x)
  overflow    two clusters at +-1e19 (fp32) / +-1e154 (fp64): finite within a cluster, +inf between them; one query
              cluster sees every point at +inf
  underflow   clouds whose extent is 1e-38 .. 1e-42 (fp32) or 1e-305 .. 1e-309 (fp64): every d^2 underflows to 0
              and the cell size's inverse overflows, so nearly every row is a tie for the kd-tree replay
  mixed       a unit-cube cloud plus one outlier at 1e30: the grid collapses to about one occupied cell

Metrics on rows that find nothing: such a row counts as -1 in the Hausdorff maximum (the reference's padded
distance), so the Hausdorff results match the oracle.  The fused Chamfer distance is +inf as soon as one row of
either direction finds nothing (DESIGN.md section 3); the reference instead indexes x[-1] there.
"""
import zlib
from contextlib import closing

import numpy as np
import pytest

from meshes import to_numpy

F32, F64 = np.float32, np.float64
DTYPES = [F32, F64]
KS_MAX = [1, 3, 8, 20, 40]     # thread lists of capacity 4 / 8 / 16 / 32, the warp pass and the k > 32 descent
KS_OTHER = [1, 4, 40]


def boundary_xy(dtype):
    """(X, Y) with fl(X * X) one ulp below the largest finite value and fl(fl(X * X) + fl(Y * Y)) equal to it."""
    top = np.finfo(dtype).max
    x = dtype(np.sqrt(np.float64(top)))
    with np.errstate(over="ignore"):
        while not x * x < top:
            x = np.nextafter(x, dtype(0))
        while True:
            up = np.nextafter(x, dtype(np.inf))
            if not up * up < top:
                break
            x = up
        # Y^2 between half an ulp and one and a half ulps of the top: rounds the sum up to the top, not to +inf
        ulp = top - np.nextafter(top, dtype(0))
        y = dtype(np.sqrt(np.float64(ulp) * 0.8) if dtype == F32 else np.sqrt(ulp * 0.8))
    return x, y


def rounded_d2(q, p):
    """The metric's squared distance, rounded like nanoflann's L2_Simple, for every (query, point) pair."""
    with np.errstate(over="ignore", under="ignore"):
        d = q[:, None, :] - p[None, :, :]
        s = d * d
        return (s[..., 0] + s[..., 1]) + s[..., 2]


def _small(rng, n, dtype, spread_z=0.0):
    """n points with x, y in (-64, 64) and z in (-64, 64) or spread over +-spread_z."""
    xy = rng.uniform(-64.0, 64.0, (n, 2))
    z = rng.uniform(-spread_z, spread_z, n) if spread_z else rng.uniform(-64.0, 64.0, n)
    return np.column_stack([xy, z]).astype(dtype)


def family(name, dtype):
    """(queries, dataset) of one family, both C-contiguous in `dtype`."""
    rng = np.random.default_rng([zlib.crc32(name.encode()), np.dtype(dtype).itemsize])
    X, Y = boundary_xy(dtype)
    big = dtype(2e19 if dtype == F32 else 2e154)   # big^2 overflows: points offset by it along y are at +inf
    if name.startswith("max_"):
        spread = 1e12 if name.startswith("max_spread") else 0.0
        # A single boundary point is what shows a wrong admission: several of them tie at the largest value, and a
        # tied row is answered by the kd-tree replay.
        n_near = {"max_only": 0, "max_single": 0, "max_mixed": 5}.get(name, 2)
        n_bound = {"max_only": 8}.get(name, 1)
        n_query = 3000 if name.startswith("max_spread") else 200
        q = _small(rng, n_query, dtype, spread)
        near = _small(rng, n_near, dtype, spread)
        bz = _small(rng, n_bound, dtype, spread)[:, 2]
        bound = np.column_stack([np.full(n_bound, X), np.full(n_bound, Y), bz]).astype(dtype)
        fill = int(name.rsplit("_", 1)[1]) if name.startswith("max_spread") else 0
        filler = np.column_stack([rng.uniform(0.0, 1.0, fill) * np.float64(X), np.full(fill, np.float64(big)),
                                  rng.uniform(-1e12, 1e12, fill)]).astype(dtype)
        d = np.concatenate([near, bound, filler])
        d = d[rng.permutation(len(d))]
    elif name.startswith("overflow"):
        c = 1e19 if dtype == F32 else 1e154
        def cluster(n, centre):
            return (np.asarray(centre, np.float64) * c * (1.0 + 0.1 * rng.random((n, 3)))).astype(dtype)
        # overflow: 24 points at +C and 3000 at -C; overflow_lone: one point at -C, so that a row of the +C queries
        # has a single +inf candidate after its 24 finite ones (nothing ties with it)
        a, b = cluster(24, [1, 1, 1]), cluster(3000 if name == "overflow" else 1, [-1, -1, -1])
        d = np.concatenate([a, b])
        d = d[rng.permutation(len(d))]
        q = np.concatenate([cluster(300, [1, 1, 1]), cluster(300, [-1, -1, -1]), cluster(300, [1, -1, 1])])
    elif name.startswith("underflow"):
        ext = float(name.split("_")[1])
        q = (rng.random((2000, 3)) * ext).astype(dtype)
        d = (rng.random((2000, 3)) * ext).astype(dtype)
    elif name == "mixed":
        d = np.concatenate([rng.random((10000, 3)), [[1e30, 1e30, 1e30]]]).astype(dtype)
        q = np.concatenate([rng.random((3000, 3)), [[1e30, 1e30, 1e30], [-1e30, 0.0, 0.0]]]).astype(dtype)
    else:
        raise ValueError(name)
    return np.ascontiguousarray(q), np.ascontiguousarray(d)


MAX_FAMILIES = ["max_only", "max_single", "max_mixed", "max_spread_0", "max_spread_400", "max_spread_6000"]
UNDERFLOW = {F32: ["underflow_1e-38", "underflow_1e-40", "underflow_1e-42"], F64: ["underflow_1e-305", "underflow_1e-309"]}
# extents below which even a single cell's inverse size overflows (finer grids overflow sooner)
INV_H_OVERFLOWS = {"underflow_1e-40", "underflow_1e-42", "underflow_1e-309"}
CASES = ([(f, dt, k) for f in MAX_FAMILIES for dt in DTYPES for k in KS_MAX] +
         [(f, dt, k) for f in ("overflow", "overflow_lone") for dt in DTYPES for k in KS_OTHER + [25]] +
         [(f, dt, k) for dt in DTYPES for f in UNDERFLOW[dt] for k in KS_OTHER] +
         [("mixed", dt, k) for dt in DTYPES for k in KS_OTHER])
FAMILIES = [(f, dt) for f in MAX_FAMILIES + ["overflow", "overflow_lone", "mixed"] for dt in DTYPES] + \
           [(f, dt) for dt in DTYPES for f in UNDERFLOW[dt]]


def _id(case):
    return "-".join(str(c) if not isinstance(c, type) else np.dtype(c).name for c in case)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_boundary_point_lands_on_the_largest_finite_value(dtype):
    X, Y = boundary_xy(dtype)
    top = np.finfo(dtype).max
    assert X * X == np.nextafter(top, dtype(0))
    d2 = rounded_d2(np.zeros((1, 3), dtype), np.array([[X, Y, 0]], dtype))[0, 0]
    assert d2 == top
    if dtype == F32:
        assert X == F32(1.8446743e19)


@pytest.mark.parametrize("name,dtype", FAMILIES, ids=[_id(c) for c in FAMILIES])
def test_families_reach_their_boundaries(name, dtype):
    q, d = family(name, dtype)
    assert q.dtype == d.dtype == dtype and len(d) <= 20001 and np.isfinite(q).all() and np.isfinite(d).all()
    d2 = rounded_d2(q, d)
    top = np.finfo(dtype).max
    if name.startswith("max_"):
        X, _ = boundary_xy(dtype)
        on = d2 == top
        bound = d[:, 0] == X
        assert on[:, bound].all(), "every boundary point must sit exactly at the largest finite d^2 of every query"
        assert not np.isinf(d2[:, bound]).any()
        rest = d2[:, ~bound]
        if name in ("max_only", "max_single"):
            assert rest.size == 0
        elif name == "max_mixed":
            assert (rest < top).all() and rest.shape[1] == 5     # fewer near points than most k
        if name != "max_only":
            assert bound.sum() == 1
        else:
            near = (np.abs(d[~bound, 1]) < 1e3)
            assert (rest[:, near] < top).all() and np.isinf(rest[:, ~near]).all()
    elif name.startswith("overflow"):
        fin = np.isfinite(d2)
        assert fin.any() and (~fin).any()
        per_row = fin.sum(axis=1)
        assert (per_row == 0).sum() == 300           # the third query cluster sees only +inf
        assert (per_row == 24).sum() == 300          # the small cluster: rows padded at k = 25 and 40
        if name == "overflow_lone":
            assert ((~fin).sum(axis=1)[per_row == 24] == 1).all()
        assert (d2[fin] < top).all()
    elif name.startswith("underflow"):
        ext = float(name.split("_")[1])
        assert (d2 == 0).mean() > 0.99 and len(np.unique(d, axis=0)) > 1
        with np.errstate(over="ignore"):
            # the cell size h is at most the extent, so 1 / h overflows in the input precision at least here
            assert np.isinf(dtype(1.0 / ext)) == (name in INV_H_OVERFLOWS)
        if name in INV_H_OVERFLOWS:
            assert (np.abs(d) < np.finfo(dtype).tiny).all()   # subnormal coordinates
    elif name == "mixed":
        out = d[:, 0] == dtype(1e30)
        assert out.sum() == 1
        if dtype == F32:
            assert np.isinf(d2[:-2][:, out]).all()      # the outlier is at +inf from the unit cube
        assert np.isinf(d2[-1]).all() == (dtype == F32)  # the query at -1e30 finds nothing in fp32


def _admissible_brute(q, d, k, squared):
    """(dist, idx) of the k nearest admissible points (d^2 < largest finite) ordered by (d^2, index), -1 padded;
    rows whose answer depends on tie order (equal d^2 inside the list or at its edge) are marked in `tied`."""
    d2 = rounded_d2(q, d)
    top = np.finfo(d.dtype).max
    order = np.lexsort((np.broadcast_to(np.arange(len(d)), d2.shape), d2), axis=-1)
    srt = np.take_along_axis(d2, order, axis=1)
    ok = srt < top
    n = len(q)
    idx = np.full((n, k), -1, np.int64)
    dist = np.full((n, k), -1.0, d.dtype)
    m = min(k, len(d))
    keep = ok[:, :m]
    idx[:, :m] = np.where(keep, order[:, :m], -1)
    dist[:, :m] = np.where(keep, srt[:, :m] if squared else np.sqrt(srt[:, :m]), -1.0)
    tied = np.zeros(n, bool)
    if len(d) > 1:
        eq = (srt[:, 1:] == srt[:, :-1]) & ok[:, 1:]
        tied = eq[:, :min(k, len(d) - 1)].any(axis=1)
    return dist, idx, tied


@pytest.mark.parametrize("name,dtype", FAMILIES, ids=[_id(c) for c in FAMILIES])
def test_oracle_back_ends_agree(name, dtype, oracle):
    """The restatement and the reference's own nanoflann (where it could be built) agree on every family, and
    both agree with a brute-force search under the admission rule on every row whose answer no tie decides."""
    q, d = family(name, dtype)
    sub = slice(0, 400)                       # brute force is quadratic: a slice of the queries
    impls = ["port"] + (["reference"] if oracle.have_reference() else [])
    for k in (1, 8, 40):
        for sq in (False, True):
            res = [oracle.k_nearest_neighbors(q, d, k, sq, impl=impl) for impl in impls]
            for dist, idx in res[1:]:
                np.testing.assert_array_equal(idx, res[0][1])
                np.testing.assert_array_equal(dist, res[0][0])
            bd, bi, tied = _admissible_brute(q[sub], d, k, sq)
            gd = res[0][0].reshape(len(q), k)[sub]
            gi = res[0][1].reshape(len(q), k)[sub]
            np.testing.assert_array_equal(gi[~tied], bi[~tied])
            np.testing.assert_array_equal(gd[~tied], bd[~tied])
            # whatever ties decide, the same number of admissible neighbours is found
            np.testing.assert_array_equal((gi >= 0).sum(axis=1), (bi >= 0).sum(axis=1))
        hs = [oracle.hausdorff_distance(q, d, return_index=True, impl=impl) for impl in impls]
        assert all(h == hs[0] for h in hs)


# ------------------------------------------------------------------------------------------------ GPU
def _forms(pcu, q, d, k):
    """(label, query argument, dataset argument, closer) for every entry point of k_nearest_neighbors."""
    import torch
    qt, dt = torch.from_numpy(q).cuda(), torch.from_numpy(d).cuda()
    yield "numpy", q, d
    yield "cuda", qt, dt
    for kk in (None, k):
        for label, qa, da in (("numpy", q, d), ("cuda", qt, dt)):
            cloud = pcu.prepare_cloud(da, k=kk)
            try:
                yield "prepared(%s, k=%s)" % (label, kk), qa, cloud
            finally:
                cloud.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype,k", CASES, ids=[_id(c) for c in CASES])
def test_knn_matches_oracle(name, dtype, k, pcu, oracle):
    q, d = family(name, dtype)
    for sq in (False, True):
        rd, ri = oracle.k_nearest_neighbors(q, d, k, sq)
        for label, qa, da in _forms(pcu, q, d, k):
            gd, gi = pcu.k_nearest_neighbors(qa, da, k, sq)
            gd, gi = to_numpy(gd), to_numpy(gi)
            bad = np.flatnonzero((gi.reshape(len(q), -1) != ri.reshape(len(q), -1)).any(axis=1) |
                                 (gd.reshape(len(q), -1).view(np.uint8).reshape(len(q), -1) !=
                                  rd.reshape(len(q), -1).view(np.uint8).reshape(len(q), -1)).any(axis=1))
            assert bad.size == 0, "%s squared=%s: %d rows differ, first %s: gpu %s %s, oracle %s %s" % (
                label, sq, bad.size, bad[:5], gi.reshape(len(q), -1)[bad[0]], gd.reshape(len(q), -1)[bad[0]],
                ri.reshape(len(q), -1)[bad[0]], rd.reshape(len(q), -1)[bad[0]])


def _unfound_rows(q, d):
    return int((rounded_d2(q, d).min(axis=1) >= np.finfo(d.dtype).max).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", FAMILIES, ids=[_id(c) for c in FAMILIES])
def test_metrics_match_oracle(name, dtype, pcu, oracle):
    import torch
    q, d = family(name, dtype)
    qt, dt = torch.from_numpy(q).cuda(), torch.from_numpy(d).cuda()
    for sq in (False, True):
        for src, tgt, s_np, t_np in ((q, d, q, d), (d, q, d, q), (qt, dt, q, d), (dt, qt, d, q)):
            ref = oracle.one_sided_hausdorff_distance(s_np, t_np, True, sq)
            assert pcu.one_sided_hausdorff_distance(src, tgt, True, sq) == ref
            with closing(pcu.prepare_cloud(tgt)) as cloud:
                assert pcu.one_sided_hausdorff_distance(src, cloud, True, sq) == ref
        ref = oracle.hausdorff_distance(q, d, return_index=True, squared_distances=sq)
        assert pcu.hausdorff_distance(q, d, return_index=True, squared_distances=sq) == ref
        assert pcu.hausdorff_distance(qt, dt, return_index=True, squared_distances=sq) == ref
        with closing(pcu.prepare_cloud(dt)) as cloud:
            assert pcu.hausdorff_distance(qt, cloud, return_index=True, squared_distances=sq) == ref
        with closing(pcu.prepare_cloud(d)) as cloud:
            assert pcu.hausdorff_distance(q, cloud, return_index=True, squared_distances=sq) == ref

    # Chamfer: +inf as soon as a row of either direction has no admissible neighbour, else the oracle's value
    unfound = _unfound_rows(q, d) + _unfound_rows(d, q)
    ref = float(oracle.chamfer_distance(q, d))
    values = [float(pcu.chamfer_distance(q, d)), float(pcu.chamfer_distance(qt, dt))]
    with closing(pcu.prepare_cloud(d)) as cloud:
        values.append(float(pcu.chamfer_distance(q, cloud)))
    with closing(pcu.prepare_cloud(dt)) as cloud:
        values.append(float(pcu.chamfer_distance(qt, cloud)))
    if dtype == F32:
        n = min(len(q), len(d))
        xb, yb = np.stack([q[:n], q[:n]]), np.stack([d[:n], d[:n]])
        unfound_b = _unfound_rows(q[:n], d[:n]) + _unfound_rows(d[:n], q[:n])
        ref_b = float(oracle.chamfer_distance(q[:n], d[:n]))
        for got in list(to_numpy(pcu.batched_chamfer_distance(xb, yb))) + \
                list(to_numpy(pcu.batched_chamfer_distance(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda()))):
            if unfound_b:
                assert np.isinf(got) and got > 0
            else:
                assert got == pytest.approx(ref_b, rel=1e-5, abs=0)
    for got in values:
        if unfound:
            assert np.isinf(got) and got > 0, (got, ref)
        else:
            assert got == pytest.approx(ref, rel=1e-5, abs=0)
    # the per-point path with indices follows the reference literally (numpy indexes x[-1] on unfound rows), for
    # numpy, CUDA-tensor and CPU-tensor inputs alike
    rcham, rxy, ryx = oracle.chamfer_distance(q, d, return_index=True)
    for xa, ya in ((q, d), (qt, dt), (qt.cpu(), dt.cpu())):
        cham, cxy, cyx = pcu.chamfer_distance(xa, ya, return_index=True)
        np.testing.assert_array_equal(to_numpy(cxy), rxy)
        np.testing.assert_array_equal(to_numpy(cyx), ryx)
        cham = float(cham)
        assert cham == pytest.approx(float(rcham), rel=1e-5, abs=0), (type(xa), cham, rcham)


@pytest.mark.gpu
@pytest.mark.parametrize("fill", [0, 400, 6000])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_spread_families_reach_the_slow_passes(dtype, fill, pcu, oracle):
    """A max_spread dataset without its near points leaves every query with the boundary point (exactly the largest
    finite d^2) and the fillers (+inf): no query has a neighbour.  Without fillers the grid is one cell, the main
    pass's wall bound is +inf and every query settles there; fillers stretch the grid, so the main pass settles no
    query and every one goes on to the far pass (and from there to the very-far descent), which the statistics
    record counts in n_far."""
    import torch
    q, d = family("max_spread_%d" % fill, dtype)
    X, _ = boundary_xy(dtype)
    lone = np.ascontiguousarray(d[(d[:, 0] == X) | (np.abs(d[:, 1]) > 1e3)])
    assert len(lone) == fill + 1 and _unfound_rows(q, lone) == len(q)
    qt, lt = torch.from_numpy(q).cuda(), torch.from_numpy(lone).cuda()
    buf, _ = pcu._stats_device(qt, lt, True, 10)
    rec = pcu._stats_from_tensor(buf, 0)
    assert rec["n_far"] == (0 if fill == 0 else len(q)), rec
    assert (rec["max_sq_dist"], rec["argmax_query"], rec["argmax_data"]) == (-1.0, 0, -1)
    assert np.isinf(rec["sum_dist"]) and np.isinf(rec["sum_sq_dist"])
    for sq in (False, True):
        ref = oracle.one_sided_hausdorff_distance(q, lone, True, sq)
        assert ref == (-1.0, 0, -1)
        assert pcu.one_sided_hausdorff_distance(qt, lt, True, sq) == ref
    for k in KS_MAX:
        gd, gi = pcu.k_nearest_neighbors(qt, lt, k)
        assert (to_numpy(gi) == -1).all() and (to_numpy(gd) == -1).all()
