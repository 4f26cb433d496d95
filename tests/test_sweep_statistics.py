"""The fused Chamfer / Hausdorff sweeps (the statistics-only k = 1 kernels) checked query by query.

Those sweeps write no per-point result, only one pcu_b200_nn_stats record per direction.  A Chamfer value
compared at 1e-6 cannot see a handful of queries that got a farther neighbour than their nearest, but the
record's two fp64 sums can:

  sum_sq_dist = sum of d2_min over the queries, d2_min in the input precision;
  sum_dist    = sum of sqrt(d2_min), a correctly rounded sqrt in the input precision, widened.

The reference's terms are the oracle's k_nearest_neighbors(q, d, 1, squared_distances=True), and math.fsum of
them is the correctly rounded exact sum.  Whatever order the device adds n non-negative terms in, its sum is
within gamma_(n-1) * sum of the exact one, so one wrong query is visible unless its two candidate distances
(nearly) tie.  On dyadic inputs -- coordinates k / 2^10 -- every d2 is a multiple of 2^-20; while the total
stays below 2^33, every partial sum is exact and sum_sq_dist must equal the reference's sum bit for bit.

The GPU tests run every entry point of the statistics sweeps (host staging, CUDA tensors, prepared clouds in
both directions, the batch) under every grid build, on the input families where the sweeps branch.  The CPU
test at the end shows that the checks reject a single wrong query.
"""
import contextlib
import math
import zlib
from functools import lru_cache

import numpy as np
import pytest

U = 2.0 ** -53
DYADIC_STEP = 2.0 ** -20   # d2 of two points with coordinates k / 2^10
STATS_WORDS = 10           # sizeof(pcu_b200_nn_stats) / 8


# ---- reference terms and the record check -------------------------------------------------------
def sum_bound(n, total):
    """Largest |device sum - fsum| for n non-negative fp64 terms summing to `total`, in any order:
    gamma_(n-1) * total for the device's rounding plus one rounding of fsum."""
    g = (n - 1) * U
    return (g / (1.0 - g) + U) * total


class Terms:
    """One direction of the reference: each query's nearest squared distance in the input precision."""

    def __init__(self, d2, dtype):
        d2 = np.asarray(d2, dtype=dtype).reshape(-1)
        w = d2.astype(np.float64)
        self.n = len(w)
        self.w = w
        self.roots = np.sqrt(d2).astype(np.float64)    # IEEE sqrt in the input precision, widened
        self.sq = math.fsum(w)
        self.root = math.fsum(self.roots)
        self.argmax = int(np.argmax(w))                # first maximal row, as Eigen's maxCoeff
        self.max = float(w[self.argmax])
        scaled = w / DYADIC_STEP
        self.exact = bool(np.all(scaled == np.floor(scaled))) and math.fsum(scaled) < 2.0 ** 53


def record_errors(rec, t):
    """What is wrong with one direction's record `rec` against the reference terms `t` (empty: nothing)."""
    errs = []
    if rec["n_queries"] != t.n:
        errs.append("n_queries %d, expected %d" % (rec["n_queries"], t.n))
    if t.exact:
        if rec["sum_sq_dist"] != t.sq:
            errs.append("sum_sq_dist %r, exact sum %r" % (rec["sum_sq_dist"], t.sq))
    elif not abs(rec["sum_sq_dist"] - t.sq) <= sum_bound(t.n, t.sq):
        errs.append("sum_sq_dist %r, reference %r, bound %.3g" % (rec["sum_sq_dist"], t.sq, sum_bound(t.n, t.sq)))
    if not abs(rec["sum_dist"] - t.root) <= sum_bound(t.n, t.root):
        errs.append("sum_dist %r, reference %r, bound %.3g" % (rec["sum_dist"], t.root, sum_bound(t.n, t.root)))
    if rec["max_sq_dist"] != t.max or rec["argmax_query"] != t.argmax:
        errs.append("max (%r, row %d), reference (%r, row %d)" % (rec["max_sq_dist"], rec["argmax_query"], t.max, t.argmax))
    return errs


_TERMS = {}


def reference_terms(oracle, q, d, dtype):
    """Terms of q -> d, computed once per pair of arrays (the cache keeps the arrays, so ids stay theirs)."""
    key = (id(q), id(d), np.dtype(dtype).str)
    hit = _TERMS.get(key)
    if hit is None or hit[0] is not q or hit[1] is not d:
        d2, _ = oracle.k_nearest_neighbors(q, d, 1, squared_distances=True)
        hit = _TERMS[key] = (q, d, Terms(d2, dtype))
    return hit[2]


def check_record(oracle, rec, q, d, dtype, other=None):
    """rec: the q -> d record of one call.  other: the d -> q record of the same bidirectional call, whose pair
    value both carry (chamfer_of64: sum_dist / n of one plus that of the other); None for a one-way call."""
    errs = record_errors(rec, reference_terms(oracle, q, d, dtype))
    if other is None:
        want = rec["sum_dist"] / rec["n_queries"]
    else:
        want = rec["sum_dist"] / rec["n_queries"] + other["sum_dist"] / other["n_queries"]
    if rec["pair_value"] != want:
        errs.append("pair_value %r, recomputed %r" % (rec["pair_value"], want))
    assert not errs, errs


def check_pair(oracle, recs, x, y, dtype, value=None):
    check_record(oracle, recs[0], x, y, dtype, recs[1])
    check_record(oracle, recs[1], y, x, dtype, recs[0])
    if value is not None:   # the scalar of the input precision, rounded from the fp64 pair value
        assert float(value) == float(np.dtype(dtype).type(recs[0]["pair_value"])), (float(value), recs[0]["pair_value"])


def decode_records(words):
    """pcu_b200_nn_stats records from their raw int64 words (what a device buffer holds)."""
    w = np.asarray(words, dtype=np.int64).reshape(-1, STATS_WORDS)
    f = w.view(np.float64)
    return [{"sum_dist": float(f[r, 0]), "sum_sq_dist": float(f[r, 1]), "max_sq_dist": float(f[r, 2]),
             "argmax_query": int(w[r, 3]), "argmax_data": int(w[r, 4]), "n_queries": int(w[r, 5]),
             "n_tied": int(w[r, 6]), "n_far": int(w[r, 7]), "witness_tied": int(w[r, 8]), "pair_value": float(f[r, 9])}
            for r in range(len(w))]


# ---- input families ------------------------------------------------------------------------------
def dyadic(rng, n, extent=1.0):
    """n points with coordinates k / 2^10 in [0, extent)^3: every squared distance is a multiple of 2^-20."""
    return np.floor(rng.random((n, 3)) * (1024 * extent)) / 1024


def _uniform(n, m, extent=1.0):
    return lambda rng: (dyadic(rng, n, extent), dyadic(rng, m, extent))


def _oversized(clustered_side):
    """40 000 points in a cube 1.2e-4 wide share one cell, so their slab outgrows the shared-memory staging."""
    def make(rng):
        cloud = np.concatenate([0.3 + 1.2e-4 * rng.random((40000, 3)), rng.random((60000, 3))])
        cloud = cloud[rng.permutation(len(cloud))]
        other = rng.random((50000, 3))
        return (cloud, other) if clustered_side == "queries" else (other, cloud)
    return make


def _disjoint(rng):
    """Boxes 40 apart: no query has a neighbour within its 3 x 3 x 3 cells (every query takes the far pass)."""
    return dyadic(rng, 20000), dyadic(rng, 30000) * np.array([1.0, 2.0, 1.0]) + np.array([40.0, -25.0, 3.0])


def _blobs(rng):
    """Uniform queries against three tight blobs in an empty box: most queries are beyond the rings (very-far
    list, pyramid pass); in the other direction the blobs search the uniform cloud."""
    blobs = np.concatenate([rng.normal(c, 0.002, (5000, 3)) for c in ((0.1, 0.1, 0.1), (0.9, 0.2, 0.7), (0.5, 0.95, 0.3))])
    return rng.random((20000, 3)), blobs


def _planar(rng):
    x, y = dyadic(rng, 30000, 4.0), dyadic(rng, 20000, 4.0)
    x[:, 2] = y[:, 2] = 0.25
    return x, y


def _collinear(rng):
    x, y = dyadic(rng, 20000, 64.0), dyadic(rng, 15000, 64.0)
    x[:, 1:] = (0.5, 0.75)
    y[:, 1:] = (0.5, 0.75)
    return x, y


def _identical(rng):
    return dyadic(rng, 5000), np.tile([[0.25, 0.5, 0.75]], (3000, 1))


def _shift4096(rng):
    return dyadic(rng, 20000) + 4096.0, dyadic(rng, 15000) + 4096.0


def _lattice(rng):
    """Integer lattice with 100 duplicated points, and the lattice shifted by half a cell: every query has
    several equally near neighbours."""
    lat = np.stack(np.meshgrid(*[np.arange(12.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = np.concatenate([lat, lat[:100]])
    return lat + 0.5, lat[rng.permutation(len(lat))]


def _walls(rng):
    """Near ties straddling cell walls, the case the row pruning of the main pass decides.  Dataset: columns along
    y on a square (x, z) lattice 3072 units of 2^-10 apart, one point every 4095 units along a column, each column
    at its own random phase.  Queries: on the columns, one unit below the middle of every gap, so the point above
    is 2047 units away and the point below 2048; the other columns are 3072 units away.  A query's upper neighbour
    lies in the row above whenever a y wall falls between them; when that wall is within about three units of the
    upper point (a few in a thousand queries), that row's lower bound is within 0.2 % of the lower point's
    distance, found first.  A sweep that prunes such a row on anything but `bound > best` answers the lower point."""
    cols, per, step, spacing = 48, 24, 4095, 3072
    cx, cz = (a.reshape(-1) * spacing for a in np.meshgrid(np.arange(cols), np.arange(cols), indexing="ij"))
    ys = rng.integers(0, step, cols * cols)[:, None] + step * np.arange(per)[None, :]
    qy = ys[:, :-1] + (step + 1) // 2
    data = np.stack([np.repeat(cx, per), ys.reshape(-1), np.repeat(cz, per)], -1)
    queries = np.stack([np.repeat(cx, per - 1), qy.reshape(-1), np.repeat(cz, per - 1)], -1)
    return queries[rng.permutation(len(queries))] / 1024.0, data[rng.permutation(len(data))] / 1024.0


def _sphere(rng, n, radius):
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v * radius + 0.5


F32, F64 = np.float32, np.float64
# name: (maker, dtypes).  The uniform sizes sit on either side of the build thresholds of Plan::layout: one CTA
# per cloud up to 8192 points, the cell-wise passes for a single pair up to 65536, the slab build above.  More
# than kSlabTile = 2048 slabs take the point-by-point partition: 3.3e6 fp64 points (1536 per slab) and 7e6 fp32
# points (3072 per slab).
FAMILIES = {
    "uniform_8191": (_uniform(8191, 8191), (F32, F64)),
    "uniform_8193": (_uniform(8193, 8191), (F32, F64)),
    "uniform_65535": (_uniform(65535, 60000), (F32, F64)),
    "uniform_65537": (_uniform(65537, 65535), (F32, F64)),
    "uniform_1e5_7e4": (_uniform(100000, 70000, 4.0), (F32, F64)),
    "uniform_1e6": (_uniform(1000000, 1000000, 16.0), (F32,)),
    "pointwise_3e6_f64": (_uniform(3300000, 100000, 16.0), (F64,)),
    "pointwise_7e6_f32": (_uniform(7000000, 50000, 16.0), (F32,)),
    "oversized_queries": (_oversized("queries"), (F32, F64)),
    "oversized_dataset": (_oversized("dataset"), (F32, F64)),
    "disjoint": (_disjoint, (F32, F64)),
    "blobs": (_blobs, (F32, F64)),
    "planar": (_planar, (F32, F64)),
    "collinear": (_collinear, (F32, F64)),
    "identical": (_identical, (F32, F64)),
    "single_query": (lambda rng: (dyadic(rng, 1), dyadic(rng, 7000)), (F32, F64)),
    "single_point_dataset": (lambda rng: (dyadic(rng, 7000), dyadic(rng, 1)), (F32, F64)),
    "shift4096": (_shift4096, (F32,)),
    "lattice": (_lattice, (F32, F64)),
    "walls": (_walls, (F32, F64)),
}
DYADIC_FAMILIES = {"uniform_8191", "uniform_8193", "uniform_65535", "uniform_65537", "uniform_1e5_7e4", "uniform_1e6",
                   "pointwise_3e6_f64", "pointwise_7e6_f32", "disjoint", "planar", "collinear", "identical",
                   "single_query", "single_point_dataset", "shift4096", "lattice", "walls"}
OCCUPANCY_FAMILIES = ("uniform_65537", "oversized_dataset", "blobs", "planar", "lattice", "walls")
CASES = [(name, dt) for name, (_, dts) in FAMILIES.items() for dt in dts]


def _seed(name):
    return zlib.crc32(name.encode())


@lru_cache(maxsize=None)
def case(name, dtype):
    x, y = FAMILIES[name][0](np.random.default_rng(_seed(name)))
    return np.ascontiguousarray(x, dtype=dtype), np.ascontiguousarray(y, dtype=dtype)


def builds(n, m):
    """Grid builds to run: automatic, cell-wise, slab; and first, one CTA per cloud where its cell counters fit in
    shared memory (kSmallMaxCells at the default 1.5 points per cell).  Binning 2 falls back to the cell-wise
    passes when they do not fit: for thin sets (planar, collinear, identical) the grid refinement learnt from a
    workspace's previous call with the same shapes can push the later calls of a case past that limit."""
    return (2, 0, 1, 3) if max(n, m) <= 65537 else (0, 1, 3)


@contextlib.contextmanager
def library_defaults(pcu, **kw):
    pcu._pcu_internal._set_defaults(**kw)
    try:
        yield
    finally:
        pcu._pcu_internal._set_defaults()


# ---- GPU: single pair ----------------------------------------------------------------------------
def _tensor(a):
    import torch
    return torch.from_numpy(a).cuda()


def _check_plain_calls(pcu, oracle, x, y, dtype, xt, yt):
    """_chamfer_stats (numpy, host staging) and _stats_device both ways and one way (CUDA tensors)."""
    value, sxy, syx = pcu._pcu_internal._chamfer_stats(x, y)
    check_pair(oracle, (sxy, syx), x, y, dtype, value)
    buf, val = pcu._stats_device(xt, yt, True, 10)
    recs = decode_records(buf.cpu().numpy())
    check_pair(oracle, recs, x, y, dtype, val.item())
    buf, _ = pcu._stats_device(xt, yt, False, 10)
    check_record(oracle, decode_records(buf.cpu().numpy())[0], x, y, dtype)
    return sxy, syx


def _check_prepared_calls(pcu, oracle, x, y, dtype, xt):
    """_stats_prepared (numpy) and _stats_prepared_device, bidirectional and one way, on handles prepared for
    Chamfer calls and for k = 16 k-NN calls (another cell size)."""
    for k in (None, 16):
        cloud = pcu.prepare_cloud(y, k=k)
        try:
            for both in (True, False):
                _, _, val, recs = pcu._prepared_stats(x, cloud, both, 10, None)
                if both:
                    check_pair(oracle, recs, x, y, dtype, val)
                else:
                    check_record(oracle, recs[0], x, y, dtype)
                _, _, val, (buf, _) = pcu._prepared_stats(xt, cloud, both, 10, None)
                recs = decode_records(buf.cpu().numpy())
                if both:
                    check_pair(oracle, recs, x, y, dtype, val.item())
                else:
                    check_record(oracle, recs[0], x, y, dtype)
        finally:
            cloud.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", CASES, ids=["%s-%s" % (n, np.dtype(d).name) for n, d in CASES])
def test_every_entry_point_and_build(pcu, oracle, name, dtype):
    x, y = case(name, dtype)
    xt, yt = _tensor(x), _tensor(y)
    for b in builds(len(x), len(y)):
        with library_defaults(pcu, binning=b):
            sxy, syx = _check_plain_calls(pcu, oracle, x, y, dtype, xt, yt)
            _check_prepared_calls(pcu, oracle, x, y, dtype, xt)
        if name == "disjoint":
            assert sxy["n_far"] == len(x) and syx["n_far"] == len(y), (b, sxy["n_far"], syx["n_far"])


@pytest.mark.gpu
@pytest.mark.parametrize("occupancy", [0.5, 8.0])
@pytest.mark.parametrize("name", OCCUPANCY_FAMILIES)
def test_cell_walls_moved(pcu, oracle, name, occupancy):
    """0.5 and 8 points per cell (three times finer and about five times coarser than the k = 1 default of 1.5)
    move every wall relative to the points."""
    for dtype in FAMILIES[name][1]:
        x, y = case(name, dtype)
        xt, yt = _tensor(x), _tensor(y)
        for b in (0, 1, 3):
            with library_defaults(pcu, binning=b, cell_occupancy=occupancy):
                _check_plain_calls(pcu, oracle, x, y, dtype, xt, yt)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_sphere_surfaces_through_grid_refinement(pcu, oracle, dtype):
    """Surfaces fill few cells, so from the second call with the same shapes the library refines the grid
    (per workspace: the numpy path and the tensor path each learn it).  Every call must stay exact."""
    rng = np.random.default_rng(_seed("sphere"))
    x = np.ascontiguousarray(_sphere(rng, 60000, 0.45), dtype=dtype)
    y = np.ascontiguousarray(_sphere(rng, 45000, 0.4), dtype=dtype)
    xt, yt = _tensor(x), _tensor(y)
    for b in (0, 1, 3):
        with library_defaults(pcu, binning=b):
            for _ in range(4):
                _check_plain_calls(pcu, oracle, x, y, dtype, xt, yt)


# ---- GPU: batch ----------------------------------------------------------------------------------
def _batch_pairs(rng, n, m):
    """Nine (n, m) pairs, each a different family at its own scale and offset, so every pair has its own grid."""
    def sized(make, scale, offset):
        a, b = make(rng)
        a = a[rng.integers(0, len(a), n)] if len(a) < n else a[:n]
        b = b[rng.integers(0, len(b), m)] if len(b) < m else b[:m]
        return a * scale + offset, b * scale + offset

    def oversized(r):
        cluster = 0.3 + 1.2e-4 * r.random((8000, 3))
        return np.concatenate([cluster, r.random((n - 8000, 3))])[r.permutation(n)], r.random((m, 3))

    return [sized(_uniform(n, m), 1.0, 0.0),
            sized(_disjoint, 0.5, -3.0),
            sized(_blobs, 8.0, 100.0),
            sized(oversized, 2.0, -50.0),
            sized(_planar, 0.25, 7.0),
            sized(_collinear, 1.0 / 64, 0.0),
            sized(lambda r: (dyadic(r, n), np.tile([[0.25, 0.5, 0.75]], (m, 1))), 4.0, 1.0),
            sized(lambda r: (_sphere(r, n, 0.45), _sphere(r, m, 0.4)), 1000.0, -500.0),
            sized(_shift4096, 1.0, 0.0)]


@lru_cache(maxsize=None)
def batch_case(name):
    rng = np.random.default_rng(_seed(name))
    if name == "families":
        pairs = _batch_pairs(rng, 20000, 9000)
    elif name == "uniform_130":
        pairs = [(dyadic(rng, 65536, 4.0), dyadic(rng, 65536, 4.0)) for _ in range(130)]
    elif name == "walls":   # four near-tie pairs at power-of-two scales and their own offsets
        pairs = [(q * s + o, d * s + o) for (q, d), s, o in zip((_walls(rng) for _ in range(4)), (1.0, 2.0, 0.25, 8.0),
                                                                (0.0, -100.0, 37.0, 1000.0))]
    else:   # "tiny_16400": more pairs than one launch slice (16384) holds
        pairs = [(dyadic(rng, 24), dyadic(rng, 17)) for _ in range(16400)]
    pairs = [(np.ascontiguousarray(a, dtype=F32), np.ascontiguousarray(b, dtype=F32)) for a, b in pairs]
    return pairs, np.stack([a for a, _ in pairs]), np.stack([b for _, b in pairs])


@pytest.fixture(scope="module", autouse=True)
def _release_cases():
    """The cached cases and their reference terms come to about a gigabyte of host memory: free them when the
    module is done, before the rest of the suite runs."""
    yield
    _TERMS.clear()
    case.cache_clear()
    batch_case.cache_clear()


@pytest.mark.gpu
@pytest.mark.parametrize("binning", [0, 1, 3])
@pytest.mark.parametrize("name,checked", [("families", None), ("uniform_130", None), ("walls", None),
                                          ("tiny_16400", (0, 16383, 16384, 16399))])
def test_batch_records(pcu, oracle, name, checked, binning):
    import torch
    pairs, xs, ys = batch_case(name)
    B = len(pairs)
    xt, yt = _tensor(xs), _tensor(ys)
    stats = torch.empty(2 * B * STATS_WORDS, dtype=torch.int64, device=xt.device)
    per_pair = torch.empty(B, dtype=torch.float32, device=xt.device)
    with library_defaults(pcu, binning=binning):
        pcu._pcu_internal._batched_chamfer_stats_device(xt.data_ptr(), yt.data_ptr(), B, xs.shape[1], ys.shape[1],
                                                        stats.data_ptr(), per_pair.data_ptr(), 10, xt.device.index or 0,
                                                        torch.cuda.current_stream(xt.device).cuda_stream)
        public = pcu.batched_chamfer_distance(xt, yt)
    recs = decode_records(stats.cpu().numpy())
    per_pair = per_pair.cpu().numpy()
    for p in range(B):   # the batch's value of every pair is chamfer_of<float> of its two records
        r0, r1 = recs[2 * p], recs[2 * p + 1]
        assert per_pair[p] == np.float32(r0["sum_dist"] / r0["n_queries"] + r1["sum_dist"] / r1["n_queries"]), p
    assert np.array_equal(public.cpu().numpy(), per_pair)
    for p in (range(B) if checked is None else checked):
        x, y = pairs[p]
        check_pair(oracle, (recs[2 * p], recs[2 * p + 1]), x, y, F32)
    if name == "families":
        assert recs[2]["n_far"] == len(pairs[1][0]) and recs[3]["n_far"] == len(pairs[1][1])   # the disjoint pair


# ---- CPU: the checks have teeth ------------------------------------------------------------------
def _two_nearest_terms(q, d, dtype):
    """Each query's nearest and second-nearest squared distance, rounded like the reference's metric."""
    from scipy.spatial import cKDTree
    _, idx = cKDTree(d.astype(np.float64)).query(q.astype(np.float64), k=2, workers=-1)
    q = q.astype(dtype)
    d = d.astype(dtype)

    def d2(i):
        diff = q - d[i]
        return (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]

    a, b = d2(idx[:, 0]), d2(idx[:, 1])
    return np.minimum(a, b), np.maximum(a, b)


def _with_one_wrong_query(t, i, w2, r2):
    """The record a sweep would produce if query i had taken its second-nearest neighbour (w2, sqrt r2)."""
    mx, arg = t.max, t.argmax
    if w2 > mx or (w2 == mx and i < arg):
        mx, arg = w2, i
    s = t.root + (r2 - t.roots[i])
    return {"n_queries": t.n, "sum_sq_dist": t.sq + (w2 - t.w[i]), "sum_dist": s, "max_sq_dist": mx,
            "argmax_query": arg, "pair_value": s / t.n}


TEETH_CASES = [("uniform_1e5_7e4", F32), ("uniform_1e6", F32), ("pointwise_3e6_f64", F64), ("oversized_dataset", F32),
               ("disjoint", F64), ("blobs", F32), ("planar", F32), ("collinear", F64), ("single_query", F32),
               ("shift4096", F32), ("walls", F32)]


def test_one_wrong_query_is_rejected():
    """In every family (the 10^6 x 10^6 one included) the check rejects a record in which one query took its
    second-nearest neighbour, for at least 99 % of the queries whose two nearest distances differ.  A query
    whose two nearest are equally far has no wrong answer the statistics could show; the all-identical and
    lattice families have (almost) only such queries and are left out.  The dyadic families meet the
    precondition of the exact comparison."""
    rng = np.random.default_rng(1)
    for name, dtype in TEETH_CASES:
        x, y = case(name, dtype)
        for q, d in ((x, y), (y, x)):
            if len(d) < 2:
                continue
            w1, w2 = _two_nearest_terms(q, d, dtype)
            t = Terms(w1, dtype)
            assert record_errors(_with_one_wrong_query(t, 0, t.w[0], t.roots[0]), t) == []
            assert t.exact == (name in DYADIC_FAMILIES), name
            differ = np.flatnonzero(w2 != w1)
            assert len(differ) > 0, name
            rows = differ if len(differ) <= 20000 else rng.choice(differ, 20000, replace=False)
            w2d = w2.astype(np.float64)
            r2d = np.sqrt(w2).astype(np.float64)
            caught = sum(bool(record_errors(_with_one_wrong_query(t, int(i), float(w2d[i]), float(r2d[i])), t)) for i in rows)
            assert caught >= 0.99 * len(rows), (name, len(q), caught, len(rows))
