"""Poisson-disk downsampling (downsample_point_cloud_poisson_disk; /root/reference/src/sample_point_cloud.cpp:14-109,
:240-333).

The reference's subset (libigl blue noise, std::mt19937, hash-map order) cannot be reproduced, so the library defines
the sample exactly (csrc/poisson.cuh) and this file restates that definition sequentially: rows visited by ascending
key (mix32(seed ^ mix32(row * 0x9E3779B9 + 0x85EBCA6B)), row), each kept unless its rounded squared distance to a kept
row is below rr = fl(r * r).  The GPU result must equal that restatement row for row."""
import inspect

import numpy as np
import pytest
from scipy.spatial import cKDTree

from conftest import load_golden

GOLDEN_SETS = ["clustered", "duplicates", "lattice_self", "lattice_half", "planar", "collinear", "offset"]


# ---- the sequential definition -------------------------------------------------------------------------------------
def _mix32(h):
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x7FEB352D)
    h = h ^ (h >> np.uint32(15))
    h = h * np.uint32(0x846CA68B)
    return h ^ (h >> np.uint32(16))


def key_hash(rows, seed):
    r = np.asarray(rows, dtype=np.uint32)
    with np.errstate(over="ignore"):
        return _mix32(np.uint32(seed & 0xFFFFFFFF) ^ _mix32(r * np.uint32(0x9E3779B9) + np.uint32(0x85EBCA6B)))


def _d2(points, i, cand):
    """((dx*dx + dy*dy) + dz*dz), every operation rounded in the cloud's precision (numpy does not fuse)."""
    d = points[i] - points[cand]
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def poisson_disk_indices(points, radius, seed):
    """The greedy maximal independent set in key order, with a kd-tree ball (widened past every rounding of the
    metric) as the candidate set of each kept row and the exact rounded metric as the test."""
    points = np.ascontiguousarray(points)
    T = points.dtype.type
    with np.errstate(over="ignore", under="ignore"):
        r = T(radius)
        rr = T(r * r)
    n = points.shape[0]
    order = np.lexsort((np.arange(n), key_hash(np.arange(n), seed)))
    tiny = float(np.finfo(T).smallest_subnormal)
    reach = np.sqrt((float(rr) + 4.0 * tiny) * (1.0 + 1e-5)) * (1.0 + 1e-9)
    tree = cKDTree(points.astype(np.float64))
    blocked = np.zeros(n, dtype=bool)
    kept = []
    for i in order:
        if blocked[i]:
            continue
        kept.append(i)
        if not rr > 0:
            continue
        cand = np.asarray(tree.query_ball_point(points[i].astype(np.float64), reach), dtype=np.int64)
        with np.errstate(over="ignore", invalid="ignore"):
            blocked[cand[_d2(points, i, cand) < rr]] = True
    return np.sort(np.asarray(kept, dtype=np.int64)).astype(np.int32)


def target_mode(points, target, seed, tol=0.04, sample=None):
    """:278-326 transcribed line by line around `sample` (default: the definition above).  Returns (rows, radii
    tried, bisection steps)."""
    points = np.ascontiguousarray(points)
    T = points.dtype.type
    n = points.shape[0]
    radii = []

    def run(r):
        radii.append(r)
        return (sample or (lambda rad: poisson_disk_indices(points, rad, seed)))(r)

    if target >= n:
        return np.arange(n, dtype=np.int32), radii, 0
    tol = np.float32(tol)
    num_samples_min = int(T(target) * T(np.float32(1.0) - tol))
    num_samples_max = int(T(target) * T(np.float32(1.0) + tol))
    bmin, bmax = points.min(axis=0), points.max(axis=0)
    e = (bmax - bmin).astype(T)
    bbsize = T(np.sqrt(T(T(e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])))
    if bbsize == 0:
        return run(T(1)), radii, 0          # the divergence: any positive radius gives one sample
    range_min_rad = T(float(bbsize) / 50.0)
    range_max_rad = T(float(bbsize) / 50.0)
    while True:
        range_min_rad = T(float(range_min_rad) / 2.0)
        ret = run(range_min_rad)
        if not len(ret) < target:
            break
    while True:
        range_max_rad = T(float(range_max_rad) * 2.0)
        ret = run(range_max_rad)
        if not len(ret) > target:
            break
    iter_count = 0
    while iter_count < 20 and (len(ret) < num_samples_min or len(ret) > num_samples_max):
        iter_count += 1
        current_rad = T(float(T(range_min_rad + range_max_rad)) / 2.0)
        ret = run(current_rad)
        if len(ret) > target:
            range_min_rad = current_rad
        if len(ret) < target:
            range_max_rad = current_rad
    return ret, radii, iter_count


def _check_sample(points, radius, idx):
    """Separation and maximality by brute force (small clouds)."""
    T = points.dtype.type
    rr = T(T(radius) * T(radius))
    s = points[idx]
    for j in range(len(idx)):
        d2 = _d2(s, j, np.arange(len(idx)))
        d2[j] = np.inf
        assert np.all(d2 >= rr)
    inside = np.zeros(len(points), dtype=bool)
    inside[idx] = True
    for i in np.nonzero(~inside)[0]:
        assert np.any(_d2(points, i, idx) < rr)


# ---- CPU: interface, arguments, the definition itself -------------------------------------------------------------
def test_signature(pcu):
    sig = inspect.signature(pcu.downsample_point_cloud_poisson_disk)
    ps = list(sig.parameters.values())
    assert [p.name for p in ps] == ["v", "radius", "target_num_samples", "random_seed", "sample_num_tolerance", "device"]
    assert [p.default for p in ps[2:5]] == [-1, 0, 0.04]
    assert ps[0].default is inspect.Parameter.empty and ps[1].default is inspect.Parameter.empty
    assert all(p.kind == inspect.Parameter.POSITIONAL_OR_KEYWORD for p in ps[:5])
    assert ps[5].kind == inspect.Parameter.KEYWORD_ONLY and ps[5].default is None
    assert "downsample_point_cloud_poisson_disk" in pcu.__all__


def test_argument_errors(pcu):
    pts = np.random.default_rng(0).random((50, 3))
    f = pcu.downsample_point_cloud_poisson_disk
    with pytest.raises(ValueError, match="Cannot have both num_samples <= 0 and radius <= 0"):
        f(pts, 0.0)
    with pytest.raises(ValueError, match="Cannot have both num_samples <= 0 and radius <= 0"):
        f(pts, -1.0, target_num_samples=0)
    with pytest.raises(ValueError, match=r"sample_num_tolerance must be in \(0, 1\]"):
        f(pts, 0.1, sample_num_tolerance=0.0)
    with pytest.raises(ValueError, match=r"sample_num_tolerance must be in \(0, 1\]"):
        f(pts, 0.1, sample_num_tolerance=1.5)
    with pytest.raises(ValueError, match="scalar type"):
        f(pts.astype(np.int32), 0.1)
    with pytest.raises(ValueError, match="shape"):
        f(pts[:, :2], 0.1)
    with pytest.raises(ValueError, match="NumPy array"):
        f(pts.tolist(), 0.1)


def test_trivial_inputs_stay_on_the_host(pcu):
    pts = np.random.default_rng(1).random((40, 3)).astype(np.float32)
    out = pcu.downsample_point_cloud_poisson_disk(pts, 0.1, target_num_samples=40)          # :279-283
    assert out.dtype == np.int32 and np.array_equal(out, np.arange(40))
    out = pcu.downsample_point_cloud_poisson_disk(pts, 0.1, target_num_samples=1000)
    assert np.array_equal(out, np.arange(40))
    empty = pcu.downsample_point_cloud_poisson_disk(np.zeros((0, 3)), 0.1)
    assert empty.dtype == np.int32 and empty.shape == (0,)


def test_key_function_is_pinned():
    assert [hex(int(h)) for h in key_hash([0, 1, 2, 1000003], 1)] == ["0xf34cbb46", "0x1d933028", "0x8760c00d", "0xee56527d"]
    assert [hex(int(h)) for h in key_hash([0, 1, 2, 1000003], 12345)] == ["0xf80bec16", "0x79f29964", "0xb1899220", "0xdd32ba99"]
    assert [hex(int(h)) for h in key_hash([0, 1, 2, 1000003], 0xFFFFFFFF)] == ["0x48c12747", "0xe2c141dd", "0xe53895b3", "0x35cb2437"]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("radius", [0.04, 0.1, 0.25])
def test_definition_is_separated_and_maximal(dtype, radius):
    pts = np.random.default_rng(7).random((1500, 3)).astype(dtype)
    idx = poisson_disk_indices(pts, radius, 99)
    assert 0 < len(idx) < len(pts)
    _check_sample(pts, radius, idx)
    # it is the greedy in key order: the first row in key order is always a sample
    first = np.lexsort((np.arange(len(pts)), key_hash(np.arange(len(pts)), 99)))[0]
    assert first in idx
    assert not np.array_equal(idx, poisson_disk_indices(pts, radius, 100))


def test_definition_matches_a_quadratic_greedy():
    pts = np.random.default_rng(8).random((400, 3)).astype(np.float32)
    r = np.float32(0.15)
    rr = np.float32(r * r)
    order = np.lexsort((np.arange(400), key_hash(np.arange(400), 5)))
    kept = []
    for i in order:
        if not kept or np.all(_d2(pts, i, np.asarray(kept)) >= rr):
            kept.append(i)
    assert np.array_equal(poisson_disk_indices(pts, r, 5), np.sort(kept).astype(np.int32))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_target_search_follows_the_reference_loop(pcu, dtype):
    """The package's search (pcu_b200._poisson.target_search) and the transcription above try the same radii, in the
    same order, when both drive the same sampler."""
    from pcu_b200._poisson import target_search
    pts = (np.random.default_rng(9).random((800, 3)) * [2.0, 1.0, 0.5]).astype(dtype)
    for target in (40, 200, 555):
        rows, radii, _ = target_mode(pts, target, 3)
        seen = []

        def sample(r):
            seen.append(r)
            return len(poisson_disk_indices(pts, r, 3))
        T = np.dtype(dtype).type
        e = (pts.max(axis=0) - pts.min(axis=0)).astype(T)
        bbsize = T(np.sqrt(T(T(e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])))
        count = target_search(sample, dtype, bbsize, target, 0.04)
        assert [type(r) for r in seen] == [T] * len(seen)
        assert seen == radii and count == len(rows)


# ---- GPU: exact equality with the definition ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("radius", [0.012, 0.03, 0.08])
def test_uniform_matches_the_definition(pcu, dtype, radius):
    pts = np.random.default_rng(11).random((20000, 3)).astype(dtype)
    got = pcu.downsample_point_cloud_poisson_disk(pts, radius, random_seed=77)
    assert got.dtype == np.int32
    assert np.array_equal(got, poisson_disk_indices(pts, radius, 77))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("name", GOLDEN_SETS)
def test_golden_point_sets_match_the_definition(pcu, name, dtype):
    pts = load_golden("%s_%s" % (name, dtype))["dataset"]
    ext = float(np.linalg.norm(pts.max(axis=0).astype(np.float64) - pts.min(axis=0)))
    for frac in (0.01, 0.08):
        radius = frac * ext
        got = pcu.downsample_point_cloud_poisson_disk(pts, radius, random_seed=5)
        assert np.array_equal(got, poisson_disk_indices(pts, radius, 5)), (name, frac)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_edge_cases_match_the_definition(pcu, dtype):
    f = pcu.downsample_point_cloud_poisson_disk
    # a lattice whose spacing is exactly r: neighbours at d2 == rr do not conflict (strict <), one ulp more and they do
    g = np.stack(np.meshgrid(np.arange(12), np.arange(10), np.arange(8), indexing="ij"), -1).reshape(-1, 3)
    lattice = (g * 0.25).astype(dtype)
    assert np.array_equal(f(lattice, 0.25, random_seed=3), np.arange(len(lattice)))
    above = float(np.nextafter(dtype(0.25), dtype(1)))
    got = f(lattice, above, random_seed=3)
    assert np.array_equal(got, poisson_disk_indices(lattice, above, 3)) and len(got) < len(lattice)
    # one row
    assert np.array_equal(f(np.ones((1, 3), dtype=dtype), 0.5, random_seed=3), [0])
    # every row the same point: the row of smallest key
    same = np.full((300, 3), 0.3, dtype=dtype)
    got = f(same, 0.01, random_seed=3)
    assert len(got) == 1 and np.array_equal(got, poisson_disk_indices(same, 0.01, 3))
    # a radius beyond the box diagonal: one sample
    pts = np.random.default_rng(12).random((5000, 3)).astype(dtype)
    got = f(pts, 2.0, random_seed=4)
    assert len(got) == 1 and np.array_equal(got, poisson_disk_indices(pts, 2.0, 4))
    # r * r underflows to 0: nothing conflicts, every row is a sample
    tiny = 1e-30 if dtype == np.float32 else 1e-170
    assert np.array_equal(f(pts, tiny, random_seed=4), np.arange(len(pts)))
    # a tight cluster: 40000 points in a 1e-4 cube, the radius a tenth of the cube
    cl = (0.5 + 1e-4 * np.random.default_rng(13).random((40000, 3))).astype(dtype)
    got = f(cl, 1e-5, random_seed=6)
    assert np.array_equal(got, poisson_disk_indices(cl, 1e-5, 6))


# ---- GPU: full size, checked with the library's exact k-NN ----------------------------------------------------------
def _sphere(rng, n):
    v = rng.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["uniform", "sphere"])
def test_full_size_is_separated_and_maximal(pcu, shape):
    import torch
    rng = np.random.default_rng(21)
    pts = rng.random((1000000, 3), dtype=np.float32) if shape == "uniform" else _sphere(rng, 1000000)
    radius = 0.02 if shape == "uniform" else 0.01
    rr = np.float32(np.float32(radius) * np.float32(radius))
    x = torch.from_numpy(pts).cuda()
    idx = pcu.downsample_point_cloud_poisson_disk(x, radius, random_seed=123)
    assert idx.dtype == torch.int32 and idx.is_cuda
    idx_h = idx.cpu().numpy()
    assert np.all(np.diff(idx_h) > 0) and 1000 < len(idx_h) < 1000000
    s = x[idx.long()].contiguous()
    d, _ = pcu.k_nearest_neighbors(s, s, 2, squared_distances=True)            # separation
    assert bool((d[:, 1] >= float(rr)).all())
    d1, _ = pcu.k_nearest_neighbors(x, s, 1, squared_distances=True)           # maximality
    is_sample = torch.zeros(len(pts), dtype=torch.bool, device=x.device)
    is_sample[idx.long()] = True
    assert bool(((d1.reshape(-1) < float(rr)) | is_sample).all())


# ---- GPU: determinism, input forms, seeds -------------------------------------------------------------------------
@pytest.mark.gpu
def test_determinism_and_input_forms(pcu):
    import torch
    f = pcu.downsample_point_cloud_poisson_disk
    pts = np.random.default_rng(31).random((30000, 3)).astype(np.float32)
    a = f(pts, 0.03, random_seed=9)
    assert a.dtype == np.int32 and np.all(np.diff(a) > 0)
    assert np.array_equal(a, f(pts, 0.03, random_seed=9))
    t = f(torch.from_numpy(pts).cuda(), 0.03, random_seed=9)
    assert t.is_cuda and t.dtype == torch.int32 and np.array_equal(t.cpu().numpy(), a)
    assert np.array_equal(f(pts, 0.03, random_seed=9, device=0), a)
    assert np.array_equal(f(pts, 0.03, -1, 9, 0.04, device="cuda:0"), a)           # positional order of the reference
    c = f(torch.from_numpy(pts), 0.03, random_seed=9)                               # CPU tensor -> CPU tensor
    assert isinstance(c, torch.Tensor) and not c.is_cuda and np.array_equal(c.numpy(), a)
    b = f(pts, 0.03, random_seed=10)
    assert not np.array_equal(a, b)
    assert np.array_equal(b, poisson_disk_indices(pts, 0.03, 10))                    # valid: it is the definition's set
    np.random.seed(1234)
    z1 = f(pts, 0.03)
    np.random.seed(1234)
    z2 = f(pts, 0.03)
    assert np.array_equal(z1, z2)


# ---- GPU: target mode -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_target_mode_matches_the_definition(pcu, dtype):
    pts = np.random.default_rng(41).random((20000, 3)).astype(dtype)
    for target in (500, 3000):
        got = pcu.downsample_point_cloud_poisson_disk(pts, 0.0, target_num_samples=target, random_seed=8)
        ref, radii, steps = target_mode(pts, target, 8)
        assert np.array_equal(got, ref)
        within = int(target * np.float32(0.96)) <= len(got) <= int(target * np.float32(1.04))
        assert within or steps == 20


@pytest.mark.gpu
def test_target_mode_on_identical_rows(pcu):
    same = np.full((200, 3), -2.0, dtype=np.float32)
    got = pcu.downsample_point_cloud_poisson_disk(same, 0.0, target_num_samples=10, random_seed=2)
    assert np.array_equal(got, target_mode(same, 10, 2)[0]) and len(got) == 1
    assert np.array_equal(pcu.downsample_point_cloud_poisson_disk(same, 0.0, target_num_samples=200), np.arange(200))
