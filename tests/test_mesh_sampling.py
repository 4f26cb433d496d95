"""Mesh sampling (sample_mesh_random, sample_mesh_poisson_disk; the reference's src/sample_mesh.cpp) and barycentric
interpolation (interpolate_barycentric_coords; point_cloud_utils/__init__.py:203-217).

The reference draws with std::rand and libigl, so the library defines its samples exactly (DESIGN.md §3,
csrc/meshsample.cuh) and this file restates those definitions with numpy: the GPU must match them bit for bit.  The
Poisson-disk stage is the point-cloud definition of test_poisson_disk.py."""
import inspect
import math

import numpy as np
import pytest
from scipy.stats import chi2

from meshes import icosphere
from test_poisson_disk import poisson_disk_indices

M32 = np.uint64(0xFFFFFFFF)


# ---- the definitions, restated -------------------------------------------------------------------------------------
def mix64(x):
    """splitmix64 with its +0x9E3779B97F4A7C15 step, on uint64 arrays (wrap-around arithmetic)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def sample_hash(seed, s, j):
    s = np.asarray(s, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return mix64(mix64(np.uint64(3) * s + np.uint64(j)) ^ np.uint64(seed))


def mulhi64(a, b):
    """High 64 bits of a * b for a uint64 array and a Python int, through 32-bit limbs."""
    a = np.asarray(a, dtype=np.uint64)
    b_hi, b_lo = np.uint64(b >> 32), np.uint64(b & 0xFFFFFFFF)
    a_hi, a_lo = a >> np.uint64(32), a & M32
    ll, lh, hl, hh = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (ll >> np.uint64(32)) + (lh & M32) + (hl & M32)
    return hh + (lh >> np.uint64(32)) + (hl >> np.uint64(32)) + (mid >> np.uint64(32))


def face_cdf(v, f):
    """(C, S, bad faces): A_f = |(b - a) x (c - a)| in fp64 rounded per operation, 0 when not finite or when a corner
    is outside [0, #v); S = 2^(62 - ceil(log2 m)) / max A; w = floor(A S); C = cumsum(w) (exact)."""
    nv, m = len(v), len(f)
    if f.dtype.kind == "u":
        bad = (f >= nv).any(axis=1)
    else:
        bad = ((f < 0) | (f >= nv)).any(axis=1)
    idx = np.where(bad[:, None], 0, f).astype(np.int64)
    a, b, c = (v[idx[:, k]].astype(np.float64) for k in range(3))
    e1, e2 = b - a, c - a
    nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    with np.errstate(over="ignore", invalid="ignore"):
        A = np.sqrt((nx * nx + ny * ny) + nz * nz)
    A[~np.isfinite(A) | bad] = 0.0
    k = (m - 1).bit_length()
    amax = float(A.max())
    with np.errstate(over="ignore", divide="ignore"):
        S = math.ldexp(1.0, 62 - k) / amax if amax > 0 else 0.0
    if not math.isfinite(S):
        S = 0.0
    w = np.floor(A * S).astype(np.uint64)
    return np.cumsum(w, dtype=np.uint64), S, int(bad.sum())


def dense_samples(v, f, n, seed, positions=False):
    """Samples 0 .. n-1: (face, bc rounded to v's dtype[, fp64 positions rounded to v's dtype])."""
    C, _, _ = face_cdf(v, f)
    W = int(C[-1])
    s = np.arange(n, dtype=np.uint64)
    fidx = np.searchsorted(C, mulhi64(sample_hash(seed, s, 0), W), side="right")      # first f with C_f > u
    u1 = (sample_hash(seed, s, 1) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    u2 = (sample_hash(seed, s, 2) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    a = np.sqrt(u1)
    bc64 = np.stack([1.0 - a, a * (1.0 - u2), a * u2], axis=1)
    T = v.dtype
    out = (fidx.astype(f.dtype), bc64.astype(T))
    if positions:
        corners = f[fidx].astype(np.int64)
        va, vb, vc = (v[corners[:, k]].astype(np.float64) for k in range(3))
        p = (bc64[:, :1] * va + bc64[:, 1:2] * vb) + bc64[:, 2:] * vc
        out = out + (p.astype(T),)
    return out


def dense_plan(C, S, num_samples, radius, oversampling_factor=40.0):
    total_area = float(int(C[-1])) / S / 2.0
    if radius <= 0.0 and num_samples > 0:
        radius = math.sqrt(total_area / (0.7 * math.pi * num_samples))
    n_est = float(num_samples) if num_samples > 0 else total_area / (0.7 * math.pi * (radius * radius))
    return radius, max(1, int(math.ceil(float(np.float32(oversampling_factor)) * n_est)))


def mesh_poisson(v, f, num_samples, radius, seed, oversampling_factor=40.0):
    C, S, _ = face_cdf(v, f)
    r, n_dense = dense_plan(C, S, num_samples, radius, oversampling_factor)
    fidx, bc, p = dense_samples(v, f, n_dense, seed, positions=True)
    keep = poisson_disk_indices(p, r, seed)
    return fidx[keep], bc[keep]


# ---- meshes, generated from seeds ---------------------------------------------------------------------------------
def flat_grid(n, dtype=np.float64):
    g = np.stack(np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([g / n, np.zeros((len(g), 1))], axis=1)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    i = i.reshape(-1)
    f = np.concatenate([np.stack([i, i + n + 1, i + 1], 1), np.stack([i + 1, i + n + 1, i + n + 2], 1)])
    return v.astype(dtype), f


def degenerate_mesh(dtype=np.float64):
    """Faces of zero area (a repeated corner) and collinear faces among ordinary ones."""
    v, f = flat_grid(6, dtype)
    zero = np.stack([f[:, 0], f[:, 0], f[:, 1]], 1)
    line = np.array([[0, 1, 2], [7, 8, 9], [0, 7, 14]])       # corners along one grid line / diagonal
    return v, np.concatenate([zero[:20], f[:30], line, zero[20:40], f[30:]])


def spanning_mesh(dtype=np.float64, seed=3):
    """Triangles whose areas span 10^6 : 1, unreferenced vertices between them."""
    rng = np.random.default_rng(seed)
    scales = np.geomspace(1e-3, 1.0, 40)        # areas 1e-6 .. 1
    vs, fs = [], []
    for i, s in enumerate(scales):
        base = rng.random(3) * 10
        tri = base + s * np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.3]])
        vs.append(np.concatenate([tri, rng.random((2, 3))]))         # two unreferenced vertices per triangle
        fs.append(5 * i + np.array([0, 1, 2]))
    return np.concatenate(vs).astype(dtype), np.stack(fs)


MESHES = {
    "icosphere": lambda dt: icosphere(3, 0.01, 1, dt),
    "grid": lambda dt: flat_grid(20, dt),
    "degenerate": degenerate_mesh,
    "single": lambda dt: (np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], dtype=dt), np.array([[0, 1, 2]])),
    "spanning": spanning_mesh,
}


# ---- CPU: interface, arguments, the definitions ------------------------------------------------------------------
def test_signatures(pcu):
    ps = list(inspect.signature(pcu.sample_mesh_random).parameters.values())
    assert [p.name for p in ps] == ["v", "f", "num_samples", "random_seed", "device"]
    assert ps[3].default == 0 and ps[4].kind == inspect.Parameter.KEYWORD_ONLY and ps[4].default is None
    ps = list(inspect.signature(pcu.sample_mesh_poisson_disk).parameters.values())
    assert [p.name for p in ps] == ["v", "f", "num_samples", "radius", "use_geodesic_distance", "best_choice_sampling",
                                    "random_seed", "sample_num_tolerance", "oversampling_factor", "device"]
    assert [p.default for p in ps[3:9]] == [0.0, True, True, 0, 0.04, 40.0]
    assert all(p.kind == inspect.Parameter.POSITIONAL_OR_KEYWORD for p in ps[:9])
    assert ps[9].kind == inspect.Parameter.KEYWORD_ONLY and ps[9].default is None
    ps = list(inspect.signature(pcu.interpolate_barycentric_coords).parameters.values())
    assert [p.name for p in ps] == ["f", "fi", "bc", "attribute", "device"]
    assert ps[4].kind == inspect.Parameter.KEYWORD_ONLY
    for name in ("sample_mesh_random", "sample_mesh_poisson_disk", "interpolate_barycentric_coords"):
        assert name in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    v, f = icosphere(1)
    rnd, pd = pcu.sample_mesh_random, pcu.sample_mesh_poisson_disk
    with pytest.raises(ValueError, match="num_samples must be positive"):
        rnd(v, f, 0)
    with pytest.raises(ValueError, match="num_samples must be positive"):
        rnd(v, f, -5)
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        rnd(v[:0], f, 10)
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        pd(v, f[:0], 10)
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        rnd(v[:, :2], f, 10)
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        pd(v, f[:, :2], 10)
    with pytest.raises(ValueError, match="scalar type"):
        rnd(v.astype(np.int32), f, 10)
    with pytest.raises(ValueError, match="scalar type"):
        pd(v, f.astype(np.uint32), 10)                     # the reference's Poisson binding takes int32 / int64 only
    with pytest.raises(ValueError, match="scalar type"):
        rnd(v, f.astype(np.float32), 10)
    with pytest.raises(ValueError, match="NumPy array"):
        rnd(v.tolist(), f, 10)
    with pytest.raises(ValueError, match=r"Cannot have both num_samples <= 0 and radius <= 0"):
        pd(v, f, 0)
    with pytest.raises(ValueError, match=r"Cannot have both num_samples <= 0 and radius <= 0"):
        pd(v, f, -1, radius=-2.0)
    with pytest.raises(ValueError, match=r"sample_num_tolerance must be in \(0, 1\]"):
        pd(v, f, 10, sample_num_tolerance=0.0)
    with pytest.raises(ValueError, match=r"sample_num_tolerance must be in \(0, 1\]"):
        pd(v, f, 10, sample_num_tolerance=1.5)
    with pytest.raises(ValueError, match="oversampling_factor"):
        pd(v, f, 10, oversampling_factor=0.5)
    interp = pcu.interpolate_barycentric_coords
    fi = np.array([0, 3, -1])
    bc = np.full((3, 3), 1.0 / 3.0)
    with pytest.raises(ValueError, match="attribute must have shape"):
        interp(f, fi, bc, v[:, 0])                         # 1-D attribute: a documented divergence
    with pytest.raises(ValueError, match="scalar type"):
        interp(f, fi.astype(np.float64), bc, v)
    with pytest.raises(ValueError, match="shapes"):
        interp(f, fi, bc[:2], v)
    with pytest.raises(IndexError):
        interp(f, np.array([0, len(f)]), bc[:2], v)         # face out of range
    with pytest.raises(IndexError):
        interp(f, np.array([-len(f) - 1]), bc[:1], v)
    bad_f = f.copy()
    bad_f[3, 1] = len(v)
    with pytest.raises(IndexError):
        interp(bad_f, np.array([3]), bc[:1], v)             # vertex out of range


def test_hash_literals():
    assert hex(int(mix64(0))) == "0xe220a8397b1dcdaf"
    assert hex(int(sample_hash(7, 0, 0))) == "0x64bf61b512ffabe7"
    assert [hex(int(x)) for x in sample_hash(12345, [0, 1, 1000003], 2)] == [
        hex(int(mix64(int(mix64(3 * s + 2)) ^ 12345))) for s in (0, 1, 1000003)]
    a = np.array([0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 12345], dtype=np.uint64)
    for b in (1, 0xFFFFFFFFFFFFFFFF, 0x123456789ABCDEF):
        assert [int(x) for x in mulhi64(a, b)] == [(int(x) * b) >> 64 for x in a]


def test_face_cdf_on_a_hand_computed_mesh():
    # twice the areas: 1 (legs 1, 1), 2 (legs 2, 1), 0 (a repeated corner), 0 (collinear)
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [3, 0, 0]], dtype=np.float32)
    f = np.array([[0, 1, 2], [0, 3, 2], [0, 0, 1], [0, 1, 4]], dtype=np.int32)
    C, S, bad = face_cdf(v, f)
    assert S == 2.0 ** 60 / 2.0 and bad == 0          # ceil(log2 4) = 2, max A = 2
    assert [int(c) for c in C] == [2 ** 59, 3 * 2 ** 59, 3 * 2 ** 59, 3 * 2 ** 59]
    assert float(int(C[-1])) / S / 2 == 1.5           # the total area
    f2 = np.array([[0, 1, 2], [0, 1, 5], [0, -1, 2]], dtype=np.int64)
    C, S, bad = face_cdf(v, f2)
    assert bad == 2 and [int(c) for c in C] == [2 ** 60] * 3
    # only faces of positive weight are ever drawn: u < W, first C_f > u
    fidx, bc = dense_samples(v, f, 20000, 9)
    assert set(np.unique(fidx)) == {0, 1}
    assert abs(np.mean(fidx == 1) - 2 / 3) < 0.02
    assert np.allclose(bc.sum(axis=1), 1.0, atol=1e-6) and (bc >= 0).all()


# ---- GPU: sample_mesh_random equals the definition -----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
@pytest.mark.parametrize("fdtype", [np.int32, np.int64, np.uint32, np.uint64])
def test_random_matches_the_definition(pcu, vdtype, fdtype):
    for name, make in MESHES.items():
        v, f = make(vdtype)
        f = f.astype(fdtype)
        got_f, got_bc = pcu.sample_mesh_random(v, f, 20000, random_seed=11)
        ref_f, ref_bc = dense_samples(v, f, 20000, 11)
        assert got_f.dtype == fdtype and got_bc.dtype == vdtype and got_bc.shape == (20000, 3), name
        assert np.array_equal(got_f, ref_f), name
        assert np.array_equal(got_bc.view(np.uint8), ref_bc.view(np.uint8)), name


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_random_full_size(pcu, vdtype):
    import torch
    v, f = icosphere(8, 1e-4, 5, vdtype)                 # 1 310 720 faces
    f = f.astype(np.int32)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    got_f, got_bc = pcu.sample_mesh_random(vt, ft, 10 ** 7, random_seed=2024)
    assert got_f.is_cuda and got_f.dtype == torch.int32 and got_bc.dtype == vt.dtype
    ref_f, ref_bc = dense_samples(v, f, 10 ** 7, 2024)
    assert np.array_equal(got_f.cpu().numpy(), ref_f)
    assert np.array_equal(got_bc.cpu().numpy().view(np.uint8), ref_bc.view(np.uint8))


@pytest.mark.gpu
def test_zero_area_faces_are_never_drawn(pcu):
    v, f = degenerate_mesh()
    C, _, _ = face_cdf(v, f)
    zero = np.nonzero(np.diff(np.concatenate([[0], C.astype(object)])) == 0)[0]
    assert len(zero) == 43
    got_f, _ = pcu.sample_mesh_random(v, f, 200000, random_seed=5)
    assert not np.isin(got_f, zero).any()


@pytest.mark.gpu
def test_determinism_seeds_and_input_forms(pcu):
    import torch
    v, f = icosphere(4, 0.02, 7, np.float32)
    a = pcu.sample_mesh_random(v, f, 50000, random_seed=3)
    b = pcu.sample_mesh_random(v, f, 50000, random_seed=3)
    c = pcu.sample_mesh_random(v, f, 50000, random_seed=4)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert not np.array_equal(a[0], c[0])
    assert isinstance(a[0], np.ndarray) and a[0].dtype == np.int64 and a[1].dtype == np.float32
    tc = pcu.sample_mesh_random(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), 50000, random_seed=3)
    assert all(t.is_cuda for t in tc) and tc[0].dtype == torch.int64 and tc[1].dtype == torch.float32
    assert np.array_equal(tc[0].cpu().numpy(), a[0]) and np.array_equal(tc[1].cpu().numpy(), a[1])
    cpu = pcu.sample_mesh_random(torch.from_numpy(v), torch.from_numpy(f), 50000, random_seed=3)
    assert all(isinstance(t, torch.Tensor) and not t.is_cuda for t in cpu)
    assert np.array_equal(cpu[0].numpy(), a[0]) and np.array_equal(cpu[1].numpy(), a[1])
    assert np.array_equal(pcu.sample_mesh_random(v, f, 50000, 3, device="cuda:0")[0], a[0])
    np.random.seed(77)
    z1 = pcu.sample_mesh_random(v, f, 1000)
    np.random.seed(77)
    z2 = pcu.sample_mesh_random(v, f, 1000)
    assert np.array_equal(z1[0], z2[0]) and np.array_equal(z1[1], z2[1])
    pd = pcu.sample_mesh_poisson_disk(v, f, 500, random_seed=3)
    pt = pcu.sample_mesh_poisson_disk(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), 500, random_seed=3)
    assert pd[0].dtype == np.int64 and pd[1].dtype == np.float32 and pt[0].is_cuda
    assert np.array_equal(pt[0].cpu().numpy(), pd[0]) and np.array_equal(pt[1].cpu().numpy(), pd[1])
    pc = pcu.sample_mesh_poisson_disk(torch.from_numpy(v), torch.from_numpy(f), 500, random_seed=3)
    assert not pc[0].is_cuda and np.array_equal(pc[0].numpy(), pd[0])


@pytest.mark.gpu
def test_face_counts_follow_the_areas(pcu):
    v, f = spanning_mesh()
    v, f = v.copy(), f.copy()
    f = f[20:]                                         # 20 faces, areas 1.6e-3 .. 1
    n = 4 * 10 ** 6
    got_f, _ = pcu.sample_mesh_random(v, f, n, random_seed=99)
    e1, e2 = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    area = np.linalg.norm(np.cross(e1, e2), axis=1)
    expected = n * area / area.sum()
    counts = np.bincount(got_f, minlength=len(f))
    stat = float(((counts - expected) ** 2 / expected).sum())
    assert stat < chi2.ppf(0.9999, len(f) - 1), stat


# ---- GPU: sample_mesh_poisson_disk equals the definition ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_poisson_matches_the_definition(pcu, vdtype):
    v, f = icosphere(4, 0.01, 2, vdtype)
    for num_samples, radius in ((2000, 0.0), (0, 0.06), (1000, 0.05)):   # the last: a positive radius wins
        got_f, got_bc = pcu.sample_mesh_poisson_disk(v, f, num_samples, radius=radius, random_seed=21)
        ref_f, ref_bc = mesh_poisson(v, f, num_samples, radius, 21)
        assert got_f.dtype == f.dtype and got_bc.dtype == vdtype
        assert 0 < len(got_f) and np.array_equal(got_f, ref_f), (num_samples, radius)
        assert np.array_equal(got_bc.view(np.uint8), ref_bc.view(np.uint8)), (num_samples, radius)
    v, f = flat_grid(30, vdtype)
    got = pcu.sample_mesh_poisson_disk(v, f.astype(np.int32), 3000, random_seed=8, oversampling_factor=50.0)
    ref = mesh_poisson(v, f.astype(np.int32), 3000, 0.0, 8, 50.0)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    assert got[0].dtype == np.int32


@pytest.mark.gpu
def test_poisson_full_size_is_the_point_cloud_sample(pcu):
    """4 * 10^6 dense points: the result is downsample_point_cloud_poisson_disk of the dense positions, which are
    separated and maximal (checked with the library's exact k-NN)."""
    import torch
    v, f = icosphere(6, 1e-3, 9, np.float32)
    seed, num_samples = 31, 10 ** 5
    C, S, _ = face_cdf(v, f)
    r, n_dense = dense_plan(C, S, num_samples, 0.0)
    assert n_dense == 4 * 10 ** 6
    got_f, got_bc = pcu.sample_mesh_poisson_disk(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), num_samples,
                                                 random_seed=seed)
    dense_f, dense_bc, p = dense_samples(v, f, n_dense, seed, positions=True)
    pt = torch.from_numpy(p).cuda()
    keep = pcu.downsample_point_cloud_poisson_disk(pt, r, random_seed=seed)
    kh = keep.cpu().numpy()
    assert np.array_equal(got_f.cpu().numpy(), dense_f[kh]) and np.array_equal(got_bc.cpu().numpy(), dense_bc[kh])
    assert 0.5 * num_samples < len(kh) < 2 * num_samples
    rr = float(np.float32(np.float32(r) * np.float32(r)))
    s = pt[keep.long()].contiguous()
    d, _ = pcu.k_nearest_neighbors(s, s, 2, squared_distances=True)
    assert bool((d[:, 1] >= rr).all())
    d1, _ = pcu.k_nearest_neighbors(pt, s, 1, squared_distances=True)
    is_kept = torch.zeros(n_dense, dtype=torch.bool, device=pt.device)
    is_kept[keep.long()] = True
    assert bool(((d1.reshape(-1) < rr) | is_kept).all())


@pytest.mark.gpu
def test_bad_meshes_raise_without_a_fault(pcu):
    v, f = flat_grid(4)
    flat = v.copy()
    flat[:, 1] = 0.0                                   # every face collinear: zero area
    with pytest.raises(ValueError, match="Mesh has zero area"):
        pcu.sample_mesh_random(flat, f, 100, random_seed=1)
    with pytest.raises(ValueError, match="Mesh has zero area"):
        pcu.sample_mesh_poisson_disk(flat, f, 100, random_seed=1)
    with pytest.raises(ValueError, match="Mesh has zero area"):
        pcu.sample_mesh_poisson_disk(flat, f, 0, radius=0.1, random_seed=1)
    for bad in (len(v), 10 ** 9, -1):
        g = f.copy()
        g[5, 2] = bad
        with pytest.raises(ValueError, match="outside"):
            pcu.sample_mesh_random(v, g, 100, random_seed=1)
        with pytest.raises(ValueError, match="outside"):
            pcu.sample_mesh_poisson_disk(v, g, 100, random_seed=1)
    g = f.astype(np.uint64)
    g[0, 0] = np.uint64(2 ** 64 - 1)
    with pytest.raises(ValueError, match="outside"):
        pcu.sample_mesh_random(v, g, 100, random_seed=1)
    ok_f, ok_bc = pcu.sample_mesh_random(v, f, 1000, random_seed=1)      # the device is fine afterwards
    ref_f, ref_bc = dense_samples(v, f, 1000, 1)
    assert np.array_equal(ok_f, ref_f) and np.array_equal(ok_bc, ref_bc)


# ---- GPU: interpolation ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("adtype", [np.float32, np.float64])
@pytest.mark.parametrize("bdtype", [np.float32, np.float64])
@pytest.mark.parametrize("idtype", [np.int32, np.int64, np.uint32, np.uint64])
def test_interpolation_is_the_reference_expression(pcu, adtype, bdtype, idtype):
    rng = np.random.default_rng(17)
    v, f = icosphere(3, 0.01, 4)
    fi = rng.integers(0, len(f), 50000)
    if np.dtype(idtype).kind == "i":
        fi = np.where(rng.random(len(fi)) < 0.3, fi - len(f), fi)          # negative indices wrap
    fi = fi.astype(idtype)
    ff = f.astype(idtype)
    bc = rng.random((len(fi), 3)).astype(bdtype)
    for dim in (1, 3, 7):
        attr = rng.standard_normal((len(v), dim)).astype(adtype)
        ref = (attr[ff[fi]] * bc[:, :, np.newaxis]).sum(1)
        got = pcu.interpolate_barycentric_coords(ff, fi, bc, attr)
        assert got.dtype == ref.dtype and got.shape == ref.shape
        assert np.array_equal(got.view(np.uint8), ref.view(np.uint8)), dim
    if np.dtype(idtype).kind == "i":
        fneg = np.where(rng.random(f.shape) < 0.3, f - len(v), f).astype(idtype)   # negative corners wrap too
        attr = rng.standard_normal((len(v), 3)).astype(adtype)
        got = pcu.interpolate_barycentric_coords(fneg, fi, bc, attr)
        assert np.array_equal(got, (attr[fneg[fi]] * bc[:, :, np.newaxis]).sum(1))


@pytest.mark.gpu
def test_interpolation_index_errors_and_forms(pcu):
    import torch
    v, f = icosphere(2)
    bc = np.full((4, 3), 1.0 / 3.0)
    attr = v.copy()
    fi = np.array([0, 1, 2, 3])
    ct = [torch.from_numpy(x).cuda() for x in (f, fi, bc, attr)]
    got = pcu.interpolate_barycentric_coords(*ct)
    assert got.is_cuda and got.dtype == torch.float64
    assert np.array_equal(got.cpu().numpy(), (attr[f[fi]] * bc[:, :, None]).sum(1))
    cpu = pcu.interpolate_barycentric_coords(*[torch.from_numpy(x) for x in (f, fi, bc, attr)])
    assert not cpu.is_cuda and np.array_equal(cpu.numpy(), got.cpu().numpy())
    with pytest.raises(IndexError):
        pcu.interpolate_barycentric_coords(ct[0], torch.tensor([0, len(f), 1, 2], device="cuda"), ct[2], ct[3])
    g = f.copy()
    g[2, 1] = -len(v) - 1
    with pytest.raises(IndexError):
        pcu.interpolate_barycentric_coords(torch.from_numpy(g).cuda(), ct[1], ct[2], ct[3])
    assert np.array_equal(pcu.interpolate_barycentric_coords(*ct).cpu().numpy(), got.cpu().numpy())


# ---- GPU: the whole pipeline on CUDA tensors ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_sample_interpolate_chamfer_end_to_end(pcu, oracle):
    import torch
    va, fa = icosphere(5, 0.0, 0, np.float32)
    vb, fb = icosphere(5, 0.01, 6, np.float32)
    ta, tfa, tb, tfb = (torch.from_numpy(x).cuda() for x in (va, fa, vb, fb))
    fia, bca = pcu.sample_mesh_random(ta, tfa, 200000, random_seed=1)
    fib, bcb = pcu.sample_mesh_poisson_disk(tb, tfb, 20000, random_seed=2)
    pa = pcu.interpolate_barycentric_coords(tfa, fia, bca, ta)
    pb = pcu.interpolate_barycentric_coords(tfb, fib, bcb, tb)
    assert pa.is_cuda and pa.dtype == torch.float32 and pa.shape == (200000, 3)
    c = pcu.chamfer_distance(pa, pb)
    a, b = pa.cpu().numpy(), pb.cpu().numpy()
    assert np.array_equal(a, (va[fa[fia.cpu().numpy()]] * bca.cpu().numpy()[:, :, None]).sum(1))
    ref = float(oracle.chamfer_distance(a, b))
    assert abs(float(c) - ref) <= 1e-5 * ref
