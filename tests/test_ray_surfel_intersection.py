"""ray_surfel_intersection, RaySurfelIntersector and pointcloud_surfel_geometry: the surfel fan of DESIGN.md §3 restated
op by op with numpy and self-checked; on the GPU, the geometry and the casts bit for bit against the restatement (the
casts through the ray-mesh restatement of test_ray_mesh_intersection), against the materialized route, the handle
against the function, edge cases and full size."""
import inspect
import math

import numpy as np
import pytest

from meshes import to_numpy
from test_closest_points import assert_bits
from test_ray_mesh_intersection import _as, ray_sets, restate

F32 = np.float32
SUBDIVS = [4, 5, 7, 16]


# ---- the restatement -----------------------------------------------------------------------------------------------
def table(s):
    """(c_j, s_j) = fl32(cos / sin of the reference's fp32 angle), from the C library in fp64."""
    den = F32(F32(s + 1) - F32(1))
    th = [float(F32(F32(F32(j) / den) * F32(math.pi)) * F32(2)) for j in range(s)]
    return np.array([math.cos(x) for x in th], F32), np.array([math.sin(x) for x in th], F32)


def _unit(a):
    return a / np.sqrt((a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2])[:, None]


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def fan(p, n, r, s, compute):
    """(vertices (N, s + 1, 3) in `compute`: rim 0 .. s - 1 then the centre; faces ((s N, 3) int64)) for points p,
    normals n and radii r (all in p's dtype T), every op rounded on its own."""
    T, C = p.dtype.type, np.dtype(compute).type
    cs, sn = table(s)
    with np.errstate(all="ignore"):
        nh = _unit(n.astype(C))
        c = p.astype(C)
        dot = (C(0) * nh[:, 0] + C(1) * nh[:, 1]) + C(0) * nh[:, 2]
        near_y = np.abs(np.abs(dot).astype(np.float64) - 1.0) < 1e-5
        axis = np.where(near_y[:, None], np.array([1, 0, 0], C), np.array([0, 1, 0], C))
        right = _unit(_cross(nh, axis))
        up = _unit(_cross(nh, right))
        x0 = (r.astype(T)[:, None] * cs.astype(T)[None, :]).astype(F32).astype(C)
        y0 = (r.astype(T)[:, None] * sn.astype(T)[None, :]).astype(F32).astype(C)
        rim = np.stack([((right[:, k, None] * x0 + up[:, k, None] * y0) + nh[:, k, None] * C(0)) + c[:, k, None]
                        for k in range(3)], -1)
    v = np.concatenate([rim, c[:, None, :]], 1)
    i = np.arange(len(p))[:, None] * (s + 1)
    j = np.arange(s)[None, :]
    f = np.stack([np.broadcast_to(i + s, (len(p), s)), i + j, i + (j + 1) % s], -1).reshape(-1, 3)
    return v, f


def restate_surfels(p, n, r, s, o, d, near=0.0, far=np.inf):
    """(pid, t) by the definition: the fp32 fans of the finite surfels through the ray-mesh restatement, pid = fid // s."""
    v, f = fan(p, n, r, s, F32)
    finite = np.isfinite(v).all((1, 2))
    keep = np.repeat(finite, s)
    fid_of = np.nonzero(keep)[0]
    d = np.asarray(d).reshape(-1, 3)
    if not keep.any():
        return np.full(len(d), -1, np.int64), np.full(len(d), np.inf, F32)
    fid, _, _, t = restate(o, d, v.reshape(-1, 3), f[keep], near, far)
    pid = np.where(fid >= 0, fid_of[np.maximum(fid, 0)] // s, -1)
    return pid, t


def cloud(seed, m=48, dtype=np.float64):
    """Points on a jittered grid with random normals, some exactly along +-y and just inside / outside the 1e-5 test."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(3), indexing="ij"), -1).reshape(-1, 3)[:m]
    p = g * 0.5 + 0.05 * rng.standard_normal((m, 3))
    n = rng.standard_normal((m, 3))
    n[0], n[1], n[2] = [0, 1, 0], [0, -2, 0], [1e-3, 1, 0]                 # on the +-y axis, just inside the band
    ny = 1 - 2e-5
    n[3] = [0, ny, np.sqrt(1 - ny * ny)]                                    # just outside it
    r = 0.2 + 0.1 * rng.random(m)
    return p.astype(dtype), n.astype(dtype), r.astype(dtype)


def surfel_rays(p, n, v, seed):
    """ray_sets of the fan mesh, plus rays at the centres, rim vertices and spoke midpoints from both sides."""
    s = v.shape[1] - 1
    flat = v.reshape(-1, 3).astype(np.float64)
    f = fan(p[:1], n[:1], np.ones(1, p.dtype), s, F32)[1]
    faces = (np.arange(len(p))[:, None, None] * (s + 1) + f[None]).reshape(-1, 3)
    finite = np.isfinite(flat).all(1)
    sets = ray_sets(flat[finite] if finite.any() else np.zeros((1, 3)), _finite_faces(flat, faces), seed)
    rng = np.random.default_rng(seed)
    vv = v.astype(np.float64)
    targets = np.concatenate([vv[:, s], vv[:, 0], vv[:, s // 2], 0.5 * (vv[:, s] + vv[:, 1])])
    nn = np.concatenate([n] * 4).astype(np.float64)
    nn /= np.maximum(np.linalg.norm(nn, axis=1, keepdims=True), 1e-300)
    for side in (1.0, -1.0):
        o = targets + side * 1.5 * nn + 0.2 * rng.standard_normal(targets.shape)
        ok = np.isfinite(o).all(1) & np.isfinite(targets).all(1)
        sets.append(("aimed %+d" % side, o[ok], targets[ok] - o[ok]))
    return sets


def _finite_faces(flat, faces):
    ok = np.isfinite(flat[faces]).all((1, 2))
    if not ok.any():
        return np.zeros((1, 3), np.int64)
    # remap to the finite vertex list
    keep = np.isfinite(flat).all(1)
    remap = np.cumsum(keep) - 1
    return remap[faces[ok]]


# ---- CPU: the restatement checks itself ------------------------------------------------------------------------------
@pytest.mark.parametrize("s", SUBDIVS)
def test_fan_lies_on_the_disk(s):
    p, n, r = cloud(1, dtype=np.float32)
    v, f = fan(p, n, r, s, F32)
    rim = v[:, :s].astype(np.float64) - p[:, None, :].astype(np.float64)
    nh = n / np.linalg.norm(n.astype(np.float64), axis=1, keepdims=True)
    # each coordinate carries at most a few fp32 roundings of magnitude |p| + r: bound them by 8 ulp of that
    scale = (np.abs(p).max(1) + r).astype(np.float64)[:, None]
    eps = 8 * 2.0 ** -23 * scale
    assert (np.abs(np.linalg.norm(rim, axis=2) - r[:, None]) <= 4 * eps).all()
    assert (np.abs((rim * nh[:, None, :]).sum(2)) <= 4 * eps).all()
    assert np.array_equal(v[:, s], p)
    # the faces: (centre, rim j, rim (j + 1) % s) of each point's own block of s + 1 vertices
    assert f.shape == (len(p) * s, 3)
    i = np.arange(len(p) * s) // s
    j = np.arange(len(p) * s) % s
    assert np.array_equal(f[:, 0], i * (s + 1) + s)
    assert np.array_equal(f[:, 1], i * (s + 1) + j)
    assert np.array_equal(f[:, 2], i * (s + 1) + (j + 1) % s)


def test_basis_branches():
    # n^_y = 1 - 2^-24 is within 1e-5 of 1: right = n^ x e_x; 1 - 2e-5 is outside: right = n^ x e_y
    for ny, along_x in ((1.0, True), (1 - 2.0 ** -24, True), (1 - 9e-6, True), (1 - 2e-5, False), (0.5, False)):
        nz = math.sqrt(max(0.0, 1 - ny * ny))
        n = np.array([[0.0, ny, nz]], F32)
        v, _ = fan(np.zeros((1, 3), F32), n, np.ones(1, F32), 4, F32)
        nh = _unit(n)
        expect = _unit(_cross(nh, np.array([[1, 0, 0]] if along_x else [[0, 1, 0]], F32)))
        # rim 0 sits at angle 0: right * fl32(r cos 0) = right
        assert np.array_equal(v[0, 0], ((expect[0] * F32(1) + _unit(_cross(nh, expect))[0] * F32(0)) + nh[0] * F32(0)) + F32(0)), ny


def test_table_matches_the_angles():
    c, s = table(7)
    assert c[0] == 1 and s[0] == 0 and c.dtype == F32
    th = 2 * np.pi * np.arange(7) / 7
    assert np.allclose(c, np.cos(th), atol=1e-6) and np.allclose(s, np.sin(th), atol=1e-6)


def test_restatement_picks_the_nearest_and_lowest():
    p = np.array([[0, 0, 0], [0, 0, 1], [0, 0, 0]], F32)
    n = np.array([[0, 0, 1]] * 3, F32)
    pid, t = restate_surfels(p, n, np.ones(3, F32), 7, np.array([0.1, 0.1, 5], F32), np.array([[0, 0, -1]], F32))
    assert pid[0] == 1 and t[0] == 4
    pid, t = restate_surfels(p, n, np.ones(3, F32), 7, np.array([0.1, 0.1, -5], F32), np.array([[0, 0, 1]], F32))
    assert pid[0] == 0 and abs(t[0] - 5) < 1e-5     # surfels 0 and 2 are identical: the lower id


# ---- CPU: interface --------------------------------------------------------------------------------------------------
def test_signatures(pcu):
    ps = list(inspect.signature(pcu.ray_surfel_intersection).parameters.values())
    assert [q.name for q in ps] == ["p", "n", "ray_o", "ray_d", "r", "subdivs", "ray_near", "ray_far", "device"]
    assert ps[4].default == 0.1 and ps[5].default == 4 and ps[6].default == 0.0 and ps[7].default == np.inf
    assert ps[8].kind == inspect.Parameter.KEYWORD_ONLY
    ps = list(inspect.signature(pcu.RaySurfelIntersector).parameters.values())
    assert [q.name for q in ps] == ["p", "n", "r", "subdivs", "device"] and ps[2].default == 0.1 and ps[3].default == 7
    ps = list(inspect.signature(pcu.RaySurfelIntersector.intersect_rays).parameters.values())
    assert [q.name for q in ps] == ["self", "ray_o", "ray_d", "ray_near", "ray_far"]
    ps = list(inspect.signature(pcu.pointcloud_surfel_geometry).parameters.values())
    assert [q.name for q in ps] == ["p", "n", "r", "subdivs", "device"] and ps[2].default == 0.1 and ps[3].default == 7
    for name in ("ray_surfel_intersection", "RaySurfelIntersector", "pointcloud_surfel_geometry"):
        assert name in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    p, n, r = cloud(2)
    o, d = np.zeros((4, 3)), np.ones((4, 3))
    calls = [lambda *a, **k: pcu.ray_surfel_intersection(a[0], a[1], o, d, *a[2:], **k),
             lambda *a, **k: pcu.RaySurfelIntersector(*a, **k),
             lambda *a, **k: pcu.pointcloud_surfel_geometry(*a, **k)]
    for call in calls:
        with pytest.raises(ValueError, match="Argument r must be a scalar or numpy array"):
            call(p, n, {"r": 1})
        with pytest.raises(ValueError, match="Argument r have the same number of rows as p"):
            call(p, n, r[:3])
        with pytest.raises(ValueError, match=r"Invalid shape for argument r, must have shape \(N,\) or \(N, 1\)"):
            call(p, n, np.ones((len(p), 2)))
        with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'v'"):
            call(p.astype(np.int32), n, 0.1)
        with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'n'. Expected it to match"):
            call(p, n.astype(F32), 0.1)
        with pytest.raises(ValueError, match=r"Only 3D inputs are supported: v must have shape \(n, 3\)"):
            call(p[:, :2], n, 0.1)
        with pytest.raises(ValueError, match=r"Invalid shape for normals: must have shape \(n, 3\)"):
            call(p, n[:, :2], 0.1)
        with pytest.raises(ValueError, match="Number of normals must match number of points"):
            call(p, n[:5], 0.1)
        with pytest.raises(ValueError, match="Invalid geometry_subdivisions_1 is less than or equal to 4."):
            call(p, n, 0.1, 3)
    rs = pcu.ray_surfel_intersection
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'ray_o'. Expected it to match argument 'v'"):
        rs(p, n, o.astype(F32), d)
    with pytest.raises(ValueError, match="ray_o and ray_d must have the same number of rows"):
        rs(p, n, o[:2], d)
    with pytest.raises(ValueError, match=r"Invalid shape for ray_d must have shape \(N, 3\) but got \(4, 2\)."):
        rs(p, n, o, d[:, :2])
    with pytest.raises(ValueError, match="NumPy array"):
        rs(p, n, o.tolist(), d)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _forms(pcu, form, *xs):
    import torch
    if form == "numpy":
        return xs
    ts = [torch.from_numpy(np.ascontiguousarray(x)) for x in xs]
    return [t.cuda() for t in ts] if form == "cuda" else ts


def _r_form(r, k):
    return [float(r[0]), r, r[:, None], list(r)][k % 4]


def _r_value(r, k, dtype):
    """The radii the library works with for form k, in p's dtype."""
    return np.full(len(r), float(r[0])).astype(dtype) if k % 4 == 0 else np.asarray(r).astype(dtype)


def _assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, what
    both_nan = np.isnan(a) & np.isnan(b) if a.dtype.kind == "f" else np.zeros(a.shape, bool)
    bits = a.view(np.uint32 if a.itemsize == 4 else np.uint64) == b.view(np.uint32 if b.itemsize == 4 else np.uint64)
    assert (bits | both_nan).all(), what


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", SUBDIVS)
def test_geometry_matches_the_restatement(pcu, dtype, s):
    p, n, r = cloud(3 + s, dtype=dtype)
    n[5] = 0                                      # a zero normal: NaN fan, written as computed
    for k, form in enumerate(("numpy", "cuda", "cpu", "numpy")):
        pf, nf = _forms(pcu, form, p, n)
        v, f = pcu.pointcloud_surfel_geometry(pf, nf, _r_form(r, k), s)
        ev, ef = fan(p, n, _r_value(r, k, dtype), s, dtype)
        ev = ev.reshape(-1, 3)[np.concatenate([np.arange(len(p))[:, None] * (s + 1) + np.arange(s + 1)]).ravel()]
        assert type(v) is type(pf) or form != "numpy"
        _assert_same(to_numpy(v), ev.astype(dtype), "%s %s v" % (form, k))
        assert to_numpy(f).dtype == np.int32 and np.array_equal(to_numpy(f), ef), form


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", SUBDIVS)
def test_casts_match_the_restatement(pcu, dtype, s):
    p, n, r = cloud(7 + s, dtype=dtype)
    v, _ = fan(p, n, r, s, F32)
    isect = pcu.RaySurfelIntersector(p, n, r, s)
    other = np.float64 if dtype == np.float32 else np.float32
    for k, (name, o, d) in enumerate(surfel_rays(p, n, v, s)):
        o, d = _as(dtype, o, d)
        for near, far in ((0.0, np.inf), (0.5, np.inf), (0.0, 2.0)):
            epid, et = restate_surfels(p, n, r, s, o, d, near, far)
            form = ("numpy", "cuda", "cpu")[k % 3]
            args = _forms(pcu, form, p, n, o, d)
            pid, t = pcu.ray_surfel_intersection(*args, _r_form(r, k) if k % 4 != 0 else r, s, near, far)
            pid, t = to_numpy(pid), to_numpy(t)
            what = "%s %s %s" % (name, form, (near, far))
            assert pid.dtype == np.int32 and np.array_equal(pid, epid), what
            assert_bits(t, et.astype(dtype), what + " t")
            hp, ht = isect.intersect_rays(o, d, near, far)
            assert np.array_equal(hp, pid) and assert_bits(ht, t, what + " handle") is None
            hp, ht = isect.intersect_rays(o.astype(other), d.astype(other), near, far)
            assert np.array_equal(hp, pid) and ht.dtype == other, what
            assert_bits(ht, et.astype(other), what + " handle, other precision")
    isect.close()
    with pytest.raises(ValueError, match="has been closed"):
        isect.intersect_rays(o, d)


@pytest.mark.gpu
@pytest.mark.parametrize("s", SUBDIVS)
def test_fp32_equals_the_materialized_route(pcu, s):
    p, n, r = cloud(20 + s, dtype=F32)
    v, f = pcu.pointcloud_surfel_geometry(p, n, r, s)
    fan_v = fan(p, n, r, s, F32)[0]
    for name, o, d in surfel_rays(p, n, fan_v, 30 + s):
        o, d = _as(F32, o, d)
        pid, t = pcu.ray_surfel_intersection(p, n, o, d, r, s)
        fid, _, mt = pcu.ray_mesh_intersection(v, f, o, d)
        assert np.array_equal(pid, np.where(fid >= 0, fid // s, -1)), name
        assert_bits(t, mt, name + " t")


@pytest.mark.gpu
def test_edge_cases(pcu):
    p = np.array([[0, 0, 0], [0, 0, 1], [0, 0, 0], [3, 0, 0], [6, 0, 0], [9, 0, 0], [12, 0, 0], [15, 0, 0]], F32)
    n = np.array([[0, 0, 1]] * 8, F32)
    r = np.ones(8, F32)
    n[3] = 0                        # zero normal
    n[4] = [np.nan, 0, 1]           # non-finite normal
    p[5, 0] = np.inf                # non-finite point
    r[6] = np.nan                   # non-finite radius
    r[7] = -1                       # negative radius: a mirrored disk, still hit
    xs = np.array([0.1, 3.1, 6.1, 9.1, 12.1, 15.1], F32)
    o = np.stack([xs, np.full(6, 0.1, F32), np.full(6, 5, F32)], 1)
    d = np.tile(np.array([[0, 0, -1]], F32), (6, 1))
    pid, t = pcu.ray_surfel_intersection(p, n, o, d, r, 7)
    assert list(pid) == [1, -1, -1, -1, -1, 7] and abs(t[0] - 4) < 1e-5 and abs(t[5] - 5) < 1e-5 and np.isinf(t[1:5]).all()
    epid, et = restate_surfels(p, n, r, 7, o, d)
    assert np.array_equal(pid, epid) and np.array_equal(t, et)
    # stacked identical surfels 0 and 2, seen from below: the lowest pid
    pid, t = pcu.ray_surfel_intersection(p, n, np.array([0.1, 0.1, -5], F32), np.array([[0, 0, 1]], F32), r, 7)
    assert pid[0] == 0 and abs(t[0] - 5) < 1e-5
    # r = 0: degenerate fans never hit
    pid, _ = pcu.ray_surfel_intersection(p, n, o, d, 0.0, 7)
    assert (pid == -1).all()
    # near exclusive, far inclusive at exact t = 4
    one_o, one_d = o[:1], d[:1]
    assert pcu.ray_surfel_intersection(p, n, one_o, one_d, r, 7, 4.0)[0][0] == 0       # t = 4 excluded: surfel 0 at t = 5
    assert pcu.ray_surfel_intersection(p, n, one_o, one_d, r, 7, 0.0, 4.0)[0][0] == 1
    assert pcu.ray_surfel_intersection(p, n, one_o, one_d, r, 7, 0.0, 3.99)[0][0] == -1
    # no points: every ray misses; no rays: empty outputs
    pid, t = pcu.ray_surfel_intersection(p[:0], n[:0], o, d, 0.1, 7)
    assert (pid == -1).all() and np.isinf(t).all() and pid.dtype == np.int32 and t.dtype == F32
    isect = pcu.RaySurfelIntersector(p[:0], n[:0])
    assert (isect.intersect_rays(o, d)[0] == -1).all()
    isect.close()
    before = pcu.launch_count()
    pid, t = pcu.ray_surfel_intersection(p, n, np.zeros((0, 3), F32), np.zeros((0, 3), F32), r, 7)
    assert pid.shape == (0,) and t.shape == (0,) and pcu.launch_count() == before
    v, f = pcu.pointcloud_surfel_geometry(p[:0], n[:0])
    assert v.shape == (0, 3) and f.shape == (0, 3) and f.dtype == np.int32
    # a single origin of shape (3,) or (1, 3): its elements in order
    a = pcu.ray_surfel_intersection(p, n, o[0], d, r, 7)
    b = pcu.ray_surfel_intersection(p, n, o[:1], d, r, 7)
    c = pcu.ray_surfel_intersection(p, n, np.repeat(o[:1], 6, 0), d, r, 7)
    for x, y in ((a, c), (b, c)):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])


@pytest.mark.gpu
def test_handle_after_many_calls(pcu):
    import torch
    p, n, r = cloud(40, dtype=F32)
    isect = pcu.RaySurfelIntersector(torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda(), r, 7)
    assert isect.num_subdivs == 7 and isect.r is r
    v = fan(p, n, r, 7, F32)[0]
    sets = surfel_rays(p, n, v, 41)
    o = np.concatenate([x[1] for x in sets]).astype(F32)
    d = np.concatenate([x[2] for x in sets]).astype(F32)
    ref = pcu.ray_surfel_intersection(p, n, o, d, r, 7)
    for _ in range(20):
        got = isect.intersect_rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda())
        assert got[0].is_cuda and np.array_equal(got[0].cpu().numpy(), ref[0]) and np.array_equal(got[1].cpu().numpy(), ref[1])
    isect.close()


@pytest.mark.gpu
def test_full_size(pcu):
    import torch
    rng = np.random.default_rng(5)
    m = 10 ** 6
    p = rng.standard_normal((m, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    n = (p + 0.3 * rng.standard_normal((m, 3))).astype(F32)
    p = p.astype(F32)
    r = F32(0.004)
    o = (rng.standard_normal((m, 3)) * 2).astype(F32)
    d = (rng.standard_normal((m, 3)) * 0.3 - o).astype(F32)
    pt, nt, ot, dt = (torch.from_numpy(x).cuda() for x in (p, n, o, d))
    pid, t = pcu.ray_surfel_intersection(pt, nt, ot, dt, r, 7)
    assert (pid >= 0).float().mean() > 0.3
    v, f = pcu.pointcloud_surfel_geometry(pt, nt, r, 7)
    mesh = pcu.RayMeshIntersector(v, f)
    fid, _, mt = mesh.intersect_rays(ot, dt)
    mesh.close()
    assert torch.equal(pid, torch.where(fid >= 0, fid // 7, fid)) and torch.equal(t, mt)
    # the restatement over the whole cloud (every fan, on the GPU through torch) for a subset of the rays
    fv, ff = fan(p, n, np.full(m, r, F32), 7, F32)
    assert np.isfinite(fv).all()
    rows = torch.from_numpy(rng.choice(m, 200, replace=False)).cuda()
    efid, _, _, et = restate(ot[rows], dt[rows], torch.from_numpy(fv.reshape(-1, 3)).cuda(), torch.from_numpy(ff).cuda(), chunk=1)
    assert torch.equal(pid[rows].long(), torch.where(efid >= 0, efid // 7, efid)) and torch.equal(t[rows], et)
    assert (efid >= 0).any()
