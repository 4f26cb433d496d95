"""estimate_point_cloud_areas (DESIGN.md §3, point areas).

The rules, restated here with numpy for one row r of the (#p, k) index array i:
  1. Neighbours: x_j = p[i[r, j]] in fp64.  Column j is kept iff n0x njx + n0y njy + n0z njz > 0 (fp64, left to right),
     n0 = n[i[r, 0]].  K = the kept columns in column order.  The area is 0 unless column 0 is kept and |K| >= 3.
  2. Plane: the offsets x_j - mean(x_K) on the two right singular vectors of the largest singular values of the offsets
     (the kernel takes them from PlaneFit, which computes the same plane to its stated bound): q_j in 2-D.
  3. Star of c = q_0: candidates are the kept columns j >= 1 with q_j != c exactly.  The walk starts at j0, the candidate
     nearest c (ties: lowest column).  From edge c -> q_j the next vertex is the candidate r with orient(c, q_j, q_r) > 0
     whose circumcentre of (c, q_j, q_r) lies least far along the left normal of c -> q_j, i.e. the least
     t = (|b|^2 - a.b) / (2 a x b) with a = q_j - c, b = q_r - c (ties: lowest column); each step adds (c, q_j, q_r).  It
     stops on returning to j0, when no candidate lies strictly left, or after |K| steps.  When it did not return to j0,
     the mirrored walk runs right from j0, adding (c, q_r, q_j).
  4. Area: per counter-clockwise triangle (X = c, Y, Z), with dX = (Y-X).(Z-X), dY = (X-Y).(Z-Y), dZ = (X-Z).(Y-Z) and
     cr = orient(X, Y, Z): (|Y-X|^2 dZ + |Z-X|^2 dY) / (8 cr) when dX, dY, dZ >= 0, else cr / 4 when dX < 0, else cr / 8;
     summed in walk order and rounded once to p's dtype.
On the CPU the restatement is pinned to scipy's Delaunay star on general-position clouds, to the analytic areas of
lattices and to the rules where a row gives 0; on the GPU the kernel is checked against it."""
import inspect
import math

import numpy as np
import pytest
from scipy.spatial import Delaunay, cKDTree

from meshes import to_form, to_numpy, torus
from test_point_cloud_winding_numbers import PUBLIC_TOL, pwn_device

KS = [1, 2, 3, 8, 16, 32, 33, 64, 256]
KINDS = ["int32", "int64", "uint32", "uint64"]
FORMS = ["numpy", "cpu", "cuda"]


# ---- the restatement ------------------------------------------------------------------------------------------------
def _mixed(y, z):
    """Meyer's mixed area at X of the counter-clockwise triangle (X, Y, Z), from y = Y - X and z = Z - X."""
    cr = y[0] * z[1] - y[1] * z[0]
    dX = y[0] * z[0] + y[1] * z[1]
    dY = -y[0] * (z[0] - y[0]) + -y[1] * (z[1] - y[1])
    dZ = -z[0] * (y[0] - z[0]) + -z[1] * (y[1] - z[1])
    if dX >= 0 and dY >= 0 and dZ >= 0:
        return ((y[0] * y[0] + y[1] * y[1]) * dZ + (z[0] * z[0] + z[1] * z[1]) * dY) / (8 * cr)
    return cr / 4 if dX < 0 else cr / 8


def star_area(q):
    """Rules 3 and 4 on the projected kept points q (m, 2), q[0] the centre."""
    m = len(q)
    d = q - q[0]
    cand = ~((d[:, 0] == 0) & (d[:, 1] == 0))
    if not cand.any():
        return 0.0
    d2 = np.where(cand, d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1], np.inf)
    j0 = int(np.argmin(d2))
    total = 0.0
    for side in (1.0, -1.0):
        cur = j0
        for _ in range(m):
            a = d[cur]
            o = side * (a[0] * d[:, 1] - a[1] * d[:, 0])
            ok = cand & (o > 0)
            if not ok.any():
                break
            with np.errstate(divide="ignore", invalid="ignore"):
                t = np.where(ok, ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) - (a[0] * d[:, 0] + a[1] * d[:, 1])) / (2 * o), np.inf)
            r = int(np.argmin(t))
            y, z = (cur, r) if side > 0 else (r, cur)
            total += _mixed(d[y], d[z])
            cur = r
            if r == j0:
                return total
    return total


def project(P, N, row):
    """Rules 1 and 2: the kept points of one row projected onto their plane (None when the area is 0 by rule 1)."""
    if len(row) == 0:
        return None
    nr = N[row]
    keep = nr[:, 0] * nr[0, 0] + nr[:, 1] * nr[0, 1] + nr[:, 2] * nr[0, 2] > 0
    if not keep[0] or keep.sum() <= 2:
        return None
    x = P[row[keep]]
    off = x - x.mean(0)
    _, _, vt = np.linalg.svd(off)
    return off @ vt[:2].T


def areas_ref(p, i, n, rows=None):
    """The restated areas of the given rows (all by default) in fp64; i (#p, k) or (#p,)."""
    P, N = np.asarray(p, np.float64), np.asarray(n, np.float64)
    I = np.asarray(i).reshape(len(P), -1).astype(np.int64)
    rows = range(len(P)) if rows is None else rows
    out = []
    for r in rows:
        q = project(P, N, I[r])
        out.append(0.0 if q is None else star_area(q))
    return np.array(out)


def delaunay_area(q):
    """The centre's mixed area over its star in scipy's Delaunay triangulation of q."""
    if q is None:
        return 0.0
    total = 0.0
    for f in Delaunay(q).simplices:
        if 0 in f:
            f = list(f)
            x = f.index(0)
            y, z = f[(x + 1) % 3], f[(x + 2) % 3]
            dy, dz = q[y] - q[0], q[z] - q[0]
            if dy[0] * dz[1] - dy[1] * dz[0] < 0:
                dy, dz = dz, dy
            total += _mixed(dy, dz)
    return total


# ---- clouds ---------------------------------------------------------------------------------------------------------
def fibonacci_sphere(m, jitter=0.0, seed=0):
    """m points on the unit sphere (a Fibonacci lattice, optionally jittered along the sphere) and their radial normals."""
    g = np.arange(m) + 0.5
    phi = np.arccos(1 - 2 * g / m)
    th = np.pi * (1 + 5 ** 0.5) * g
    p = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    if jitter:
        p = p + jitter * np.random.default_rng(seed).standard_normal(p.shape)
        p /= np.linalg.norm(p, axis=1, keepdims=True)
    return p, p.copy()


def torus_cloud(nu=60, nv=30, jitter=2e-3, seed=1):
    """The vertices of meshes.torus, jittered off its grid, and the torus's normals at the unjittered positions."""
    v, _ = torus(nu, nv)
    ring = v.copy()
    ring[:, 2] = 0
    ring = ring / np.linalg.norm(ring, axis=1, keepdims=True)
    nrm = v - ring
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return v + jitter * np.random.default_rng(seed).standard_normal(v.shape), nrm


def height_field(m=3000, seed=2):
    """Random points under z = 0.3 sin(2x) cos(3y) + noise, with the normals of the smooth surface."""
    rng = np.random.default_rng(seed)
    x, y = rng.random(m) * 2 - 1, rng.random(m) * 2 - 1
    z = 0.3 * np.sin(2 * x) * np.cos(3 * y) + 1e-3 * rng.standard_normal(m)
    nrm = np.stack([-0.6 * np.cos(2 * x) * np.cos(3 * y), 0.9 * np.sin(2 * x) * np.sin(3 * y), np.ones(m)], 1)
    return np.stack([x, y, z], 1), nrm / np.linalg.norm(nrm, axis=1, keepdims=True)


def knn_rows(p, k):
    """k nearest neighbours of every point (itself first), from scipy's tree."""
    _, i = cKDTree(p).query(p, k)
    return i.reshape(len(p), k)


CLOUDS = {"sphere": lambda: fibonacci_sphere(2000, 1e-3), "torus": torus_cloud, "height field": height_field}


# ---- CPU: the restatement --------------------------------------------------------------------------------------------
def test_signature(pcu):
    ps = list(inspect.signature(pcu.estimate_point_cloud_areas).parameters.values())
    assert [p.name for p in ps] == ["p", "i", "n", "device"]
    assert ps[3].kind == inspect.Parameter.KEYWORD_ONLY and ps[3].default is None
    assert "estimate_point_cloud_areas" in pcu.__all__


@pytest.mark.parametrize("name", sorted(CLOUDS))
@pytest.mark.parametrize("k", [8, 16, 30])
def test_restatement_is_the_delaunay_star(name, k):
    p, n = CLOUDS[name]()
    i = knn_rows(p, k)
    rows = np.random.default_rng(k).choice(len(p), 400, replace=False)
    ours = areas_ref(p, i, n, rows)
    theirs = np.array([delaunay_area(project(p, n, i[r])) for r in rows])
    assert (ours > 0).all()
    assert np.abs(ours - theirs).max() <= 1e-12 * np.abs(theirs).max(), np.abs(ours - theirs).max()


def test_sphere_total():
    p, n = fibonacci_sphere(4000, 1e-3)
    a = areas_ref(p, knn_rows(p, 16), n)
    assert abs(a.sum() - 4 * math.pi) <= 2e-3 * 4 * math.pi, a.sum()


def lattice(h=0.1, size=20):
    xs, ys = np.meshgrid(np.arange(size) * h, np.arange(size) * h)
    p = np.stack([xs.ravel(), ys.ravel(), np.zeros(size * size)], 1)
    return p, np.tile([0.0, 0.0, 1.0], (len(p), 1))


def hex_lattice(size=20):
    p = np.array([[x + 0.5 * (y % 2), y * math.sqrt(3) / 2, 0.0] for y in range(size) for x in range(size)])
    return p, np.tile([0.0, 0.0, 1.0], (len(p), 1))


LATTICE_CASES = [  # (cloud, k, row, area)
    ("square", 9, 10 * 20 + 10, 0.01), ("square", 9, 10, 0.005), ("square", 9, 0, 0.0025), ("square", 9, 399, 0.0025),
    ("hex", 7, 10 * 20 + 10, math.sqrt(3) / 2),
]


def lattice_cloud(name):
    return lattice() if name == "square" else hex_lattice()


@pytest.mark.parametrize("name,k,row,area", LATTICE_CASES)
def test_lattices(name, k, row, area):
    p, n = lattice_cloud(name)
    a = areas_ref(p, knn_rows(p, k), n, [row])[0]
    assert a == pytest.approx(area, rel=1e-12)


def zero_rule_cases():
    """(name, p, i, n, expected areas of every row or None, rows to compare with): rows where rule 1 or 3 leaves
    nothing, and rows whose dropped columns must not matter."""
    p, n = lattice()
    c = 10 * 20 + 10
    base = knn_rows(p, 9)[c]
    ring = base[1:]
    cases = []
    cases.append(("k = 2", p, knn_rows(p, 2), n, np.zeros(len(p))))
    n0 = n.copy()
    n0[c] = 0
    cases.append(("zero centre normal", p, np.tile(base, (len(p), 1)), n0, np.zeros(len(p))))
    flip = n.copy()
    flip[ring[2:]] *= -1                                                  # 2 of 8 neighbours kept: |K| = 3
    perp = n.copy()
    perp[ring[3:]] = [1.0, 0.0, 0.0]                                      # a zero dot product is dropped too
    cases.append(("opposing normals", p, np.tile(base, (len(p), 1)), flip, None))
    cases.append(("perpendicular normals", p, np.tile(base, (len(p), 1)), perp, None))
    t = np.linspace(-1, 1, 12)
    line = np.stack([t, 0 * t, 0 * t], 1)                               # on an axis
    cases.append(("collinear on an axis", line, knn_rows(line, 6), np.tile([0.0, 0.0, 1.0], (12, 1)), np.zeros(12)))
    same = np.tile([[0.3, -0.2, 0.7]], (10, 1))
    cases.append(("coincident", same, np.tile(np.arange(10), (10, 1)), np.tile([0.0, 1.0, 0.0], (10, 1)), np.zeros(10)))
    return cases


def test_zero_and_filter_rules():
    for name, p, i, n, expect in zero_rule_cases():
        a = areas_ref(p, i, n)
        if expect is not None:
            assert np.array_equal(a, expect), name
    p, n = lattice()
    c = 10 * 20 + 10
    row = knn_rows(p, 9)[c]
    # opposing normals: the row is the row without those columns
    flip = n.copy()
    flip[row[5:]] *= -1
    full = np.tile(row, (len(p), 1))
    assert areas_ref(p, full, flip, [0])[0] == areas_ref(p, np.tile(row[:5], (len(p), 1)), n, [0])[0]
    # collinear points in a general direction: the projection's rounding leaves slivers of ~u times the spacing squared
    t = np.linspace(-1, 1, 12)[:, None]
    line = t * np.array([[0.3, -0.5, 0.8]]) + np.array([[1.0, 2.0, 3.0]])
    assert np.abs(areas_ref(line, knn_rows(line, 6), np.tile([0.0, 0.0, 1.0], (12, 1)))).max() <= 1e-14 * (2 / 11) ** 2
    # duplicates of the centre are not candidates: the planar row keeps its area
    dup = np.concatenate([row, [c, c]])
    assert areas_ref(p, np.tile(dup, (len(p), 1)), n, [0])[0] == pytest.approx(0.01, rel=1e-12)
    # a centre on the hull: only the right walk's triangles
    half = np.array([r for r in knn_rows(p, 25)[c] if p[r, 1] >= p[c, 1]])
    assert areas_ref(p, np.tile(half, (len(p), 1)), n, [0])[0] == pytest.approx(0.005, rel=1e-12)


def test_argument_errors_come_before_the_device(pcu):
    f = pcu.estimate_point_cloud_areas
    p, n = fibonacci_sphere(50)
    i = knn_rows(p, 4)
    before = pcu.launch_count()
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'p'. Expected one of"):
        f(p.astype(np.int32), i, n)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'i'. Expected one of \['int32', 'int64', "
                                         r"'uint32', 'uint64'\]"):
        f(p, i.astype(np.float64), n)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int16\) for argument 'i'"):
        f(p, i.astype(np.int16), n)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'n'. Expected it to match argument 'p' "
                                         r"which is of type float64."):
        f(p, i, n.astype(np.float32))
    with pytest.raises(ValueError, match=r"Only 3D inputs are supported: v must have shape \(n, 3\) \(n > 0\). Got "
                                         r"points.shape =\(50, 2\)."):
        f(p[:, :2], i, n)
    with pytest.raises(ValueError, match=r"Invalid shape for normals: must have shape \(n, 3\) \(n > 0\). Got "
                                         r"normals.shape =\(50, 2\)."):
        f(p, i, n[:, :2])
    with pytest.raises(ValueError, match=r"Invalid input point cloud. Number of normals must match number of points. Got "
                                         r"points.shape =\(50, 3\) and normals.shape = 5, 3$"):
        f(p, i, n[:5])
    msg = r"Invalid shape for i \(knn indices\), must be \(#p, k\) where #p is the number of input points \(50\). Got \(%d, %d\)$"
    with pytest.raises(ValueError, match=msg % (49, 4)):
        f(p, i[:-1], n)
    with pytest.raises(ValueError, match=msg % (49, 1)):
        f(p, i[:-1, 0], n)
    with pytest.raises(ValueError, match=msg % (200, 1)):
        f(p, i.reshape(50, 2, 2), n)
    big = np.zeros((50, 257), np.int64)
    with pytest.raises(ValueError, match=r"at most 256 neighbours per point are supported, got k = 257"):
        f(p, big, n)
    with pytest.raises(ValueError, match="NumPy array"):
        f(p.tolist(), i, n)
    assert pcu.launch_count() == before
    # no points: an empty result of p's dtype, without a device call
    for dt in (np.float32, np.float64):
        a = f(p[:0].astype(dt), i[:0], n[:0].astype(dt))
        assert isinstance(a, np.ndarray) and a.dtype == dt and a.shape == (0,)
    assert pcu.launch_count() == before


# ---- GPU --------------------------------------------------------------------------------------------------------------
def bunny():
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    return np.load(os.path.join(here, "golden", "bunny_vertices.npy")).astype(np.float64)


def knn_normals(pcu, p):
    """Normals from estimate_point_cloud_normals_knn (k = 12), oriented away from the centroid; dropped points get 0."""
    view = p - p.mean(0)
    view /= np.linalg.norm(view, axis=1, keepdims=True)
    idx, nrm = pcu.estimate_point_cloud_normals_knn(p, 12, view)
    n = np.zeros_like(p)
    n[idx] = nrm
    return n


def gpu_clouds(pcu):
    p, n = fibonacci_sphere(3000, 2e-3, 3)
    yield "sphere", p, n
    p, n = torus_cloud()
    yield "torus", p, n
    p = bunny()
    yield "bunny", p, knn_normals(pcu, p)


def assert_close(a, ref, dtype, what):
    """fp64: within 1e-12 of the restatement relative to each area (and to 1e-12 of the largest one near zero); fp32:
    within one float32 ulp of the restatement rounded to float32."""
    a = np.asarray(a)
    assert a.dtype == dtype, what
    if dtype == np.float64:
        err = np.abs(a - ref)
        tol = 1e-12 * np.maximum(np.abs(ref), np.abs(ref).max())
        assert (err <= tol).all(), "%s: %d rows, worst %.3g" % (what, int((err > tol).sum()), (err / np.maximum(np.abs(ref), 1e-300)).max())
    else:
        r32 = ref.astype(np.float32)
        err = np.abs(a.astype(np.float64) - r32.astype(np.float64))
        ulp = np.spacing(np.abs(r32)).astype(np.float64)
        assert (err <= ulp).all(), "%s: %d rows beyond one ulp" % (what, int((err > ulp).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kernel_matches_the_restatement(pcu, dtype):
    import torch
    combo = 0
    for name, p, n in gpu_clouds(pcu):
        p, n = p.astype(dtype), n.astype(dtype)
        rows = np.sort(np.random.default_rng(len(p)).choice(len(p), 500, replace=False))
        for k in KS:
            i = knn_rows(p.astype(np.float64), k)
            ref = areas_ref(p, i, n, rows)
            kind, form = KINDS[combo % 4], FORMS[(combo // 4) % 3]
            combo += 1
            a = to_numpy(pcu.estimate_point_cloud_areas(*(to_form(form, x) for x in (p, i.astype(kind), n))), form)
            assert a.shape == (len(p),)
            assert_close(a[rows], ref, dtype, "%s k=%d %s %s" % (name, k, kind, form))
            if k == 1:
                assert not a.any()
                assert not to_numpy(pcu.estimate_point_cloud_areas(p, i[:, 0], n)).any()    # the squeezed (#p,) form
        # i straight from k_nearest_neighbors as a CUDA tensor
        pt, nt = torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda()
        _, it = pcu.k_nearest_neighbors(pt, pt, 16)
        a = pcu.estimate_point_cloud_areas(pt, it, nt)
        assert a.is_cuda and a.dtype == pt.dtype
        assert_close(a.cpu().numpy()[rows], areas_ref(p, it.cpu().numpy(), n, rows), dtype, "%s from k_nearest_neighbors" % name)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_index_kinds_and_input_forms_agree(pcu, dtype):
    p, n = torus_cloud()
    p, n = p.astype(dtype), n.astype(dtype)
    i = knn_rows(p.astype(np.float64), 16)
    a = pcu.estimate_point_cloud_areas(p, i, n)
    for kind in KINDS:
        for form in FORMS:
            b = to_numpy(pcu.estimate_point_cloud_areas(*(to_form(form, x) for x in (p, i.astype(kind), n))), form)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (kind, form)
    assert np.array_equal(a, pcu.estimate_point_cloud_areas(p, i, n, device="cuda:0"))
    assert np.array_equal(a, pcu.estimate_point_cloud_areas(np.asfortranarray(p), i[:, ::-1][:, ::-1], n))
    one = pcu.estimate_point_cloud_areas(p[:1], i[:1, :1] * 0, n[:1])      # one point: squeezed like the reference's
    assert one.shape == () and one == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,k,row,area", LATTICE_CASES)
def test_kernel_lattices(pcu, name, k, row, area):
    p, n = lattice_cloud(name)
    a = pcu.estimate_point_cloud_areas(p, knn_rows(p, k), n)
    assert a[row] == pytest.approx(area, rel=1e-12)


@pytest.mark.gpu
def test_kernel_zero_rules(pcu):
    for name, p, i, n, expect in zero_rule_cases():
        a = pcu.estimate_point_cloud_areas(p, i, n)
        assert_close(a, areas_ref(p, i, n), np.float64, name)
        if expect is not None:
            assert np.array_equal(a, expect), name


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_invariances(pcu, dtype):
    p, n = fibonacci_sphere(3000, 2e-3, 4)
    p = (np.round(p * 2.0 ** 16) / 2.0 ** 16).astype(dtype)                # so that the translation below is exact
    n = n.astype(dtype)
    i = knn_rows(p.astype(np.float64), 16)
    a = pcu.estimate_point_cloud_areas(p, i, n)
    assert np.array_equal(a.view(np.uint8), pcu.estimate_point_cloud_areas(p, i, n).view(np.uint8)), "second call"
    for e in (-6, 3, 20):
        s = pcu.estimate_point_cloud_areas(p * dtype(2.0 ** e), i, n)
        assert np.array_equal(s, a * dtype(4.0 ** e)), e
    t = p + np.array([3.0, -5.0, 7.0], dtype)
    assert np.array_equal(t - np.array([3.0, -5.0, 7.0], dtype), p)
    b = pcu.estimate_point_cloud_areas(t, i, n)
    if dtype == np.float64:
        assert np.abs(b - a).max() <= 1e-10 * np.abs(a).max()
    else:
        assert (np.abs(b.astype(np.float64) - a) <= np.spacing(np.abs(a))).all()


@pytest.mark.gpu
def test_out_of_range_indices_raise(pcu):
    import torch
    p, n = fibonacci_sphere(500)
    i = knn_rows(p, 8)
    for kind in KINDS:
        bad = i.astype(kind)
        bad[7, 3] = 500
        bad[9, 0] = 10 ** 6
        with pytest.raises(ValueError, match=r"Invalid knn indices: 2 entries of i are outside \[0, #p\)"):
            pcu.estimate_point_cloud_areas(p, bad, n)
    neg = i.copy()
    neg[3, 5] = -1
    with pytest.raises(ValueError, match=r"1 entries of i are outside"):
        pcu.estimate_point_cloud_areas(p, neg, n)
    # k > #p: k_nearest_neighbors pads its rows with -1
    pt, nt = torch.from_numpy(p[:20]).cuda(), torch.from_numpy(n[:20]).cuda()
    _, it = pcu.k_nearest_neighbors(pt, pt, 24)
    with pytest.raises(ValueError, match=r"Invalid knn indices: 80 entries of i are outside \[0, #p\)"):
        pcu.estimate_point_cloud_areas(pt, it, nt)


# The workflow the function exists for: areas of a sampled sphere (Fibonacci lattice, 10^5 points, radial normals, k =
# 16) fed to point_cloud_fast_winding_number.  The restated areas with the exact fp64 dipole sum (exact_pw), on the CPU:
# sum(a) - 4 pi = -5.1e-4; over the queries below, max |w - 1| = 4.1e-5 at radius 0.5 and max |w| = 1.0e-7 at radius 2.
# The thresholds are twice those, plus 1e-5 for the fp32 evaluation of the field (the bound of the winding-number tests'
# exact mode).  The public call adds its far-field expansion's error, at most PUBLIC_TOL there.
SPHERE_TOTAL_TOL = 1.1e-3
INSIDE_TOL, OUTSIDE_TOL = 2 * 4.1e-5 + 1e-5, 2 * 1.0e-7 + 1e-5


def workflow_queries():
    rng = np.random.default_rng(11)
    u = rng.standard_normal((500, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return 0.5 * u, 2.0 * u


@pytest.mark.gpu
def test_areas_feed_the_winding_number(pcu):
    import torch
    p, n = fibonacci_sphere(10 ** 5)
    pt, nt = torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda()
    _, it = pcu.k_nearest_neighbors(pt, pt, 16)
    a = pcu.estimate_point_cloud_areas(pt, it, nt)
    rows = np.random.default_rng(0).choice(len(p), 1000, replace=False)
    assert_close(a.cpu().numpy()[rows], areas_ref(p, it.cpu().numpy(), n, rows), np.float64, "sphere rows")
    assert abs(float(a.sum()) - 4 * math.pi) <= SPHERE_TOTAL_TOL, float(a.sum())
    inside, outside = workflow_queries()
    w_in = pwn_device(pcu, p, n, a.cpu().numpy(), inside, float("inf"))
    w_out = pwn_device(pcu, p, n, a.cpu().numpy(), outside, float("inf"))
    print("exact: max |w - 1| at radius 0.5: %.3g, max |w| at radius 2: %.3g" % (np.abs(w_in - 1).max(), np.abs(w_out).max()))
    assert np.abs(w_in - 1).max() <= INSIDE_TOL and np.abs(w_out).max() <= OUTSIDE_TOL
    w_in = pcu.point_cloud_fast_winding_number(pt, nt, a, torch.from_numpy(inside).cuda()).cpu().numpy()
    w_out = pcu.point_cloud_fast_winding_number(pt, nt, a, torch.from_numpy(outside).cuda()).cpu().numpy()
    print("public: max |w - 1| at radius 0.5: %.3g, max |w| at radius 2: %.3g" % (np.abs(w_in - 1).max(), np.abs(w_out).max()))
    assert np.abs(w_in - 1).max() <= INSIDE_TOL + PUBLIC_TOL and np.abs(w_out).max() <= OUTSIDE_TOL + PUBLIC_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_full_size(pcu, dtype):
    import torch
    p, n = fibonacci_sphere(10 ** 6, 1e-4, 6)
    p, n = p.astype(dtype), n.astype(dtype)
    pt, nt = torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda()
    _, it = pcu.k_nearest_neighbors(pt, pt, 16)
    a = pcu.estimate_point_cloud_areas(pt, it, nt)
    assert a.is_cuda and a.shape == (10 ** 6,)
    rows = np.sort(np.random.default_rng(7).choice(10 ** 6, 1000, replace=False))
    ref = areas_ref(p, it.cpu().numpy(), n, rows)
    assert_close(a.cpu().numpy()[rows], ref, dtype, "full size")
