"""pointcloud_apss_curvature and project_points_onto_apss (DESIGN.md §3).

A numpy restatement of the rules -- exact ball membership in p's dtype, the nine fp64 sums, the closed-form sphere fit,
the stable step and the stopping rule -- is pinned on the CPU to exact spheres and planes, to a cylinder, a torus and a
noisy sphere against their analytic mean curvatures, and to the undetermined rules; on the GPU both functions are
checked against it over dtypes, input forms and clouds, and for exact scaling, translation, determinism and a workflow
from raw points."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from meshes import to_form, to_numpy

STEPS, TOL = 20, 1e-10


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


class Apss:
    """The rules of DESIGN.md §3, one query at a time."""

    def __init__(self, p, n, r):
        self.T = p.dtype.type
        self.p = p
        self.pd = p.astype(np.float64)
        nd = n.astype(np.float64)
        ln = np.sqrt(_dot(nd, nd))
        with np.errstate(invalid="ignore", divide="ignore"):
            self.nh = np.where((ln > 0)[:, None], nd / ln[:, None], 0.0)
        self.has = (self.nh != 0).any(1)
        self.r, self.rr = float(r), float(r) * float(r)
        self.r2 = self.T(self.rr)
        self.tree = cKDTree(self.pd) if len(p) else None

    def members(self, x):
        """N(x): d2(fl_T(x), p_j) < (T)(r r) in p's dtype, zero normals left out."""
        if self.tree is None:
            return np.zeros(0, np.int64)
        c = x.astype(self.T)
        js = np.asarray(self.tree.query_ball_point(c.astype(np.float64), self.r * (1 + 1e-5) + 1e-300), np.int64)
        d = c - self.p[js]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        js = js[d2 < self.r2]
        return js[self.has[js]]

    def project(self, q):
        """(x, nx, kh) for one query, or None when it is undetermined."""
        x = np.asarray(q, np.float64).copy()
        for _ in range(STEPS):
            js = self.members(x)
            if len(js) < 4:
                return None
            o = self.pd[js] - x
            oo = _dot(o, o)
            t = np.maximum(0.0, 1.0 - oo / self.rr)
            t2 = t * t
            w = t2 * t2
            nh = self.nh[js]
            W, P, N = w.sum(), (w[:, None] * o).sum(0), (w[:, None] * nh).sum(0)
            PN, PP = (w * _dot(o, nh)).sum(), (w * oo).sum()
            if not W > 0:
                return None
            den = PP - _dot(P, P) / W
            u4 = 0.5 * (PN - _dot(P, N) / W) / den if den > 1e-12 * PP else 0.0
            u = (N - 2.0 * u4 * P) / W
            u0 = -(_dot(u, P) + u4 * PP) / W
            g = np.sqrt(_dot(u, u))
            D = g * g - 4.0 * u0 * u4
            if not g > 0 or D < 0:
                return None
            y = -2.0 * u0 / (g + np.sqrt(D)) * (u / g)
            x = x + y
            if np.sqrt(_dot(y, y)) <= TOL * self.r:
                break
        return x, u / g, 2.0 * u4 / np.sqrt(D)

    def run(self, q):
        """(x, nx, kh) in fp64 for every query, undetermined ones as NaN, 0, NaN."""
        q = np.asarray(q)
        x, nx, kh = np.full((len(q), 3), np.nan), np.zeros((len(q), 3)), np.full(len(q), np.nan)
        for i, qi in enumerate(q):
            out = self.project(qi)
            if out is not None:
                x[i], nx[i], kh[i] = out
        return x, nx, kh


# ---- clouds -------------------------------------------------------------------------------------------------------------
def fibonacci_sphere(m, R=1.0, dtype=np.float64):
    """m points of a Fibonacci lattice on the sphere of radius R, with their outward unit normals."""
    k = np.arange(m) + 0.5
    z = 1 - 2 * k / m
    phi = np.pi * (1 + 5 ** 0.5) * k
    s = np.sqrt(1 - z * z)
    u = np.stack([s * np.cos(phi), s * np.sin(phi), z], 1)
    return (R * u).astype(dtype), u.astype(dtype)


def noisy_sphere(m, R=1.0, noise=0.002, seed=0, dtype=np.float64):
    """m uniform directions at radius R (1 + noise N(0, 1)), with exact radial normals."""
    rng = np.random.default_rng(seed)
    u = rng.standard_normal((m, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (u * R * (1 + noise * rng.standard_normal((m, 1)))).astype(dtype), u.astype(dtype)


def torus_cloud(m, a=0.35, seed=0, dtype=np.float64):
    """m points uniform in both angles of the torus of major radius 1 and minor radius a, outward normals, and the
    analytic mean curvature (1 + 2 a cos v) / (2 a (1 + a cos v)) at each."""
    rng = np.random.default_rng(seed)
    uu, vv = rng.uniform(0, 2 * np.pi, m), rng.uniform(0, 2 * np.pi, m)
    nrm = np.stack([np.cos(vv) * np.cos(uu), np.cos(vv) * np.sin(uu), np.sin(vv)], 1)
    p = np.stack([np.cos(uu), np.sin(uu), 0 * uu], 1) + a * nrm
    return p.astype(dtype), nrm.astype(dtype), (1 + 2 * a * np.cos(vv)) / (2 * a * (1 + a * np.cos(vv)))


def cylinder(m, length=8.0, seed=0):
    """m points uniform on the side of the unit cylinder about z, |z| <= length / 2, outward normals."""
    rng = np.random.default_rng(seed)
    th, z = rng.uniform(0, 2 * np.pi, m), rng.uniform(-length / 2, length / 2, m)
    n = np.stack([np.cos(th), np.sin(th), 0 * th], 1)
    return n + z[:, None] * np.array([0.0, 0.0, 1.0]), n


def _bunny():
    import os
    g = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    v = np.load(os.path.join(g, "bunny_vertices.npy")).astype(np.float64)
    f = np.load(os.path.join(g, "bunny_faces.npy")).astype(np.int64)
    # area-weighted vertex normals of the mesh, outward
    cr = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], cr)
    return v, n


def spacing(p, area):
    return float(np.sqrt(area / len(p)))


def _sphere_case():
    p, n = fibonacci_sphere(3000, 2.0)
    return p, n, 3 * spacing(p, 16 * np.pi)


def _torus_case():
    p, n, _ = torus_cloud(4000, seed=1)
    return p, n, 3 * spacing(p, 4 * np.pi ** 2 * 0.35)


def _bunny_case():
    v, n = _bunny()
    return v, n, 4 * float(np.median(cKDTree(v).query(v, 2)[0][:, 1]))


def _noisy_case():
    p, n = noisy_sphere(3000, 1.0, 0.01, seed=4)
    n = n + 0.05 * np.random.default_rng(5).standard_normal(n.shape)
    n[::97] = 0.0   # some points without a normal
    return p, n, 4 * spacing(p, 4 * np.pi)


CLOUDS = {"sphere": _sphere_case, "torus": _torus_case, "bunny": _bunny_case, "noisy": _noisy_case}


def queries(p, r, m=300, seed=0):
    """m cloud points moved off the surface by up to r / 4, plus three far-away queries (empty balls)."""
    rng = np.random.default_rng(seed)
    q = p[rng.choice(len(p), m, replace=False)].astype(np.float64) + rng.uniform(-0.25, 0.25, (m, 3)) * r
    return np.concatenate([q, [[1e3, 0, 0], [0, -1e3, 0], [0, 0, 1e3]]]).astype(p.dtype)


# ---- CPU: the restatement on analytic surfaces ----------------------------------------------------------------------------
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_restatement_exact_sphere(sign):
    R = 2.0
    p, n = fibonacci_sphere(4000, R)
    r = 4 * spacing(p, 4 * np.pi * R * R)
    rng = np.random.default_rng(0)
    d = rng.standard_normal((120, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    q = d * R * rng.choice([0.95, 1.05], (120, 1))
    x, nx, kh = Apss(p, sign * n, r).run(q)
    assert np.abs(kh * R - sign).max() < 1e-12
    assert np.abs(np.linalg.norm(x, axis=1) - R).max() < 1e-12 * R
    assert np.abs(nx - sign * x / R).max() < 1e-12


def test_restatement_plane():
    rng = np.random.default_rng(1)
    g = np.stack(np.meshgrid(np.arange(40.0), np.arange(40.0), indexing="ij"), -1).reshape(-1, 2)
    g += rng.uniform(-0.3, 0.3, g.shape)
    p = np.concatenate([g, np.zeros((len(g), 1))], 1)
    n = np.tile([0.0, 0.0, 1.0], (len(p), 1))
    r = 3.0
    q = np.concatenate([rng.uniform(10, 30, (100, 2)), rng.uniform(-1, 1, (100, 1))], 1)
    x, nx, kh = Apss(p, n, r).run(q)
    assert np.abs(kh).max() < 1e-12 / r
    assert np.abs(x[:, :2] - q[:, :2]).max() < 1e-12 * r and np.abs(x[:, 2]).max() < 1e-12 * r
    assert np.abs(nx - [0.0, 0.0, 1.0]).max() < 1e-12


def test_restatement_cylinder():
    # the median kh of 300 points away from the ends against the mean curvature 1/2: measured 0.5045, 0.4984 and 0.5039
    # at r = 3, 6 and 12 mean spacings (a sphere fitted to a cylinder: single points range from 0.17 to 0.81 at r = 3)
    p, n = cylinder(20000)
    h = spacing(p, 2 * np.pi * 8.0)
    rows = np.flatnonzero(np.abs(p[:, 2]) < 2.0)[:300]
    for k in (3, 6, 12):
        kh = Apss(p, n, k * h).run(p[rows])[2]
        assert abs(np.median(kh) - 0.5) < 0.01, (k, np.median(kh))


def test_restatement_torus():
    # |kh - H| / max H over 400 points at r = 4 mean spacings: measured median 0.075, largest 0.35
    p, n, H = torus_cloud(20000, seed=2)
    r = 4 * spacing(p, 4 * np.pi ** 2 * 0.35)
    rows = np.arange(400)
    kh = Apss(p, n, r).run(p[rows])[2]
    err = np.abs(kh - H[rows]) / np.abs(H[rows]).max()
    assert np.median(err) < 0.1 and err.max() < 0.5, (np.median(err), err.max())


def test_restatement_noisy_sphere():
    # position noise 0.002 R, exact normals: median |kh R - 1| measured 0.0045 at r = 3 mean spacings, 0.0011 at r = 6
    p, n = noisy_sphere(20000, 1.0, 0.002, seed=3)
    h = spacing(p, 4 * np.pi)
    rows = np.arange(300)
    for k, bound in ((3, 0.008), (6, 0.002)):
        kh = Apss(p, n, k * h).run(p[rows])[2]
        assert np.median(np.abs(kh - 1)) < bound, (k, np.median(np.abs(kh - 1)))


def test_restatement_undetermined():
    p, n = fibonacci_sphere(500)
    r = 0.3
    # fewer than 4 members
    x, nx, kh = Apss(p[:3], n[:3], r).run(p[:3])
    assert np.isnan(x).all() and not nx.any() and np.isnan(kh).all()
    # all normals zero
    x, nx, kh = Apss(p, 0 * n, r).run(p[:5])
    assert np.isnan(x).all() and not nx.any() and np.isnan(kh).all()
    # a query with an empty ball next to a determined one
    x, nx, kh = Apss(p, n, r).run(np.array([[5.0, 5.0, 5.0], p[0]]))
    assert np.isnan(x[0]).all() and not nx[0].any() and np.isnan(kh[0])
    assert np.isfinite(kh[1]) and np.isfinite(x[1]).all()
    # no points at all
    x, nx, kh = Apss(p[:0], n[:0], r).run(p[:4])
    assert np.isnan(x).all() and not nx.any() and np.isnan(kh).all()


def test_empty_cloud_curvature_before_any_device_call(pcu):
    import torch
    p = np.zeros((0, 3))
    kh = pcu.pointcloud_apss_curvature(p, p, 1.0)
    assert isinstance(kh, np.ndarray) and kh.shape == (0,) and kh.dtype == np.float64
    kh = pcu.pointcloud_apss_curvature(torch.zeros((0, 3), dtype=torch.float32), torch.zeros((0, 3), dtype=torch.float32), 1.0)
    assert isinstance(kh, torch.Tensor) and kh.shape == (0,) and kh.dtype == torch.float32


@pytest.mark.parametrize("form", ["numpy", "cpu"])
def test_argument_errors_before_any_device_call(pcu, form):
    p, n = fibonacci_sphere(50)
    P, N, Q = to_form(form, p), to_form(form, n), to_form(form, p[:5])
    for bad in (0.0, -1.0, float("nan"), float("inf"), "a", None):
        with pytest.raises(ValueError, match="Invalid radius"):
            pcu.pointcloud_apss_curvature(P, N, bad)
        with pytest.raises(ValueError, match="Invalid radius"):
            pcu.project_points_onto_apss(P, N, Q, bad)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.pointcloud_apss_curvature(P, to_form(form, n.astype(np.float32)), 0.3)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.project_points_onto_apss(P, N, to_form(form, p[:5].astype(np.float32)), 0.3)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.pointcloud_apss_curvature(to_form(form, p.astype(np.int32)), to_form(form, n.astype(np.int32)), 0.3)
    with pytest.raises(ValueError, match="Number of normals must match"):
        pcu.pointcloud_apss_curvature(P, to_form(form, n[:-1].copy()), 0.3)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.pointcloud_apss_curvature(to_form(form, p[:, :2].copy()), to_form(form, n[:, :2].copy()), 0.3)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.project_points_onto_apss(P, N, to_form(form, p[:5, :2].copy()), 0.3)
    with pytest.raises(ValueError, match="zero points"):
        pcu.project_points_onto_apss(P, N, to_form(form, p[:0]), 0.3)
    if form == "numpy":
        with pytest.raises(ValueError, match="must be a NumPy array"):
            pcu.pointcloud_apss_curvature(p.tolist(), n, 0.3)


# ---- GPU ------------------------------------------------------------------------------------------------------------------
def _compare(got, want, r, dtype):
    """(x, nx, kh) against the restatement: the same undetermined rows; in fp64 x within 1e-9 r, nx within 1e-9 and kh
    within 1e-9 / r (the stopping test may fall on the other side of 1e-10 r in one of the two); in fp32 two spacings of
    the fp32 value on top."""
    x, nx, kh = (np.asarray(a, np.float64) for a in got)
    wx, wn, wk = want
    bad = np.isnan(wk)
    assert (np.isnan(kh) == bad).all() and np.isnan(x[bad]).all() and not nx[bad].any()
    ok = ~bad

    def close(g, w, tol):
        if dtype == np.float32:
            tol = tol + 2 * np.spacing(np.abs(w).astype(np.float32)).astype(np.float64)
        err = np.abs(g - w)
        assert (err <= tol).all(), (err - tol).max()

    close(x[ok], wx[ok], 1e-9 * r)
    close(nx[ok], wn[ok], 1e-9)
    close(kh[ok], wk[ok], 1e-9 / r)


FORMS = ["numpy", "cpu", "cuda"]


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["curvature", "project"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(CLOUDS))
def test_against_restatement(pcu, name, dtype, fn):
    p, n, r = CLOUDS[name]()
    p, n = p.astype(dtype), n.astype(dtype)
    ref = Apss(p, n, r)
    for form in FORMS:
        if fn == "curvature":
            kh = to_numpy(pcu.pointcloud_apss_curvature(to_form(form, p), to_form(form, n), r), form)
            assert kh.dtype == dtype and kh.shape == (len(p),)
            rows = np.random.default_rng(1).choice(len(p), min(len(p), 400), replace=False)
            x, nx, wk = ref.run(p[rows])
            _compare((x, nx, kh[rows]), (x, nx, wk), r, dtype)
        else:
            q = queries(p, r)
            got = [to_numpy(a, form) for a in pcu.project_points_onto_apss(to_form(form, p), to_form(form, n), to_form(form, q), r)]
            assert all(a.dtype == dtype for a in got)
            assert got[0].shape == (len(q), 3) and got[1].shape == (len(q), 3) and got[2].shape == (len(q),)
            _compare(got, ref.run(q), r, dtype)


@pytest.mark.gpu
def test_empty_cloud_and_undetermined(pcu):
    p, n = fibonacci_sphere(500)
    q = np.concatenate([p[:5], [[5.0, 5.0, 5.0]]])
    x, nx, kh = pcu.project_points_onto_apss(p[:0], n[:0], q, 0.3)
    assert np.isnan(x).all() and not nx.any() and np.isnan(kh).all() and x.shape == (6, 3)
    x, nx, kh = pcu.project_points_onto_apss(p, 0 * n, q, 0.3)
    assert np.isnan(x).all() and not nx.any() and np.isnan(kh).all()
    assert np.isnan(pcu.pointcloud_apss_curvature(p[:3], n[:3], 0.3)).all()
    x, nx, kh = pcu.project_points_onto_apss(p, n, q, 0.3)
    assert np.isnan(kh[5]) and np.isnan(x[5]).all() and not nx[5].any() and np.isfinite(kh[:5]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("e", [3, -2])
def test_exact_scaling(pcu, dtype, e):
    p, n, r = _noisy_case()
    p, n = p.astype(dtype), n.astype(dtype)
    q = queries(p, r)
    s = dtype(2.0 ** e)
    a = pcu.project_points_onto_apss(p, n, q, r)
    b = pcu.project_points_onto_apss(p * s, n, q * s, r * float(s))
    assert np.array_equal(b[0], a[0] * s, equal_nan=True)
    assert np.array_equal(b[1], a[1], equal_nan=True)
    assert np.array_equal(b[2], a[2] / s, equal_nan=True)
    assert np.array_equal(pcu.pointcloud_apss_curvature(p * s, n, r * float(s)), pcu.pointcloud_apss_curvature(p, n, r) / s, equal_nan=True)


@pytest.mark.gpu
def test_translation(pcu):
    p, n, r = _torus_case()
    q = queries(p, r)
    t = np.array([3.0, -2.0, 0.5])
    x, nx, kh = pcu.project_points_onto_apss(p, n, q, r)
    y, ny, kt = pcu.project_points_onto_apss(p + t, n, q + t, r)
    assert np.array_equal(np.isnan(kh), np.isnan(kt))
    ok = ~np.isnan(kh)
    assert np.abs(y[ok] - t - x[ok]).max() < 1e-9 * r
    assert np.abs(ny[ok] - nx[ok]).max() < 1e-8 and np.abs(kt[ok] - kh[ok]).max() < 1e-8 / r


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_deterministic_and_curvature_is_projection(pcu, dtype):
    import torch
    p, n, r = _bunny_case()
    p, n = torch.from_numpy(p.astype(dtype)).cuda(), torch.from_numpy(n.astype(dtype)).cuda()
    a = pcu.project_points_onto_apss(p, n, p, r)
    b = pcu.project_points_onto_apss(p, n, p, r)
    assert all(torch.equal(u.nan_to_num(7.0), v.nan_to_num(7.0)) and u.is_cuda for u, v in zip(a, b))
    k1 = pcu.pointcloud_apss_curvature(p, n, r)
    k2 = pcu.pointcloud_apss_curvature(p, n, r)
    assert k1.is_cuda and torch.equal(k1.nan_to_num(7.0), k2.nan_to_num(7.0))
    assert torch.equal(k1.nan_to_num(7.0), a[2].nan_to_num(7.0))


@pytest.mark.gpu
def test_workflow_from_raw_points(pcu):
    """A noisy 10^5-point sphere (R = 1, position noise 0.001): normals from estimate_point_cloud_normals_knn with 32
    neighbours, oriented by outward view directions, then the curvature and the projection of every point at r = 10 mean
    spacings.  Measured with the restatement on the CPU (numpy PCA normals of the same 32 neighbours, 1 000 rows): median
    |kh R - 1| 0.040, mean ||x| - R| 1.1e-4 against the input's 7.7e-4.  Normal noise dominates the curvature: with 16
    neighbours and r = 6 spacings the median is 0.18."""
    p, u = noisy_sphere(100000, 1.0, 0.001, seed=6)
    idx, n = pcu.estimate_point_cloud_normals_knn(p, 32, view_directions=u)
    assert len(idx) == len(p)
    r = 10 * spacing(p, 4 * np.pi)
    kh = pcu.pointcloud_apss_curvature(p, n, r)
    assert np.median(np.abs(kh - 1)) < 0.06
    x, nx, kx = pcu.project_points_onto_apss(p, n, p, r)
    assert np.isfinite(x).all() and np.array_equal(kx, kh)
    before, after = np.abs(np.linalg.norm(p, axis=1) - 1).mean(), np.abs(np.linalg.norm(x, axis=1) - 1).mean()
    assert after < 0.25 * before, (after, before)
    assert np.median(_dot(nx, x / np.linalg.norm(x, axis=1, keepdims=True))) > 0.999


@pytest.mark.gpu
def test_full_size(pcu):
    """10^6 points (noise 0.001, exact normals) at r = 6 mean spacings: every point determined, median |kh R - 1| measured
    0.013 on 300 rows of the restatement; sampled rows and queries against the restatement."""
    import torch
    p, n = noisy_sphere(10 ** 6, 1.0, 0.001, seed=7)
    r = 6 * spacing(p, 4 * np.pi)
    pt, nt = torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda()
    kh = pcu.pointcloud_apss_curvature(pt, nt, r).cpu().numpy()
    assert np.isfinite(kh).all() and np.median(np.abs(kh - 1)) < 0.02
    rows = np.random.default_rng(8).choice(len(p), 200, replace=False)
    ref = Apss(p, n, r)
    x, nx, wk = ref.run(p[rows])
    _compare((x, nx, kh[rows]), (x, nx, wk), r, np.float64)
    q = queries(p, r, 200, seed=9)
    got = [a.cpu().numpy() for a in pcu.project_points_onto_apss(pt, nt, torch.from_numpy(q).cuda(), r)]
    _compare(got, ref.run(q), r, np.float64)
