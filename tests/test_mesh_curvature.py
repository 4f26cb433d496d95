"""mesh_principal_curvatures and mesh_mean_and_gaussian_curvatures (DESIGN.md §3).

A numpy restatement of both modes -- the one-ring tensor estimate (r <= 0) and the quadric fit over a ball (r > 0) -- is
pinned on the CPU to analytic surfaces (sphere, torus, saddle, plane); on the GPU every output is checked against it
over dtypes, face index kinds, input forms and meshes with boundaries, degenerate faces, an isolated vertex and a
non-manifold edge.  The ball restatement reproduces the neighbour sets exactly: d2 in v's dtype, ((dx dx + dy dy) + dz dz)
< (T)(r r)."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from meshes import icosphere, noisy_icosphere, to_form, to_numpy, torus


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def frame(n):
    s = np.where(np.signbit(n[..., 2]), -1.0, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = -1.0 / (s + n[..., 2])
    b = n[..., 0] * n[..., 1] * a
    t1 = np.stack([1.0 + s * n[..., 0] * n[..., 0] * a, s * b, -s * n[..., 0]], -1)
    t2 = np.stack([b, s + n[..., 1] * n[..., 1] * a, -n[..., 1]], -1)
    return t1, t2


def eigen(a, b, c):
    m, p = 0.5 * (a + c), 0.5 * (a - c)
    h = np.hypot(p, b)
    x = np.where(p >= 0, h + p, b)
    y = np.where(p >= 0, b, h - p)
    ln = np.hypot(x, y)
    with np.errstate(invalid="ignore", divide="ignore"):
        x, y = np.where(h == 0, 1.0, x / ln), np.where(h == 0, 0.0, y / ln)
    return m + h, m - h, x, y


def directions(d, n):
    with np.errstate(invalid="ignore", divide="ignore"):
        d = d / np.sqrt(_dot(d, d))[..., None]
    j = np.argmax(np.abs(d), -1)   # first maximum: the lowest axis on a tie
    sgn = np.where(np.take_along_axis(d, j[..., None], -1)[..., 0] < 0, -1.0, 1.0)
    d = d * sgn[..., None]
    return d, _cross(n, d)


def vertex_normals(v, f):
    p = v[f]
    cr = _cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    A = np.sqrt(_dot(cr, cr))
    with np.errstate(invalid="ignore", divide="ignore"):
        unit = np.where(A[:, None] > 0, cr / A[:, None], 0.0)
        e1 = p[:, [1, 2, 0]] - p
        e2 = p[:, [2, 0, 1]] - p
        w = np.where(A[:, None] > 0, A[:, None] / (_dot(e1, e1) * _dot(e2, e2)), 0.0)
    s = np.zeros((len(v), 3))
    np.add.at(s, f.ravel(), (w[..., None] * unit[:, None, :]).reshape(-1, 3))
    ln = np.sqrt(_dot(s, s))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(ln[:, None] > 0, s / ln[:, None], 0.0), unit, A


def ring(v, f):
    v = np.asarray(v, np.float64)
    nv = len(v)
    n, unit, A = vertex_normals(v, f)
    p = v[f]
    nn = n[f]
    e = p[:, [2, 0, 1]] - p[:, [1, 2, 0]]
    dn = nn[:, [2, 0, 1]] - nn[:, [1, 2, 0]]
    len2 = _dot(e, e)
    dots = np.stack([_dot(p[:, (k + 1) % 3] - p[:, k], p[:, (k + 2) % 3] - p[:, k]) for k in range(3)], 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        hc = np.where(A[:, None] == 0, 0.0, 0.5 * (dots / A[:, None]))
        obt = (hc < 0).any(1)
        cw = np.empty_like(hc)
        for k in range(3):
            j, l = (k + 1) % 3, (k + 2) % 3
            cw[:, k] = np.where(obt, np.where(hc[:, k] < 0, 0.25 * A, 0.125 * A), 0.25 * (len2[:, j] * hc[:, j] + len2[:, l] * hc[:, l]))
        cw[A == 0] = 0.0
        u = e[:, 0] / np.sqrt(len2[:, 0])[:, None]
        w = unit
        vv = _cross(w, u)
        eu, ev = _dot(e, u[:, None]), _dot(e, vv[:, None])
        nu, nw = _dot(dn, u[:, None]), _dot(dn, vv[:, None])
        M00 = (eu * eu).sum(1); M01 = (eu * ev).sum(1); M11 = (eu * eu + ev * ev).sum(1); M12 = (eu * ev).sum(1); M22 = (ev * ev).sum(1)
        y0 = (eu * nu).sum(1); y1 = (ev * nu + eu * nw).sum(1); y2 = (ev * nw).sum(1)
        L00 = np.sqrt(M00); L10 = M01 / L00
        q1 = M11 - L10 * L10; L11 = np.sqrt(q1); L21 = M12 / L11
        q2 = M22 - L21 * L21; L22 = np.sqrt(q2)
        z0 = y0 / L00; z1 = (y1 - L10 * z0) / L11; z2 = (y2 - L21 * z1) / L22
        G = z2 / L22; F = (z1 - L21 * G) / L11; E = (z0 - L10 * F) / L00
    ok = (A != 0) & (M00 > 0) & (q1 > 0) & (q2 > 0)
    # corners
    t = np.repeat(np.arange(len(f)), 3)
    vi = f.ravel()
    okc = ok[t]
    t, vi, wt = t[okc], vi[okc], cw.ravel()[okc]
    ni = n[vi]
    t1, t2 = frame(ni)
    wc, uc, vc = w[t], u[t], vv[t]
    nd = _dot(wc, ni)
    perp = ni - nd[:, None] * wc
    with np.errstate(invalid="ignore", divide="ignore"):
        dperp = (wc + ni) / (1.0 + nd)[:, None]
    ru = uc - dperp * _dot(uc, perp)[:, None]
    rv = vc - dperp * _dot(vc, perp)[:, None]
    flip = nd <= -1.0
    ru[flip], rv[flip] = -uc[flip], -vc[flip]
    u1, v1, u2, v2 = _dot(t1, ru), _dot(t1, rv), _dot(t2, ru), _dot(t2, rv)
    Ec, Fc, Gc = E[t], F[t], G[t]
    acc = np.zeros((nv, 4))
    np.add.at(acc, vi, np.stack([wt * (Ec * u1 * u1 + 2.0 * Fc * u1 * v1 + Gc * v1 * v1),
                                 wt * (Ec * u1 * u2 + Fc * (u1 * v2 + u2 * v1) + Gc * v1 * v2),
                                 wt * (Ec * u2 * u2 + 2.0 * Fc * u2 * v2 + Gc * v2 * v2), wt], 1))
    has_n = (n != 0).any(1)
    good = has_n & (acc[:, 3] > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        k1, k2, x, y = eigen(acc[:, 0] / acc[:, 3], acc[:, 1] / acc[:, 3], acc[:, 2] / acc[:, 3])
    T1, T2 = frame(n)
    d1, d2 = directions(x[:, None] * T1 + y[:, None] * T2, n)
    return _finish(good, k1, k2, d1, d2)


def _finish(good, k1, k2, d1, d2):
    k1 = np.where(good, k1, np.nan); k2 = np.where(good, k2, np.nan)
    d1 = np.where(good[:, None], d1, 0.0); d2 = np.where(good[:, None], d2, 0.0)
    return k1, k2, d1, d2


def ball_neighbours(v, r, rows=None):
    """For each vertex (or each of `rows`), the indices j != i with d2 < (T)(r r), d2 in v's dtype as
    ((dx dx + dy dy) + dz dz)."""
    T = v.dtype.type
    r2 = T(r * r)
    tree = cKDTree(v.astype(np.float64))
    rows = np.arange(len(v)) if rows is None else rows
    cand = tree.query_ball_point(v[rows].astype(np.float64), r * (1 + 1e-5) + 1e-30)
    out = []
    for i, c in zip(rows, cand):
        c = np.asarray(c, np.int64)
        d = v[i] - v[c]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        out.append(c[(d2 < r2) & (c != i)])
    return out


def monge(q, r, n, t1, t2):
    a, b, c, d, e = q
    g = np.sqrt(1.0 + d * d + e * e)
    l11 = np.sqrt(1.0 + d * d); l21 = d * e / l11; l22 = np.sqrt((1.0 + e * e) - l21 * l21)
    p, s = 1.0 / l11, 1.0 / l22
    t = -l21 * p * s
    B00, B01, B11 = 2.0 * a, b, 2.0 * c
    sc = -1.0 / (r * g)
    S00 = p * p * B00 * sc
    S01 = p * (t * B00 + s * B01) * sc
    S11 = (t * t * B00 + 2.0 * t * s * B01 + s * s * B11) * sc
    k1, k2, w0, w1 = eigen(np.float64(S00), np.float64(S01), np.float64(S11))
    v0, v1 = p * w0 + t * w1, s * w1
    d1 = v0 * (t1 + d * n) + v1 * (t2 + e * n)
    nf = n - d * t1 - e * t2
    nf = nf / np.sqrt(_dot(nf, nf))
    d1, d2 = directions(d1, nf)
    return k1, k2, d1, d2


def ball(v, f, r, rows=None):
    n, _, _ = vertex_normals(np.asarray(v, np.float64), f)
    rows = np.arange(len(v)) if rows is None else np.asarray(rows)
    nb = ball_neighbours(v, r, rows)
    vd = v.astype(np.float64)
    k1 = np.full(len(rows), np.nan); k2 = np.full(len(rows), np.nan)
    d1 = np.zeros((len(rows), 3)); d2 = np.zeros((len(rows), 3))
    for o, (i, js) in enumerate(zip(rows, nb)):
        ni = n[i]
        if not (ni != 0).any() or len(js) < 5:
            continue
        t1, t2 = frame(ni)
        off = vd[js] - vd[i]
        x, y, z = _dot(off, t1) / r, _dot(off, t2) / r, _dot(off, ni) / r
        phi = np.stack([x * x, x * y, y * y, x, y], 1)
        M = phi.T @ phi
        rhs = phi.T @ z
        big = M.diagonal().max()
        L = np.zeros((5, 5))
        bad = False
        for k in range(5):
            piv = M[k, k] - np.dot(L[k, :k], L[k, :k])
            if not piv > 1e-12 * big:
                bad = True
                break
            L[k, k] = np.sqrt(piv)
            for i2 in range(k + 1, 5):
                L[i2, k] = (M[i2, k] - np.dot(L[i2, :k], L[k, :k])) / L[k, k]
        if bad:
            continue
        yv = rhs.copy()
        for i2 in range(5):
            yv[i2] = (yv[i2] - np.dot(L[i2, :i2], yv[:i2])) / L[i2, i2]
        for i2 in range(4, -1, -1):
            yv[i2] = (yv[i2] - np.dot(L[i2 + 1:, i2], yv[i2 + 1:])) / L[i2, i2]
        k1[o], k2[o], d1[o], d2[o] = monge(yv, r, ni, t1, t2)
    return k1, k2, d1, d2


def curvatures(v, f, r=-1.0, rows=None):
    if r > 0:
        return ball(v, f, r, rows)
    out = ring(v, f)
    return out if rows is None else tuple(o[rows] for o in out)


# ---- meshes -----------------------------------------------------------------------------------------------------------
def _bunny():
    import os
    g = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    return np.load(os.path.join(g, "bunny_vertices.npy")).astype(np.float64), np.load(os.path.join(g, "bunny_faces.npy")).astype(np.int64)


def _grid(k=24, fn=lambda x, y: 0.3 * np.sin(2 * x) * np.cos(3 * y)):
    """An open height field over [-1, 1]^2 on a k x k vertex grid, faces facing +z."""
    g = np.linspace(-1.0, 1.0, k)
    X, Y = np.meshgrid(g, g, indexing="ij")
    v = np.stack([X.ravel(), Y.ravel(), fn(X, Y).ravel()], 1)
    idx = np.arange(k * k).reshape(k, k)
    a, b, c, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel(), idx[:-1, 1:].ravel()
    return v, np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)])


def _degenerate():
    """icosphere(2) plus a face with a repeated corner, a zero-area face through a new vertex at the position of one of
    its corners, a face on an edge that two faces already share (non-manifold) and an isolated vertex that no face uses."""
    v, f = icosphere(2)
    a, b = f[0, 0], f[0, 1]
    mid = v[a].copy()
    tip = 1.3 * v[f[0]].mean(0)
    v = np.concatenate([v, [mid, tip, [5.0, 5.0, 5.0]]])
    nv = len(v)
    f = np.concatenate([f, [[f[1, 0], f[1, 0], f[1, 1]], [a, nv - 3, b], [a, b, nv - 2]]])
    return v, f


def _mean_edge(v, f):
    v = np.asarray(v, np.float64)
    return float(np.linalg.norm(v[f[:, 0]] - v[f[:, 1]], axis=1).mean())


MESHES = {
    "icosphere3": lambda: icosphere(3, jitter=0.01, seed=3),
    "torus": lambda: torus(48, 24),
    "bunny": _bunny,
    "grid": _grid,
    "degenerate": _degenerate,
}


# ---- CPU: the restatement on analytic surfaces -----------------------------------------------------------------------
@pytest.mark.parametrize("R", [0.5, 2.0])
def test_restatement_sphere_one_ring(R):
    v, f = icosphere(5)
    k1, k2, d1, d2 = curvatures(R * v, f)
    assert np.abs(k1 * R - 1).max() < 1e-11 and np.abs(k2 * R - 1).max() < 1e-11
    k1, k2, _, _ = curvatures(R * v, f[:, ::-1].copy())
    assert np.abs(k1 * R + 1).max() < 1e-11 and np.abs(k2 * R + 1).max() < 1e-11


def test_restatement_sphere_ball():
    # measured 0.0104 at level 4, r = 3 mean edge lengths, R = 2
    v, f = icosphere(4)
    v = 2 * v
    r = 3 * _mean_edge(v, f)
    k1, k2, _, _ = curvatures(v, f, r)
    assert np.abs(k1 * 2 - 1).max() < 0.02 and np.abs(k2 * 2 - 1).max() < 0.02
    k1, k2, _, _ = curvatures(v, f[:, ::-1].copy(), r)
    assert np.abs(k1 * 2 + 1).max() < 0.02 and np.abs(k2 * 2 + 1).max() < 0.02


def _torus_truth(nu, nv):
    phi = np.tile(np.arange(nv) * 2 * np.pi / nv, nu)
    u = np.repeat(np.arange(nu) * 2 * np.pi / nu, nv)
    meridian = np.stack([-np.sin(phi) * np.cos(u), -np.sin(phi) * np.sin(u), np.cos(phi)], 1)
    return 1 / 0.35, np.cos(phi) / (1 + 0.35 * np.cos(phi)), meridian


def test_restatement_torus():
    # measured at 256 x 64: 4.3e-4 (tube), 3.1e-3 (ring), 1 - |d1 . meridian| <= 3.1e-8
    v, f = torus(256, 64)
    kt, kr, mer = _torus_truth(256, 64)
    k1, k2, d1, d2 = curvatures(v, f)
    assert np.abs(k1 - kt).max() < 1e-3 and np.abs(k2 - kr).max() < 5e-3
    assert (1 - np.abs((d1 * mer).sum(1))).max() < 1e-6


@pytest.mark.parametrize("r", [-1.0, 0.2])
def test_restatement_saddle(r):
    # z = (x^2 - y^2) / 2 at the origin: k = +-1, k1 along y with faces facing +z.  Measured: one-ring 0.9975, ball exact
    v, f = _grid(41, lambda x, y: 0.5 * (x * x - y * y))
    o = 20 * 41 + 20
    k1, k2, d1, d2 = curvatures(v, f, r)
    tol = 5e-3 if r < 0 else 1e-9
    assert abs(k1[o] - 1) < tol and abs(k2[o] + 1) < tol
    assert abs(d1[o, 1]) > 1 - 1e-9 and abs(d2[o, 0]) > 1 - 1e-9


@pytest.mark.parametrize("r", [-1.0, 0.3])
def test_restatement_plane(r):
    v, f = _grid(16, lambda x, y: 0 * x)
    k1, k2, _, _ = curvatures(v, f, r)
    assert np.nanmax(np.abs(k1)) < 1e-12 and np.nanmax(np.abs(k2)) < 1e-12


def test_restatement_degenerate():
    v, f = _degenerate()
    for r in (-1.0, 0.4):
        k1, k2, d1, d2 = curvatures(v, f, r)
        for i in (len(v) - 1, len(v) - 3):    # the isolated vertex, the copy that only a zero-area face uses
            assert np.isnan(k1[i]) and np.isnan(k2[i]) and not d1[i].any() and not d2[i].any()
        assert np.isfinite(k1[:len(v) - 3]).all()


def test_argument_errors_before_any_device_call(pcu):
    v, f = icosphere(1)
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError, match="r must be finite"):
            pcu.mesh_principal_curvatures(v, f, bad)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.mesh_principal_curvatures(v.astype(np.int32), f)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.mesh_mean_and_gaussian_curvatures(v, f.astype(np.float32))
    with pytest.raises(ValueError, match="zero elements"):
        pcu.mesh_principal_curvatures(v[:0], f)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.mesh_principal_curvatures(v[:, :2].copy(), f)
    with pytest.raises(ValueError, match="must be a NumPy array"):
        pcu.mesh_principal_curvatures(v.tolist(), f)


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _compare(got, want, dtype):
    """All four outputs against the restatement: the same NaN pattern; k to 1e-10 max|k| in fp64 and to 2 fp32 spacings
    (plus that) in fp32; directions up to the documented sign rule away from near-umbilics."""
    k1, k2, d1, d2 = (np.asarray(x, np.float64) for x in got)
    w1, w2, e1, e2 = want
    nan = np.isnan(w1)
    assert (np.isnan(k1) == nan).all() and (np.isnan(k2) == nan).all()
    assert not d1[nan].any() and not d2[nan].any()
    ok = ~nan
    if not ok.any():
        return
    scale = max(np.abs(w1[ok]).max(), np.abs(w2[ok]).max(), 1e-300)
    for g, w in ((k1, w1), (k2, w2)):
        tol = 1e-10 * scale + (2 * np.spacing(np.abs(w[ok]).astype(np.float32)).astype(np.float64) if dtype == np.float32 else 0.0)
        assert (np.abs(g[ok] - w[ok]) <= tol).all(), np.abs(g[ok] - w[ok]).max()
    # the sign rule holds on every determined vertex; each direction is a unit vector and d2 = n x d1 is orthogonal to d1
    j = np.argmax(np.abs(d1[ok]), 1)
    assert (d1[ok][np.arange(ok.sum()), j] > 0).all() or dtype == np.float32
    assert np.abs(np.linalg.norm(d1[ok], axis=1) - 1).max() < 1e-6 and np.abs((d1[ok] * d2[ok]).sum(1)).max() < 1e-6
    gap = (w1 - w2)[ok] / scale
    far = gap > 1e-4
    dir_tol = (1e-12 if dtype == np.float64 else 1e-6) / np.maximum(gap, 1e-300) + (1e-9 if dtype == np.float64 else 1e-5)
    for g, w in ((d1, e1), (d2, e2)):
        g, w = g[ok], w[ok]
        err = np.minimum(np.abs(g - w).max(1), np.abs(g + w).max(1))
        assert (err[far] <= dir_tol[far]).all(), err[far].max()
        # where two components tie in magnitude the sign rule may choose either; elsewhere it fixes the sign
        second = np.sort(np.abs(w), 1)[:, -2]
        clear = far & (np.abs(w).max(1) - second > 1e-6)
        assert (np.abs(g - w).max(1)[clear] <= dir_tol[clear] + 1e-6 * (dtype == np.float32)).all()


KINDS = ["int32", "int64", "uint32", "uint64"]
FORMS = ["numpy", "cpu", "cuda"]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ring", "ball"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(MESHES))
def test_against_restatement(pcu, name, dtype, mode):
    v, f = MESHES[name]()
    v = v.astype(dtype)
    r = 3 * _mean_edge(v, f) if mode == "ball" else -1.0
    i = list(MESHES).index(name) + 2 * (dtype == np.float64) + (mode == "ball")
    kind, form = KINDS[i % 4], FORMS[i % 3]
    got = pcu.mesh_principal_curvatures(to_form(form, v), to_form(form, f.astype(kind)), r)
    got = [to_numpy(x, form) for x in got]
    assert all(x.dtype == dtype for x in got)
    assert got[0].shape == (len(v),) and got[2].shape == (len(v), 3)
    rows = None
    if mode == "ball" and len(v) > 3000:
        rows = np.random.default_rng(1).choice(len(v), 1500, replace=False)
        got = [x[rows] for x in got]
    _compare(got, curvatures(v, f, r, rows), dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("r", [-1.0, 0.35])
def test_every_kind_and_form(pcu, r):
    v, f = icosphere(2, jitter=0.02, seed=5)
    want = curvatures(v, f, r)
    first = None
    for kind in KINDS:
        for form in FORMS:
            got = [to_numpy(x, form) for x in pcu.mesh_principal_curvatures(to_form(form, v), to_form(form, f.astype(kind)), r)]
            _compare(got, want, np.float64)
            if first is None:
                first = got
            assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, first))


@pytest.mark.gpu
def test_cuda_stays_on_device(pcu):
    import torch
    v, f = icosphere(2)
    out = pcu.mesh_principal_curvatures(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert all(isinstance(o, torch.Tensor) and o.is_cuda for o in out)
    kh, kg = pcu.mesh_mean_and_gaussian_curvatures(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert kh.is_cuda and kg.is_cuda


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_sphere_and_reversed(pcu, dtype):
    v, f = icosphere(5)
    R = 2.0
    v = (R * v).astype(dtype)
    # calibrated with the restatement: 3.6e-13 in fp64; 2.1e-5 once the vertices are rounded to fp32 (off the sphere);
    # ball at 3 mean edge lengths 2.7e-3
    tol = 1e-11 if dtype == np.float64 else 5e-5
    k1, k2, _, _ = pcu.mesh_principal_curvatures(v, f)
    assert np.abs(k1 * R - 1).max() < tol and np.abs(k2 * R - 1).max() < tol
    k1, k2, _, _ = pcu.mesh_principal_curvatures(v, f[:, ::-1].copy())
    assert np.abs(k1 * R + 1).max() < tol and np.abs(k2 * R + 1).max() < tol
    r = 3 * _mean_edge(v, f)
    k1, k2, _, _ = pcu.mesh_principal_curvatures(v, f, r)
    assert np.abs(k1 * R - 1).max() < 6e-3 and np.abs(k2 * R - 1).max() < 6e-3


@pytest.mark.gpu
def test_torus_and_saddle(pcu):
    v, f = torus(256, 64)
    kt, kr, mer = _torus_truth(256, 64)
    k1, k2, d1, _ = pcu.mesh_principal_curvatures(v, f)
    assert np.abs(k1 - kt).max() < 1e-3 and np.abs(k2 - kr).max() < 5e-3
    assert (1 - np.abs((d1 * mer).sum(1))).max() < 1e-6
    v, f = _grid(41, lambda x, y: 0.5 * (x * x - y * y))
    o = 20 * 41 + 20
    for r, tol in ((-1.0, 5e-3), (0.2, 1e-9)):
        k1, k2, d1, d2 = pcu.mesh_principal_curvatures(v, f, r)
        assert abs(k1[o] - 1) < tol and abs(k2[o] + 1) < tol
        assert d1[o, 1] > 1 - 1e-9 and abs(d2[o, 0]) > 1 - 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("r", [-1.0, 0.25])
def test_invariance(pcu, r):
    v, f = icosphere(3, jitter=0.01, seed=7)
    k1, k2, d1, d2 = pcu.mesh_principal_curvatures(v, f, r)
    scale = np.abs(np.concatenate([k1, k2])).max()
    ok = (k1 - k2) > 1e-3 * scale
    t1, t2, _, _ = pcu.mesh_principal_curvatures(v + np.array([3.0, -2.0, 0.5]), f, r)
    assert np.abs(t1 - k1).max() < 1e-7 * scale and np.abs(t2 - k2).max() < 1e-7 * scale
    s = 2.5
    s1, s2, _, _ = pcu.mesh_principal_curvatures(s * v, f, s * r)
    assert np.abs(s1 - k1 / s).max() < 1e-9 * scale and np.abs(s2 - k2 / s).max() < 1e-9 * scale
    a = 0.7
    Q = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]) @ np.array(
        [[1, 0, 0], [0, np.cos(0.4), -np.sin(0.4)], [0, np.sin(0.4), np.cos(0.4)]])
    q1, q2, e1, e2 = pcu.mesh_principal_curvatures(v @ Q.T, f, r)
    assert np.abs(q1 - k1).max() < 1e-7 * scale and np.abs(q2 - k2).max() < 1e-7 * scale
    for e, d in ((e1, d1), (e2, d2)):
        rd = d[ok] @ Q.T
        err = np.minimum(np.abs(e[ok] - rd).max(1), np.abs(e[ok] + rd).max(1))
        assert err.max() < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("r", [-1.0, 0.3])
def test_deterministic_and_wrapper(pcu, r):
    v, f = _bunny()
    r = r if r < 0 else 4 * _mean_edge(v, f)
    a = pcu.mesh_principal_curvatures(v, f, r)
    b = pcu.mesh_principal_curvatures(v, f, r)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    kh, kg = pcu.mesh_mean_and_gaussian_curvatures(v, f, r)
    assert np.array_equal(kh, 0.5 * (a[0] + a[1]), equal_nan=True) and np.array_equal(kg, a[0] * a[1], equal_nan=True)


@pytest.mark.gpu
def test_bad_corner(pcu):
    v, f = icosphere(1)
    f = f.copy()
    f[3, 1] = len(v)
    for r in (-1.0, 0.5):
        with pytest.raises(ValueError, match="1 faces have a corner outside"):
            pcu.mesh_principal_curvatures(v, f, r)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ring", "ball"])
def test_full_size(pcu, mode):
    """The 1.31e6-face icosphere(8) of radius 2: every vertex against 1 / R (one-ring: 1e-11 relative; ball at 3 mean
    edge lengths: measured 4.2e-5 on 3000 sampled vertices), sampled vertices against the restatement."""
    import torch
    v, f = icosphere(8)
    v = 2.0 * v
    r = 3 * _mean_edge(v, f) if mode == "ball" else -1.0
    out = pcu.mesh_principal_curvatures(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), r)
    k1, k2, d1, d2 = (o.cpu().numpy() for o in out)
    tol = 1e-11 if mode == "ring" else 2e-4
    assert np.abs(k1 * 2 - 1).max() < tol and np.abs(k2 * 2 - 1).max() < tol
    rows = np.random.default_rng(2).choice(len(v), 400, replace=False)
    _compare((k1[rows], k2[rows], d1[rows], d2[rows]), curvatures(v, f, r, rows), np.float64)
