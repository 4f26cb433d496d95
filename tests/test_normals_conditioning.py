"""The point-cloud normals against an exact plane fit, at the neighbourhoods a plane fit gets wrong (SURVEY.md N1).

The reference is `exact_normal`: the scatter matrix X^T X of a neighbourhood's offsets X, formed from the fp64 offsets
at 60 digits, and its eigenvector of the smallest eigenvalue from mpmath.  The offsets are the ones the kernels see:
the difference rounded in the cloud's dtype, widened to fp64, times the 'rbf' weight.  So the reference is the exact
right singular vector of exactly the matrix the kernels fit, and any error is theirs.

Metric and bound.  The error is sin(theta) = |n x n_ref| / |n|.  Its bound on a row with singular values
s1 >= s2 >= s3 is
    sin(theta) <= C u s1 / (s2 - s3),   u = 2^-53, C = 64,        plus 2^-23 for float32 outputs (their rounding).
Derivation of C, for PlaneFit (csrc/plane_fit.h) after its refining pass.  The pass forms Y = fl(sXV): each entry is a
3-term dot product, |dY| <= gamma_3 |sX| |V|, so Y is the exact product for a perturbed X with
||dX||_2 <= ||dX||_F <= 3 gamma_3 ||X||_F <= 3 * 3u * sqrt(3) s1 ~ 16u s1.  Forming Y^T Y with k-term sums adds
|dB_ij| <= gamma_k ||y_i|| ||y_j||, which perturbs the pair (2, 3) by gamma_k s2 s3 over a gap s2^2 - s3^2, i.e.
by <= (k u / 2) s1 / (s2 - s3); bounds of this kind are worst cases and rounding errors add up like sqrt(k) in
practice, so the neighbourhoods here (k <= 40) contribute at most ~ 4u s1 / (s2 - s3) typically, 20u at worst.
Jacobi's stopping test leaves at most u s1 / (s2 - s3) / 2 (plane_fit.h), the product V W and the normalisation a
few u more.  By Wedin's theorem a perturbation dX turns the singular vector by at most ||dX|| / (s2 - s3), so the sum
is ~ (16 + 20 + 1 + 4) u s1 / (s2 - s3) ~ 41 u s1 / (s2 - s3); C = 64 leaves 1.5x for the 'rbf' weights the device
computes in another order of operations than numpy could (a relative row perturbation of a few u).  A kernel that
fitted the scatter matrix alone would be off by ~ u s1^2 / (s2^2 - s3^2), i.e. s1 / (s2 + s3) times the bound: the
elongated cases below make that 10^2 ... 10^7.

Rows with s2 = s3 (the normal is any unit vector of a plane) get property checks: unit length and perpendicular to
the top singular vector within C u s1 / (s1 - s2).

The rules where no plane is defined (plane_fit.h): fewer than 3 offsets give the zero vector (the oracle pads numpy's
thin V with zeros), all-zero offsets give (0, 0, 1) (numpy's SVD of a zero matrix has V = I).  With view directions
these are oriented and filtered as usual: sign(0) = 0 and acos(0) = pi/2, so a zero normal is kept exactly when
drop_angle_threshold >= pi/2."""
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
U = 2.0 ** -53
C = 64.0
F32_OUT = 2.0 ** -23
DBL_MAX = np.finfo(np.float64).max


# ---- the exact reference --------------------------------------------------------------------------------------------
def exact_fit(off):
    """(normal, top, s1, s2, s3) of the fp64 offsets `off` (m, 3): the eigenvectors of the smallest and the largest
    eigenvalue of the exact scatter matrix, at 60 digits, and the singular values."""
    import mpmath
    mp = mpmath.mp
    mp.dps = 60
    X = [[mpmath.mpf(float(v)) for v in r] for r in np.asarray(off, dtype=np.float64)]
    M = mpmath.matrix(3, 3)
    for i in range(3):
        for j in range(i, 3):
            M[i, j] = M[j, i] = mpmath.fsum(r[i] * r[j] for r in X)
    E, Q = mp.eigsy(M)                                 # ascending
    s = [float(mpmath.sqrt(max(E[t], 0))) for t in (2, 1, 0)]
    n = np.array([float(Q[t, 0]) for t in range(3)])
    top = np.array([float(Q[t, 2]) for t in range(3)])
    return n / np.linalg.norm(n), top / np.linalg.norm(top), s[0], s[1], s[2]


def exact_normal(off):
    return exact_fit(off)[0]


def exact_top(off):
    return exact_fit(off)[1]


def _sin(n, ref):
    n = np.asarray(n, dtype=np.float64)
    return float(np.linalg.norm(np.cross(n, ref)) / np.linalg.norm(n))


def _bound(s1, s2, s3, dtype):
    return C * U * s1 / (s2 - s3) + (F32_OUT if dtype == np.float32 else 0.0)


def assert_rows_within_bound(normals, offsets, dtype, label=""):
    """normals[t] against exact_normal(offsets[t]) for every t: the per-row bound, or the properties of a tied row.
    Returns the number of rows held to the bound."""
    bounded = 0
    for t, (n, off) in enumerate(zip(normals, offsets)):
        n = np.asarray(n, dtype=np.float64)
        assert abs(np.linalg.norm(n) - 1.0) <= (1e-6 if dtype == np.float32 else 1e-14), (label, t, n)
        ref, top, s1, s2, s3 = exact_fit(off)
        if s1 > 0 and s2 - s3 > 1e-30 * s1:
            bounded += 1
            assert _sin(n, ref) <= _bound(s1, s2, s3, dtype), (label, t, _sin(n, ref), _bound(s1, s2, s3, dtype), s1, s2, s3)
        if s1 > s2:
            # perpendicular to the top singular vector (the line of a collinear neighbourhood)
            tol = C * U * s1 / (s1 - s2) + (F32_OUT if dtype == np.float32 else 0.0)
            assert abs(np.dot(n, top)) / np.linalg.norm(n) <= tol, (label, t, float(np.dot(n, top)), tol)
    return bounded


# ---- the neighbourhoods the kernels fit -----------------------------------------------------------------------------
def knn_offsets(oracle, pts, k, rows):
    _, nn = oracle.k_nearest_neighbors(pts, pts, k, True)
    nn = nn.reshape(len(pts), k)
    return [(pts[nn[i]] - pts[i]).astype(np.float64) for i in rows]


def wendland(r):
    v1, v2 = 1.0 - r, 4 * r + 1.0
    return v1 * v1 * v1 * v1 * v2             # the kernel's order of operations


def ball_offsets(oracle, pts, radius, rows, weight="constant"):
    nbrs, d2s = oracle.ball_neighbourhoods(pts, radius)
    out = []
    for i in rows:
        off = (pts[nbrs[i]] - pts[i]).astype(np.float64)
        if weight == "rbf":
            off = off * wendland(np.sqrt(d2s[i].astype(np.float64)) / float(radius))[:, None]
        out.append(off)
    return out


def _run(fn, pts, *args, **kw):
    """fn on numpy inputs and on CUDA tensors (view directions included): both give the same bits, and the NumPy
    seed is the same for both; returns the numpy result."""
    import torch
    np.random.seed(5)
    i, n = fn(pts, *args, **kw)
    tkw = {a: torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v for a, v in kw.items()}
    np.random.seed(5)
    ti, tn = fn(torch.from_numpy(np.ascontiguousarray(pts)).cuda(), *args, **tkw)
    assert ti.is_cuda and tn.is_cuda
    assert np.array_equal(ti.cpu().numpy(), i) and np.array_equal(tn.cpu().numpy(), n, equal_nan=True)
    assert i.dtype == np.int64 and n.dtype == pts.dtype
    return i, n


def estimate(pcu, kind, pts, param, dirs=None, thr=np.pi / 2, weight="constant", min_pts=3):
    if kind == "knn":
        return _run(pcu.estimate_point_cloud_normals_knn, pts, param, view_directions=dirs, drop_angle_threshold=thr)
    return _run(pcu.estimate_point_cloud_normals_ball, pts, param, view_directions=dirs, drop_angle_threshold=thr,
                min_pts_per_ball=min_pts, weight_function=weight)


def offsets_of(oracle, kind, pts, param, rows, weight="constant"):
    if kind == "knn":
        return knn_offsets(oracle, pts, param, rows)
    return ball_offsets(oracle, pts, param, rows, weight)


def _rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q


# ---- families ---------------------------------------------------------------------------------------------------------
def sphere(n, noise, seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v * (1.0 + noise * rng.normal(size=(n, 1)))


def plane(n, noise, seed):
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.random((n, 2)) * 2 - 1, noise * rng.normal(size=(n, 1))], axis=1)
    return p @ _rotation(seed).T


def cylinder(n, noise, seed, radius=0.05):
    rng = np.random.default_rng(seed)
    t = rng.random(n) * 2 * np.pi
    r = radius * (1.0 + noise * rng.normal(size=n))
    return np.stack([r * np.cos(t), r * np.sin(t), rng.random(n) * 0.4], axis=1) @ _rotation(seed + 1).T


def ribbon(ratio, seed, columns=400, rows=3, h=1e-2):
    """A rotated lattice strip: spacing h along its length, h * ratio across it (s2 / s1 ~ ratio / 2)."""
    i, j = np.meshgrid(np.arange(columns), np.arange(rows), indexing="ij")
    p = np.stack([i.ravel() * h, j.ravel() * h * ratio, np.zeros(i.size)], axis=1)
    return p @ _rotation(seed).T + np.array([0.1, -0.2, 0.3])


def helix(ratio, n=2000, h=1e-3):
    """A thin helical wire: pitch h per point, radius h * ratio, a tenth of a turn per ten points."""
    t = np.arange(n) * (2 * np.pi / 100)
    return np.stack([h * ratio * np.cos(t), h * ratio * np.sin(t), np.arange(n) * h], axis=1) @ _rotation(3).T


SMOOTH = {   # name -> (points, k, ball radius (squared reach))
    "sphere_0": (lambda: sphere(20000, 0.0, 1), 12, 2.4e-3),
    "sphere_1e-4": (lambda: sphere(20000, 1e-4, 2), 16, 2.4e-3),
    "sphere_1e-2": (lambda: sphere(20000, 1e-2, 3), 20, 2.4e-3),
    "plane_1e-6": (lambda: plane(20000, 1e-6, 4), 12, 6e-4),
    "plane_1e-3": (lambda: plane(20000, 1e-3, 5), 12, 6e-4),
    "cylinder_1e-3": (lambda: cylinder(20000, 1e-3, 6), 12, 2e-5),
}
SAMPLE = 2000      # rows of a large cloud compared with exact_normal


def _sample_rows(kept, seed=0):
    rng = np.random.default_rng(seed)
    return np.sort(rng.choice(kept, size=min(SAMPLE, len(kept)), replace=False))


KINDS = ["knn", "ball"]
DTYPES = [np.float32, np.float64]


# ---- CPU: the reference itself, and the host build of the fit -------------------------------------------------------------
ELONGATED = [1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7]


def _elongated_offsets(ratio, scale_exp=0):
    pts = ribbon(ratio, 7, columns=60) * 2.0 ** scale_exp
    d = pts[:, None, :] - pts[None, :, :]
    d2 = np.einsum("ijk,ijk->ij", d, d)
    nn = np.argsort(d2, axis=1, kind="stable")[:, :12]
    return [(pts[nn[i]] - pts[i]) for i in range(0, len(pts), 7)]


def test_exact_reference_agrees_with_numpy_svd():
    """numpy's fp64 SVD, which stands in for exact_normal on most rows of the large clouds, is within the per-row
    bound of it on the elongated and the scaled families -- and the bound is tight enough to matter: the normal of
    the scatter matrix alone misses it on the elongated rows."""
    scatter_misses = 0
    for ratio in ELONGATED:
        for e in (0, -490, -504, 300):
            for off in _elongated_offsets(ratio, e):
                ref, _, s1, s2, s3 = exact_fit(off)
                v = np.linalg.svd(off)[2][2]
                assert _sin(v, ref) <= C * U * s1 / (s2 - s3), (ratio, e, _sin(v, ref), s1, s2, s3)
                if e == 0:
                    w, q = np.linalg.eigh(off.T @ off)
                    scatter_misses += _sin(q[:, 0], ref) > C * U * s1 / (s2 - s3)
    assert scatter_misses > 0


def _host_fit_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("plane_fit") / "fit")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "point-cloud-utils_b200", "csrc"),
                    os.path.join(HERE, "plane_fit_host", "fit.cpp"), "-o", exe], check=True, capture_output=True)
    return exe


@pytest.fixture(scope="module")
def host_fit(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = _host_fit_exe(tmp_path_factory)

    def fit(offsets):
        blob = [np.array([len(offsets)], dtype=np.int64).tobytes()]
        for off in offsets:
            off = np.ascontiguousarray(off, dtype=np.float64).reshape(-1, 3)
            blob += [np.array([len(off)], dtype=np.int64).tobytes(), off.tobytes()]
        out = subprocess.run([exe], input=b"".join(blob), capture_output=True, check=True)
        return np.frombuffer(out.stdout, dtype=np.float64).reshape(-1, 3)
    return fit


def test_host_fit_elongated_and_scaled(host_fit):
    """Cases 2 and 3 on the CPU build of the fit: every elongated row within the bound, and the same bits at every
    power-of-two scale of the offsets, including where their squares overflow or underflow."""
    for ratio in ELONGATED:
        offs = _elongated_offsets(ratio)
        got = host_fit(offs)
        assert assert_rows_within_bound(got, offs, np.float64, "ratio %g" % ratio) == len(offs)
        for e in (-900, -504, -300, 300, 511):
            assert np.array_equal(host_fit([o * 2.0 ** e for o in offs]), got), (ratio, e)


def test_host_fit_degenerate_rows(host_fit):
    """Cases 4-7 on the CPU build: a hexagon whose squared offsets sum past DBL_MAX, coincident points, lines, k < 3."""
    rho = 0.45 * np.sqrt(DBL_MAX)
    ang = np.arange(6) * np.pi / 3
    hexagon = np.stack([rho * np.cos(ang), rho * np.sin(ang), np.zeros(6)], axis=1)
    offs = [hexagon - hexagon[i] for i in range(6)]
    assert not np.isfinite(np.einsum("ij,ij->", offs[0], offs[0]))
    got = host_fit(offs)
    assert np.array_equal(np.abs(got), np.tile([0.0, 0.0, 1.0], (6, 1)))
    tilted = hexagon @ _rotation(11).T * 0.5
    offs = [tilted - tilted[i] for i in range(6)]
    assert assert_rows_within_bound(host_fit(offs), offs, np.float64, "tilted hexagon") == 6
    # coincident: (0, 0, 1); fewer than three offsets: zero
    assert np.array_equal(host_fit([np.zeros((8, 3)), np.zeros((3, 3))]), [[0, 0, 1], [0, 0, 1]])
    got = host_fit([np.zeros((1, 3)), np.array([[0.0, 0, 0], [1, 2, 3]]), np.zeros((0, 3))])
    assert np.array_equal(got, np.zeros((3, 3)))
    # lines: unit, perpendicular to the line
    t = np.arange(-5, 6, dtype=np.float64)[:, None]
    lines = [t * np.array([1.0, 0, 0]), t * np.array([0, 0, 2.5]), t * _rotation(12)[0], t * _rotation(13)[1] * 1e-200]
    for off in lines:
        n = host_fit([off])[0]
        assert abs(np.linalg.norm(n) - 1) < 1e-15 and abs(np.dot(n, exact_top(off))) <= C * U


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _smooth_cloud(name, dtype):
    return SMOOTH[name][0]().astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", sorted(SMOOTH))
def test_smooth_surfaces(pcu, oracle, name, kind, dtype):
    """Case 1: a sphere, a plane and a thin cylinder at several noise levels, every sampled row within its bound."""
    pts = _smooth_cloud(name, dtype)
    _, k, radius = SMOOTH[name]
    if kind == "ball":
        pts = pts[:5000]                            # the oracle's ball search is brute force
        radius *= 4.0
    param = k if kind == "knn" else radius
    idx, nrm = estimate(pcu, kind, pts, param)
    if kind == "knn":
        assert np.array_equal(idx, np.arange(len(pts)))
    rows = _sample_rows(np.arange(len(idx)))
    offs = offsets_of(oracle, kind, pts, param, idx[rows])
    assert assert_rows_within_bound(nrm[rows], offs, dtype, name) > 0.9 * len(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind,weight", [("knn", "constant"), ("ball", "constant"), ("ball", "rbf")])
def test_elongated_neighbourhoods(pcu, oracle, kind, dtype, weight):
    """Case 2: ribbons with s2 / s1 from 1e-2 down to 1e-7 and a helical wire; every row within its bound."""
    clouds = [ribbon(r, 20 + t) for t, r in enumerate(ELONGATED)] + [helix(r) for r in (1e-2, 1e-4)]
    for t, cloud in enumerate(clouds):
        pts = cloud.astype(dtype)
        param = 12 if kind == "knn" else (6.25e-4 if t < len(ELONGATED) else 3e-5)
        idx, nrm = estimate(pcu, kind, pts, param, weight=weight)
        rows = _sample_rows(np.arange(len(idx)), t)[:300]
        offs = offsets_of(oracle, kind, pts, param, idx[rows], weight)
        assert assert_rows_within_bound(nrm[rows], offs, dtype, "cloud %d" % t) > 0


SCALES = {np.float64: [-300, -200, -100, -50, -1, 1, 50, 100, 200, 300], np.float32: [-40, -20, -1, 1, 20, 40]}
BALL_F64_SCALES = [-100, -50, -1, 1, 50, 90]   # the ball grid's cell-size floor is a float: |0.5 reach| within its range


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_power_of_two_scaling_is_exact(pcu, oracle, kind, dtype):
    """Case 3: the cloud times 2^e gives the same kept indices and the same normal bits as at e = 0 (offsets, the fit's
    scale and the neighbour search all scale exactly).  The ball's radius, a squared reach, scales by 4^e; its sums
    run in the grid's cell order, which scales exactly while the reach stays in the range of its float cell floor."""
    pts = sphere(4000, 1e-3, 31).astype(dtype)
    radius = 0.012
    dirs = sphere(4000, 0.0, 31).astype(dtype)
    param = 12 if kind == "knn" else radius
    plain = estimate(pcu, kind, pts, param)
    thr = float(np.median(np.arccos(np.abs(np.einsum("ij,ij->i", plain[1], dirs[plain[0]]).astype(np.float64)))))
    base = estimate(pcu, kind, pts, param, dirs=dirs, thr=thr)
    assert 0 < len(base[0]) < len(pts)
    scales = SCALES[dtype] if (kind == "knn" or dtype == np.float32) else BALL_F64_SCALES
    for e in scales:
        f = dtype(2.0 ** e)
        p = (pts * f).astype(dtype)
        assert np.array_equal(p / f, pts)
        prm = param if kind == "knn" else radius * 4.0 ** e
        got = estimate(pcu, kind, p, prm, dirs=dirs, thr=thr)
        assert np.array_equal(got[0], base[0]) and np.array_equal(got[1], base[1]), e
        got = estimate(pcu, kind, p, prm)
        assert np.array_equal(got[0], plain[0]) and np.array_equal(got[1], plain[1]), e


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("e", [-504, -500, -495, -490])
def test_power_of_two_scaling_near_underflow(pcu, oracle, kind, e):
    """Case 3, fp64 x 2^e where squared offsets are subnormal or zero: the oracle's kept set and neighbourhoods, and
    every row within its bound."""
    pts = (plane(600, 1e-3, 41) * 2.0 ** e).astype(np.float64)
    param = 12 if kind == "knn" else 0.02 * 4.0 ** e
    idx, nrm = estimate(pcu, kind, pts, param)
    ref_i, _ = (oracle.estimate_point_cloud_normals_knn(pts, param) if kind == "knn"
                else oracle.estimate_point_cloud_normals_ball(pts, param))
    assert np.array_equal(idx, ref_i) and len(idx) > 0
    offs = offsets_of(oracle, kind, pts, param, idx)
    assert assert_rows_within_bound(nrm, offs, np.float64, "e=%d" % e) > 0.9 * len(idx)


def _hexagons(rho, tilt):
    ang = np.arange(6) * np.pi / 3
    h = np.stack([rho * np.cos(ang), rho * np.sin(ang), np.zeros(6)], axis=1)
    return h @ _rotation(50).T if tilt else h


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("tilt", [False, True])
def test_scatter_overflow(pcu, oracle, kind, tilt):
    """Case 4: six points on a circle of radius 0.45 sqrt(DBL_MAX): every pairwise d^2 is finite, so every point is a
    neighbour of every other, but a sum of squared offsets exceeds DBL_MAX.  The normal is the plane's."""
    pts = _hexagons(0.45 * np.sqrt(DBL_MAX), tilt)
    d = pts[:, None, :] - pts[None, :, :]
    with np.errstate(over="ignore"):
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        assert np.isfinite(d2).all() and not np.isfinite(np.sum(d[0] * d[0]))
    param = 6 if kind == "knn" else DBL_MAX
    for weight in (["constant"] if kind == "knn" else ["constant", "rbf"]):
        idx, nrm = estimate(pcu, kind, pts, param, weight=weight)
        assert np.array_equal(idx, np.arange(6))
        offs = offsets_of(oracle, kind, pts, param, idx, weight)
        assert assert_rows_within_bound(nrm, offs, np.float64) == 6
        if not tilt:
            assert np.array_equal(np.abs(nrm), np.tile([0.0, 0.0, 1.0], (6, 1)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_coincident_neighbourhoods(pcu, oracle, kind, dtype):
    """Case 5: clusters of coincident points (each at least k / min_pts_per_ball copies, far apart): the scatter is zero
    and the normal is (0, 0, 1), numpy's; with view directions it is oriented and filtered as usual."""
    rng = np.random.default_rng(60)
    centres = rng.random((40, 3)) * 100
    copies = rng.integers(8, 14, size=40)
    pts = np.repeat(centres, copies, axis=0).astype(dtype)
    dirs = rng.normal(size=pts.shape)
    dirs = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True)).astype(dtype)
    param = 8 if kind == "knn" else 1.0
    idx, nrm = estimate(pcu, kind, pts, param, min_pts=8)
    assert np.array_equal(idx, np.arange(len(pts)))
    assert np.array_equal(nrm, np.tile(np.array([0, 0, 1], dtype=dtype), (len(pts), 1)))
    for thr in (np.deg2rad(60.0), np.pi / 2, np.pi):
        idx, nrm = estimate(pcu, kind, pts, param, dirs=dirs, thr=thr, min_pts=8)
        ref_i, ref_n = (oracle.estimate_point_cloud_normals_knn(pts, param, dirs, thr) if kind == "knn"
                        else oracle.estimate_point_cloud_normals_ball(pts, param, dirs, thr, 8))
        assert np.array_equal(idx, ref_i) and np.array_equal(nrm, ref_n), thr
        sgn = np.sign(dirs[idx, 2].astype(np.float64))
        assert np.array_equal(nrm[:, 2], sgn.astype(dtype)) and not nrm[:, :2].any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_collinear_neighbourhoods(pcu, oracle, kind, dtype):
    """Case 6: points on axis-aligned and rotated lines: a unit normal perpendicular to the line (no particular one)."""
    t = np.arange(-200, 200, dtype=np.float64)[:, None] * 1e-2
    dirs = [np.array([1.0, 0, 0]), np.array([0, 1.0, 0]), np.array([0, 0, 1.0]), _rotation(70)[0], _rotation(71)[2]]
    for a, d in enumerate(dirs):
        pts = (t * d + np.array([0.5, -1.0, 2.0])).astype(dtype)
        param = 10 if kind == "knn" else 2.6e-3
        idx, nrm = estimate(pcu, kind, pts, param)
        assert np.array_equal(idx, np.arange(len(pts)))
        offs = offsets_of(oracle, kind, pts, param, idx)
        assert_rows_within_bound(nrm, offs, dtype, "line %d" % a)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [1, 2])
def test_fewer_than_three_neighbours(pcu, oracle, k, dtype):
    """Case 7: k = 1 and k = 2 give zero normals, as the oracle does; with view directions sign(0) = 0 and
    acos(0) = pi/2, so the points are kept exactly when drop_angle_threshold >= pi/2.  (The ball estimator's
    min_pts_per_ball is at least 3, so its fits always have three offsets or more.)"""
    pts = sphere(3000, 1e-2, 80).astype(dtype)
    dirs = sphere(3000, 0.0, 80).astype(dtype)
    idx, nrm = estimate(pcu, "knn", pts, k)
    ref_i, ref_n = oracle.estimate_point_cloud_normals_knn(pts, k)
    assert np.array_equal(idx, np.arange(3000)) and np.array_equal(idx, ref_i)
    assert not nrm.any() and np.array_equal(nrm, ref_n)
    for thr, kept in ((np.pi / 2, True), (np.pi, True), (np.nextafter(np.pi / 2, 0.0), False), (0.0, False)):
        idx, nrm = estimate(pcu, "knn", pts, k, dirs=dirs, thr=thr)
        ref_i, ref_n = oracle.estimate_point_cloud_normals_knn(pts, k, dirs, thr)
        assert np.array_equal(idx, ref_i) and np.array_equal(nrm, ref_n)
        assert len(idx) == (3000 if kept else 0) and not nrm.any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bad", ["nan", "inf", "-inf"])
def test_non_finite_points(pcu, oracle, kind, dtype, bad):
    """Case 8: a row with a NaN or an infinite coordinate is dropped and enters no other neighbourhood.  The k-NN
    estimator gives the finite rows the bits of a call on the cloud without those rows (its sums run in neighbour
    order).  The ball estimator gives the same kept rows and normals within the bound: its sums run in the grid's
    cell order, and the grid depends on the row count and on the bounding box, which an infinite coordinate
    stretches."""
    rng = np.random.default_rng(90)
    clean = sphere(3000, 1e-3, 91).astype(dtype)
    bad_rows = np.sort(rng.choice(3000 + 40, size=40, replace=False))
    pts = np.empty((3040, 3), dtype=dtype)
    mask = np.zeros(3040, dtype=bool)
    mask[bad_rows] = True
    pts[~mask] = clean
    pts[mask] = rng.normal(size=(40, 3))
    pts[bad_rows, rng.integers(0, 3, size=40)] = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf}[bad]
    finite_rows = np.nonzero(~mask)[0]
    param = 12 if kind == "knn" else 0.01
    idx, nrm = estimate(pcu, kind, pts, param)
    ref_i, ref_n = estimate(pcu, kind, clean, param)
    assert np.array_equal(idx, finite_rows[ref_i])
    if kind == "knn":
        assert np.array_equal(nrm, ref_n)
    else:
        rows = np.arange(0, len(ref_i), 7)
        offs = offsets_of(oracle, kind, clean, param, ref_i[rows])
        assert assert_rows_within_bound(nrm[rows], offs, dtype) > 0.9 * len(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_view_direction_boundaries(pcu, oracle, kind, dtype):
    """Case 9: on a plane z = const the normal is exactly (0, 0, +-1).  A view direction in the plane makes the dot
    product exactly 0: a zero normal, kept only when the threshold is >= pi/2.  Threshold 0 with the view along the
    normal keeps every point, oriented."""
    rng = np.random.default_rng(100)
    pts = np.concatenate([rng.random((3000, 2)), np.full((3000, 1), 0.25)], axis=1).astype(dtype)
    param = 12 if kind == "knn" else 1e-3
    for weight in (["constant"] if kind == "knn" else ["constant", "rbf"]):
        idx, nrm = estimate(pcu, kind, pts, param, weight=weight)
        assert np.array_equal(np.abs(nrm), np.tile(np.array([0, 0, 1], dtype=dtype), (len(idx), 1)))
        n_all = len(idx)
        side = np.tile(np.array([1, 0, 0], dtype=dtype), (3000, 1))
        for thr, keep in ((np.pi / 2, True), (np.pi, True), (np.nextafter(np.pi / 2, 0.0), False)):
            i2, n2 = estimate(pcu, kind, pts, param, dirs=side, thr=thr, weight=weight)
            assert len(i2) == (n_all if keep else 0) and not n2.any(), thr
        for z in (1, -1):
            view = np.tile(np.array([0, 0, z], dtype=dtype), (3000, 1))
            i2, n2 = estimate(pcu, kind, pts, param, dirs=view, thr=0.0, weight=weight)
            assert np.array_equal(i2, idx) and np.array_equal(n2, view[:len(i2)])
