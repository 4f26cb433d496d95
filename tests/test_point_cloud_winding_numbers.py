"""point_cloud_fast_winding_number: the exact field of DESIGN.md §3 (point clouds) restated with array operations and
checked against closed forms; on the GPU, exact mode within the derived rounding bound, public mode against the exact
sum, scale, determinism, agreement with the triangle-soup field, edge inputs, full size and input forms."""
import inspect
import math

import numpy as np
import pytest

from meshes import icosphere
from test_closest_points import assert_bits, queries
from test_winding_numbers import CLOSED

# Twice the largest |w(beta = 2) - w(exact)| over every query set below and the full-size rows: 0.0568 (nested shells
# of opposite orientation; 0.0341 at full size), measured on an H100 80GB HBM3, the same for fp32 and fp64 inputs.
# Larger than the soup's: a point's term grows as 1 / d^2 near it, a face's solid angle stays below 2 pi.
PUBLIC_TOL = 0.114
# Twice the largest |w(face cloud) - w(soup)| at the closed meshes' well-inside and well-outside queries: 0.0158 (torus),
# measured on the same card.
SOUP_TOL = 0.032

U = 2.0 ** -24


def _gamma(k):
    return k * U / (1 - k * U)


# ---- the restatement: fp64 dipoles of the fp32-rounded data ------------------------------------------------------------
def rounded(p, n, a):
    """(p, an) as the kernels see them: p rounded to fp32, an = fl32(fl_T(a n)) with T the input precision."""
    is_torch = type(p).__module__.startswith("torch")
    if is_torch:
        an = (a.reshape(-1, 1) * n).float().double()
        return p.float().double(), an
    an = (np.asarray(a).reshape(-1, 1) * n).astype(np.float32).astype(np.float64)
    return p.astype(np.float32).astype(np.float64), an


def exact_pw(q, p, n, a, chunk=256, bound=False):
    """w = sum over points of an.d / |d|^3 / 4 pi in fp64, d = p - q (numpy arrays, or torch CUDA tensors), and with
    bound=True the rounding bound of the fp32 evaluation (DESIGN.md §3)."""
    is_torch = type(q).__module__.startswith("torch")
    xp = None
    if is_torch:
        import torch
        xp, q = torch, q.float().double()
    else:
        xp, q = np, q.astype(np.float32).astype(np.float64)
    P, AN = rounded(p, n, a)
    ws, bs = [], []
    for s in range(0, q.shape[0], chunk):
        x = q[s:s + chunk]
        d = [P[None, :, k] - x[:, None, k] for k in range(3)]
        d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
        num = d[0] * AN[None, :, 0] + d[1] * AN[None, :, 1] + d[2] * AN[None, :, 2]
        zero = d2 == 0
        den = xp.where(zero, 1.0 + 0.0 * d2, d2 * xp.sqrt(d2))
        om = xp.where(zero, 0.0 * d2, num / den)
        ws.append(om.sum(1) / (4 * math.pi))
        if bound:
            S = abs(d[0] * AN[None, :, 0]) + abs(d[1] * AN[None, :, 1]) + abs(d[2] * AN[None, :, 2])
            e = xp.where(zero, 0.0 * d2, _gamma(17) * S / den)
            b = e.sum(1) / (4 * math.pi) + P.shape[0] * 2.0 ** -53 * abs(om).sum(1) / (4 * math.pi)
            bs.append(b.cpu().numpy() if is_torch else b)
    w = xp.cat(ws) if is_torch else np.concatenate(ws)
    if not bound:
        return w
    wn = w.cpu().numpy() if is_torch else w
    return w, np.concatenate(bs) + U * abs(wn)          # the final rounding to fp32


# ---- clouds -----------------------------------------------------------------------------------------------------------
def face_cloud(v, f, dtype=None):
    """One point per face: the centroid, the unit face normal and the face's area."""
    v64 = v.astype(np.float64)
    A, B, C = (v64[f[:, k]] for k in range(3))
    c = np.cross(B - A, C - A)
    area = 0.5 * np.linalg.norm(c, axis=1)
    dt = dtype or v.dtype
    nrm = c / np.maximum(2 * area, 1e-300)[:, None]
    return ((A + B + C) / 3).astype(dt), nrm.astype(dt), area.astype(dt)


def sphere_cloud(subdivisions=4, radius=1.0, inward=False, dtype=np.float64):
    """Quadrature of a sphere: the face centroids of an icosphere pushed onto it, radial normals, and areas that sum to
    4 pi r^2."""
    v, f = icosphere(subdivisions)
    p, _, a = face_cloud(v, f, np.float64)
    u = p / np.linalg.norm(p, axis=1, keepdims=True)
    a = a * (4 * math.pi / a.sum()) * radius ** 2
    return (radius * u).astype(dtype), (-u if inward else u).astype(dtype), a.astype(dtype)


def pwn_device(pcu, p, n, a, q, beta):
    """The winding number at far-field threshold beta through the binding (beta = inf: every point exact)."""
    import torch
    pt, nt, at, qt = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (p, n, a, q))
    w = torch.empty(len(q), dtype=qt.dtype, device="cuda")
    pcu._pcu_internal._point_cloud_fast_winding_number_device(qt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), at.data_ptr(),
                                                              len(p), qt.data_ptr(), len(q), beta, w.data_ptr(), 0,
                                                              torch.cuda.current_stream().cuda_stream)
    return w.cpu().numpy()


def cloud_sets(dtype, random=True):
    """(name, p, n, a, q): one point per face of the winding-number test meshes, a sphere quadrature and (random=True)
    random points with random normals and areas of both signs."""
    for name, make in CLOSED.items():
        (v, f), _ = make(dtype)
        p, n, a = face_cloud(v, f)
        yield name, p, n, a, queries(v, f, 700, 3)
    p, n, a = sphere_cloud(4, 1.0, False, dtype)
    v, f = icosphere(4, 0.0, 0, dtype)
    yield "sphere", p, n, a, queries(v, f, 700, 4)
    if not random:
        return
    rng = np.random.default_rng(5)
    p = rng.standard_normal((3000, 3)).astype(dtype)
    n = rng.standard_normal((3000, 3)).astype(dtype)
    a = (rng.random(3000) - 0.3).astype(dtype)                      # some negative areas
    yield "random", p, n, a, rng.standard_normal((2000, 3)).astype(dtype) * 2


# ---- CPU: interface, arguments, the restatement ------------------------------------------------------------------------
def test_signature(pcu):
    ps = list(inspect.signature(pcu.point_cloud_fast_winding_number).parameters.values())
    assert [p.name for p in ps] == ["p", "n", "a", "q", "device"]
    assert ps[4].kind == inspect.Parameter.KEYWORD_ONLY and ps[4].default is None
    assert "point_cloud_fast_winding_number" in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    wn = pcu.point_cloud_fast_winding_number
    p, n, a = sphere_cloud(1)
    q = np.zeros((4, 3))
    before = pcu.launch_count()
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'p'. Expected one of"):
        wn(p.astype(np.int32), n, a, q)
    for i, name in ((1, "n"), (2, "a"), (3, "q")):
        args = [p, n, a, q]
        args[i] = args[i].astype(np.float32)
        with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument '%s'. Expected it to match "
                                             r"argument 'p' which is of type float64." % name):
            wn(*args)
    # the binding's order: every dtype first, then p's shape, n's shape, the row counts, q, and last a's size
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'q'"):
        wn(p[:, :2], n, a, q.astype(np.float32))
    with pytest.raises(ValueError, match=r"Only 3D inputs are supported: v must have shape \(n, 3\) \(n > 0\). Got "
                                         r"points.shape =\(%d, 2\)." % len(p)):
        wn(p[:, :2], n[:, :2], a, q[:0])
    with pytest.raises(ValueError, match=r"Invalid shape for normals: must have shape \(n, 3\) \(n > 0\). Got "
                                         r"normals.shape =\(%d, 2\)." % len(p)):
        wn(p, n[:, :2], a, q[:0])
    with pytest.raises(ValueError, match=r"Invalid input point cloud. Number of normals must match number of points. Got "
                                         r"points.shape =\(%d, 3\) and normals.shape = 5, 3$" % len(p)):
        wn(p, n[:5], a, q[:0])
    with pytest.raises(ValueError, match=r"Invalid input point cloud with zero points: points must have shape \(n, 3\) "
                                         r"\(n > 0\). Got points.shape =\(0, 3\)."):
        wn(p, n, a[:3], q[:0])
    with pytest.raises(ValueError, match="Only 3D inputs are supported: v must have shape"):
        wn(p, n, a, q[:, :2])
    for bad in (a[:-1], a[:, None][:-1], np.concatenate([a, a]), np.stack([a, a], 1)):
        with pytest.raises(ValueError, match=r"Invalid shape for areas: a must have #p = %d elements" % len(p)):
            wn(p, n, bad, q)
    with pytest.raises(ValueError, match="NumPy array"):
        wn(p.tolist(), n, a, q)
    assert pcu.launch_count() == before


def test_single_dipole():
    p = np.zeros((1, 3), np.float32)
    n = np.array([[0, 0, 1]], np.float32)
    a = np.array([1.0], np.float32)
    q = np.array([[0, 0, -2], [0, 0, 2], [1, 0, 0], [0, 0, 0], [0, -3, -4]], np.float32)
    w = exact_pw(q, p, n, a) * 4 * math.pi
    assert w[0] == pytest.approx(0.25, abs=1e-15) and w[1] == pytest.approx(-0.25, abs=1e-15)
    assert w[2] == 0 and w[3] == 0                       # in the dipole's plane, and on the point
    assert w[4] == pytest.approx(4 / 125, abs=1e-15)


@pytest.mark.parametrize("inward", [False, True])
def test_sphere_quadrature(inward):
    p, n, a = sphere_cloud(4, 1.0, inward)
    q = np.array([[0, 0, 0], [0.3, -0.2, 0.4], [0, 0.5, 0], [1.6, 0, 0], [0, 2, 2], [10, -3, 1]])
    w = exact_pw(q, p, n, a)
    expect = np.array([1, 1, 1, 0, 0, 0]) * (-1 if inward else 1)
    assert np.abs(w - expect).max() < 2e-3, w


def test_nested_spheres():
    outer, inner = sphere_cloud(4, 1.0), sphere_cloud(4, 0.5)
    p, n, a = (np.concatenate([x, y]) for x, y in zip(outer, inner))
    w = exact_pw(np.array([[0, 0, 0], [0.1, 0, 0.2], [0, 0.75, 0], [0, 0, 1.8]]), p, n, a)
    assert np.abs(w - [2, 2, 1, 0]).max() < 5e-3, w


def test_exact_mode_bound_is_small():
    """Away from the points the derived bound is a few fp32 ulps of the terms: below 1e-5 for queries at least 0.1 from
    the unit sphere sampled with 5120 points."""
    p, n, a = sphere_cloud(4)
    rng = np.random.default_rng(1)
    q = rng.standard_normal((400, 3))
    r = np.linalg.norm(q, axis=1)
    q = q[np.abs(r - 1) >= 0.1]
    _, b = exact_pw(q, p, n, a, bound=True)
    assert b.max() <= 1e-5, b.max()


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_exact_mode_within_the_bound(pcu, dtype):
    for name, p, n, a, q in cloud_sets(dtype):
        ref, b = exact_pw(q, p, n, a, bound=True)
        w = pwn_device(pcu, p, n, a, q, float("inf"))
        assert w.dtype == dtype
        err = np.abs(w.astype(np.float64) - ref)
        assert (err <= b).all(), "%s: %d rows outside the bound, worst %.3g (bound %.3g)" % (
            name, int((err > b).sum()), err.max(), b[np.argmax(err - b)])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_public_mode_against_the_exact_sum(pcu, dtype):
    worst = 0.0
    for name, p, n, a, q in cloud_sets(dtype, random=False):
        ref = exact_pw(q, p, n, a)
        w = pcu.point_cloud_fast_winding_number(p, n, a, q)
        assert w.dtype == dtype and w.shape == (len(q),)
        err = np.abs(w.astype(np.float64) - ref).max()
        worst = max(worst, err)
        assert err <= PUBLIC_TOL, (name, err)
    print("max |w(beta = 2) - w(exact)| %s: %.3g" % (np.dtype(dtype).name, worst))


@pytest.mark.gpu
def test_far_field_error_falls_with_beta(pcu):
    """Against exact mode (the same leaf terms, the same bits), each doubling of beta must divide the largest error by
    at least 8 (the expansion is of order 2).  Measured on an H100 80GB HBM3: 0.0466, 1.27e-3, 6.62e-5 (torus),
    0.049, 1.39e-3, 6.18e-5 (icosphere) and 0.0604, 1.49e-3, 7.12e-5 (nested) at beta = 2, 4, 8, at least 19x per step."""
    for name in ("torus", "icosphere", "nested"):
        (v, f), _ = CLOSED[name](np.float32)
        p, n, a = face_cloud(v, f)
        q = queries(v, f, 1000, 6)
        exact = pwn_device(pcu, p, n, a, q, float("inf")).astype(np.float64)
        errs = [np.abs(pwn_device(pcu, p, n, a, q, beta).astype(np.float64) - exact).max() for beta in (2.0, 4.0, 8.0)]
        print("%s: max |w(beta) - w(exact)| at beta 2, 4, 8: %.3g %.3g %.3g" % (name, *errs))
        assert errs[0] <= PUBLIC_TOL and errs[1] <= errs[0] / 8 and errs[2] <= errs[1] / 8, (name, errs)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("scale", [2.0 ** 20, 2.0 ** -14])
def test_scale_does_not_change_a_bit(pcu, dtype, scale):
    s = dtype(scale)
    for name, p, n, a, q in cloud_sets(dtype):
        w = pcu.point_cloud_fast_winding_number(p, n, a, q)
        ws = pcu.point_cloud_fast_winding_number(p * s, n, a * s * s, q * s)
        assert_bits(ws, w, "%s scaled by %g" % (name, scale))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_determinism(pcu, dtype):
    (v, f), _ = CLOSED["torus"](dtype)
    p, n, a = face_cloud(v, f)
    q = queries(v, f, 3000, 11)
    w = pcu.point_cloud_fast_winding_number(p, n, a, q)
    assert_bits(pcu.point_cloud_fast_winding_number(p, n, a, q), w, "second call")
    rng = np.random.default_rng(2)
    perm = rng.permutation(len(q))
    assert_bits(pcu.point_cloud_fast_winding_number(p, n, a, q[perm]), w[perm], "permuted queries")
    sub = np.sort(rng.choice(len(q), 100, replace=False))
    assert_bits(pcu.point_cloud_fast_winding_number(p, n, a, q[sub]), w[sub], "a subset of the queries")
    assert_bits(pcu.point_cloud_fast_winding_number(p, n, a, q[7:8]), w[7:8], "one query")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_one_point_per_face_agrees_with_the_soup(pcu, dtype):
    """Away from the surface, a closed mesh's face cloud gives about the soup's winding number; both round to the same
    integer."""
    worst = 0.0
    for name, make in CLOSED.items():
        (v, f), cases = make(dtype)
        p, n, a = face_cloud(v, f)
        q = np.array([c[0] for c in cases], dtype=dtype)
        w = pcu.point_cloud_fast_winding_number(p, n, a, q).astype(np.float64)
        ws = pcu.triangle_soup_fast_winding_number(v, f, q).astype(np.float64)
        worst = max(worst, np.abs(w - ws).max())
        assert np.abs(w - ws).max() <= SOUP_TOL, (name, w, ws)
        assert np.array_equal(np.rint(w), np.rint(ws)) and np.array_equal(np.rint(w), [c[1] for c in cases]), name
    print("max |w(face cloud) - w(soup)| %s: %.3g" % (np.dtype(dtype).name, worst))


@pytest.mark.gpu
def test_dense_samples_classify_like_the_soup(pcu):
    for name in ("icosphere", "torus", "nested", "reversed"):
        (v, f), _ = CLOSED[name](np.float64)
        fi, bc = pcu.sample_mesh_random(v, f, 200000, random_seed=3)
        fi = fi.astype(np.int64)
        x = (v[f[fi]] * bc[:, :, None]).sum(1)
        _, nrm, area = face_cloud(v, f)
        a = np.full(len(x), area.sum() / len(x))
        q = queries(v, f, 2000, 12)[:4000]
        d, _, _ = pcu.closest_points_on_mesh(q, v, f)
        away = d >= 0.05 * float((v.max(0) - v.min(0)).max())
        w = pcu.point_cloud_fast_winding_number(x, nrm[fi], a, q[away])
        ws = pcu.triangle_soup_fast_winding_number(v, f, q[away])
        assert away.sum() > 1000 and np.array_equal(np.rint(w), np.rint(ws)), (name, int((np.rint(w) != np.rint(ws)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_edge_inputs(pcu, dtype):
    wn = pcu.point_cloud_fast_winding_number
    rng = np.random.default_rng(9)
    q = rng.standard_normal((300, 3)).astype(dtype)
    # a single point
    p, n, a = np.array([[0.1, 0.2, 0.3]], dtype), np.array([[0, 1, 2]], dtype), np.array([0.5], dtype)
    assert np.abs(wn(p, n, a, q) - exact_pw(q, p, n, a)).max() <= 1e-6
    assert wn(p, n, a, p)[0] == 0
    # every point the same (equal Morton codes, every node of radius 0): a query on the point gets no term
    k = 1000
    p, n, a = np.tile(p, (k, 1)), rng.standard_normal((k, 3)).astype(dtype), rng.random(k).astype(dtype)
    w = wn(p, n, a, np.concatenate([q, p[:1]]))
    assert w[-1] == 0
    ref, b = exact_pw(q, p, n, a, bound=True)
    assert (np.abs(w[:-1].astype(np.float64) - ref) <= b).all()
    # duplicates, zero areas, zero normals and negative areas
    sp, sn, sa = sphere_cloud(3, 1.0, False, dtype)
    dp, dn, da = np.concatenate([sp, sp[:200]]), np.concatenate([sn, sn[:200]]), np.concatenate([sa, sa[:200]])
    da[:50] = 0
    dn[50:100] = 0
    da[100:150] *= -1
    ref, b = exact_pw(q, dp, dn, da, bound=True)
    assert (np.abs(pwn_device(pcu, dp, dn, da, q, float("inf")).astype(np.float64) - ref) <= b).all()
    assert np.isfinite(wn(dp, dn, da, q)).all()
    zero = wn(dp, dn, np.zeros_like(da), q)
    assert np.array_equal(zero, np.zeros_like(zero))
    # no points: w = 0
    w = wn(sp[:0], sn[:0], sa[:0], q)
    assert w.dtype == dtype and w.shape == (len(q),) and not w.any()
    # a as (#p,) and (#p, 1), and non-contiguous inputs
    w = wn(sp, sn, sa, q)
    assert_bits(wn(sp, sn, sa[:, None], q), w, "(#p, 1) areas")
    big = [np.asfortranarray(x) for x in (sp, sn, q)]
    assert_bits(wn(big[0], big[1], np.repeat(sa, 2)[::2], big[2]), w, "non-contiguous inputs")
    strided = [x[::2] for x in (dp, dn, da)]
    assert_bits(wn(*strided, q[::3]), wn(*[x.copy() for x in strided], q[::3].copy()), "strided rows")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_full_size(pcu, dtype):
    import torch
    v, f = icosphere(8, 1e-4, 5, np.float64)                 # 1 310 720 faces
    rng = np.random.default_rng(8)
    m = 10 ** 6
    fi = rng.integers(0, len(f), m)
    _, nrm, area = face_cloud(v, f)
    bc = rng.random((m, 2))
    s = np.sqrt(bc[:, :1])
    bc = np.concatenate([1 - s, s * (1 - bc[:, 1:]), s * bc[:, 1:]], 1)
    x = (v[f[fi]] * bc[:, :, None]).sum(1)
    pt = torch.from_numpy(x.astype(dtype)).cuda()
    nt = torch.from_numpy(nrm[fi].astype(dtype)).cuda()
    at = torch.full((m, 1), area.sum() / m, dtype=pt.dtype, device="cuda")
    q = queries(v, f, 2000, 6)[:4000]
    qt = torch.from_numpy(q.astype(dtype)).cuda()
    w = pcu.point_cloud_fast_winding_number(pt, nt, at, qt)
    assert w.is_cuda and w.dtype == pt.dtype and w.shape == (len(q),)
    ref = exact_pw(qt, pt, nt, at, chunk=16)
    err = float((w.double() - ref).abs().max())
    print("full size max |w(beta = 2) - w(exact)| %s: %.3g" % (np.dtype(dtype).name, err))
    assert err <= PUBLIC_TOL


@pytest.mark.gpu
def test_input_forms_and_device(pcu):
    import torch
    p, n, a = sphere_cloud(3, 1.0, False, np.float32)
    q = np.random.default_rng(1).standard_normal((500, 3)).astype(np.float32)
    w = pcu.point_cloud_fast_winding_number(p, n, a, q)
    assert isinstance(w, np.ndarray) and w.dtype == np.float32
    cuda = [torch.from_numpy(x).cuda() for x in (p, n, a, q)]
    wt = pcu.point_cloud_fast_winding_number(*cuda)
    assert wt.is_cuda
    cpu = [torch.from_numpy(x) for x in (p, n, a, q)]
    wc = pcu.point_cloud_fast_winding_number(*cpu)
    assert isinstance(wc, torch.Tensor) and not wc.is_cuda
    wd = pcu.point_cloud_fast_winding_number(p, n, a, q, device="cuda:0")
    wdt = pcu.point_cloud_fast_winding_number(*cuda, device="cuda:0")
    for x in (wt.cpu().numpy(), wc.numpy(), wd, wdt.cpu().numpy()):
        assert_bits(x, w, "forms")
    with pytest.raises(ValueError, match="contradicts" if torch.cuda.device_count() > 1 else "out of range"):
        pcu.point_cloud_fast_winding_number(*cuda, device="cuda:1")
    empty = pcu.point_cloud_fast_winding_number(*[x[:0] for x in cuda[:3]], cuda[3])
    assert empty.is_cuda and not empty.any()
