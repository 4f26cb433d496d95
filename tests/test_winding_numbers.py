"""triangle_soup_fast_winding_number and signed_distance_to_mesh: the exact winding number of DESIGN.md §3 restated with
array operations and checked against closed forms; on the GPU, exact mode within the derived rounding bound, public
mode against the exact sum, determinism, the signed distance bit for bit from the two public functions, the band, full
size, input forms and errors."""
import inspect
import math

import numpy as np
import pytest

from meshes import icosphere, torus
from test_closest_points import FDTYPES, assert_bits, queries
from test_mesh_sampling import MESHES

# Twice the largest |w(beta = 2) - w(exact)| over every query set below and the full-size rows: 0.00976, measured on
# an H100 80GB HBM3, the same for fp32 and fp64 inputs.
PUBLIC_TOL = 0.0195

U = 2.0 ** -24


def _gamma(k):
    return k * U / (1 - k * U)


# ---- the restatement: fp64 solid angles of the fp32-rounded corners seen from the fp32-rounded queries --------------
def exact_w(q, v, f, chunk=64, bound=False):
    """w = sum over faces of Omega / 4 pi in fp64 (numpy arrays, or torch CUDA tensors with f as int64), and with
    bound=True the rounding bound of the fp32 evaluation (DESIGN.md §3)."""
    is_torch = type(q).__module__.startswith("torch")
    if is_torch:
        import torch
        xp, q = torch, q.float().double()
        v, fi = v.float().double(), f.long()
    else:
        xp, q = np, q.astype(np.float32).astype(np.float64)
        v, fi = v.astype(np.float32).astype(np.float64), f.astype(np.int64)
    A, B, C = (v[fi[:, k]] for k in range(3))
    e1, e2 = B - A, C - A
    n = [e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
         e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]]
    nabs = [abs(e1[:, 1] * e2[:, 2]) + abs(e1[:, 2] * e2[:, 1]), abs(e1[:, 2] * e2[:, 0]) + abs(e1[:, 0] * e2[:, 2]),
            abs(e1[:, 0] * e2[:, 1]) + abs(e1[:, 1] * e2[:, 0])]
    ws, bs = [], []
    for s in range(0, q.shape[0], chunk):
        p = q[s:s + chunk]
        a, b, c = ([X[None, :, k] - p[:, None, k] for k in range(3)] for X in (A, B, C))
        la, lb, lc = (xp.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]) for x in (a, b, c))
        det = a[0] * n[0][None] + a[1] * n[1][None] + a[2] * n[2][None]
        ab, ac, bc = ((x[0] * y[0] + x[1] * y[1] + x[2] * y[2]) for x, y in ((a, b), (a, c), (b, c)))
        D = la * lb * lc + ab * lc + ac * lb + bc * la
        zero = (la == 0) | (lb == 0) | (lc == 0) | (det == 0)
        theta = xp.where(zero, 0.0 * det, xp.arctan2(det, D) if not is_torch else torch.atan2(det, D))
        ws.append((2 * theta).sum(1) / (4 * math.pi))
        if bound:
            dabs = abs(a[0]) * nabs[0][None] + abs(a[1]) * nabs[1][None] + abs(a[2]) * nabs[2][None]
            sabs = (la * lb * lc + (abs(a[0] * b[0]) + abs(a[1] * b[1]) + abs(a[2] * b[2])) * lc
                    + (abs(a[0] * c[0]) + abs(a[1] * c[1]) + abs(a[2] * c[2])) * lb
                    + (abs(b[0] * c[0]) + abs(b[1] * c[1]) + abs(b[2] * c[2])) * la)
            rho2 = det * det + D * D
            with np.errstate(divide="ignore", invalid="ignore"):
                e = 2 * (2 * (_gamma(8) * dabs * abs(D) + _gamma(17) * sabs * abs(det)) / rho2 + 3 * 2.0 ** -23 * abs(theta))
            e = np.where(zero & (rho2 == 0), 0.0, e)
            bs.append(e.sum(1) / (4 * math.pi) + len(fi) * 2.0 ** -53 * (2 * abs(theta)).sum(1) / (4 * math.pi))
    cat = xp.cat if is_torch else np.concatenate
    w = cat(ws)
    if not bound:
        return w
    b = np.concatenate(bs)
    return w, b + U * abs(w)          # the final rounding to fp32


# ---- meshes ---------------------------------------------------------------------------------------------------------
def nested(opposite, dtype=np.float64):
    v, f = icosphere(3, 0.0, 0, dtype)
    inner = f[:, ::-1] if opposite else f
    return np.concatenate([v, 0.5 * v]).astype(dtype), np.concatenate([f, inner + len(v)])


def reversed_sphere(dtype=np.float64):
    v, f = icosphere(3, 0.01, 1, dtype)
    return v, np.ascontiguousarray(f[:, ::-1])


def doubled(dtype=np.float64):
    v, f = icosphere(3, 0.01, 1, dtype)
    return v, np.concatenate([f, f])


ALL_MESHES = dict(MESHES)
ALL_MESHES.update({
    "torus": lambda dt: torus(40, 20, 0.4, dt),
    "nested": lambda dt: nested(False, dt),
    "nested-opposite": lambda dt: nested(True, dt),
    "reversed": reversed_sphere,
    "doubled": doubled,
})

# For the closed meshes: (query, winding number) pairs well away from the surface.
CLOSED = {
    "icosphere": lambda dt: (icosphere(3, 0.01, 1, dt), [((0, 0, 0), 1), ((0.3, -0.2, 0.5), 1), ((1.5, 0, 0), 0), ((0, 3, 1), 0)]),
    "torus": lambda dt: (torus(40, 20, 0.4, dt), [((1, 0, 0), 1), ((0, -1.1, 0.1), 1), ((0, 0, 0), 0), ((0, 0, 1), 0), ((2, 2, 0), 0)]),
    "nested": lambda dt: (nested(False, dt), [((0, 0, 0), 2), ((0, 0.75, 0), 1), ((0, 0, 2), 0)]),
    "nested-opposite": lambda dt: (nested(True, dt), [((0, 0, 0), 0), ((0, 0.75, 0), 1), ((0, 0, 2), 0)]),
    "reversed": lambda dt: (reversed_sphere(dt), [((0, 0, 0), -1), ((0.2, 0.1, 0), -1), ((0, 0, 1.5), 0)]),
}


def wn_device(pcu, v, f, p, beta):
    """The winding number at far-field threshold beta through the binding (beta = inf: every face exact)."""
    import torch
    kinds = {"int32": 0, "int64": 1, "uint32": 2, "uint64": 3}
    signed = {"uint32": np.int32, "uint64": np.int64}
    vt, pt = torch.from_numpy(np.ascontiguousarray(v)).cuda(), torch.from_numpy(np.ascontiguousarray(p)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f).view(signed.get(f.dtype.name, f.dtype))).cuda()
    w = torch.empty(len(p), dtype=pt.dtype, device="cuda")
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    pcu._pcu_internal._fast_winding_number_device(pt.dtype == torch.float64, vt.data_ptr(), len(v), ft.data_ptr(), len(f),
                                                  kinds[f.dtype.name], pt.data_ptr(), len(p), beta, w.data_ptr(), bad.data_ptr(), 0,
                                                  torch.cuda.current_stream().cuda_stream)
    assert int(bad.item()) == 0
    return w.cpu().numpy()


# ---- CPU: interface, the restatement ----------------------------------------------------------------------------------
def test_signatures(pcu):
    ps = list(inspect.signature(pcu.triangle_soup_fast_winding_number).parameters.values())
    assert [p.name for p in ps] == ["v", "f", "p", "device"]
    assert ps[3].kind == inspect.Parameter.KEYWORD_ONLY and ps[3].default is None
    ps = list(inspect.signature(pcu.signed_distance_to_mesh).parameters.values())
    assert [p.name for p in ps] == ["p", "v", "f", "lower_bound", "upper_bound", "device"]
    assert ps[3].default == -np.inf and ps[4].default == np.inf
    assert ps[5].kind == inspect.Parameter.KEYWORD_ONLY and ps[5].default is None
    assert "triangle_soup_fast_winding_number" in pcu.__all__ and "signed_distance_to_mesh" in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    wn, sd = pcu.triangle_soup_fast_winding_number, pcu.signed_distance_to_mesh
    v, f = icosphere(1)
    p = np.zeros((4, 3))
    before = pcu.launch_count()
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'v'"):
        wn(v.astype(np.int32), f, p)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'f'"):
        wn(v, f.astype(np.float64), p)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'p'. Expected it to match argument "
                                         r"'v' which is of type float64."):
        wn(v, f, p.astype(np.float32))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int64\) for argument 'p'"):
        sd(p.astype(np.int64), v, f)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'v'. Expected it to match argument "
                                         r"'p' which is of type float64."):
        sd(p, v.astype(np.float32), f)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'f'"):
        sd(p, v, f.astype(np.float32))
    for call in (lambda q, vv, ff: wn(vv, ff, q), sd):
        with pytest.raises(ValueError, match=r"Invalid input point cloud with zero points: points must have shape \(n, 3\) "
                                             r"\(n > 0\). Got points.shape =\(0, 3\)."):
            call(p[:0], v, f)
        with pytest.raises(ValueError, match="Only 3D inputs are supported: v must have shape"):
            call(p[:, :2], v, f)
        with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
            call(p, v, f[:0])
        with pytest.raises(ValueError, match="Only 3D inputs are supported: v and f must have shape"):
            call(p, v[:, :2], f)
        with pytest.raises(ValueError, match="NumPy array"):
            call(p.tolist(), v, f)
    assert pcu.launch_count() == before


def test_closed_forms():
    # the octant's triangle seen from the origin, on its axis: 4 pi / 8
    v = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32)
    f = np.array([[0, 1, 2]])
    q = np.array([[0, 0, 0], [1, 1, 1], [-2, -2, -2]], dtype=np.float32)
    w = exact_w(q, v, f)
    assert w[0] == pytest.approx(1 / 8, abs=1e-15)
    assert w[1] < 0 and w[2] > 0                 # seen from the other side, and from behind the origin
    # a cube of 12 outward triangles: 1 at its centre (each face 1/6), 0 outside
    c = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for a, b, cc, d in quads for t in ((a, b, cc), (a, cc, d))])
    w = exact_w(np.array([[0.5, 0.5, 0.5], [0.1, 0.8, 0.3], [2, 0.5, 0.5], [-1, -1, 3]], dtype=np.float32), c, f)
    assert abs(w[0] - 1) < 1e-14 and abs(w[1] - 1) < 1e-14 and abs(w[2]) < 1e-14 and abs(w[3]) < 1e-14
    w1 = exact_w(np.array([[0.5, 0.5, 0.5]], dtype=np.float32), c, f[:2])
    assert w1[0] == pytest.approx(1 / 6, abs=1e-15)


@pytest.mark.parametrize("name", sorted(CLOSED))
def test_closed_meshes_give_integers(name):
    (v, f), cases = CLOSED[name](np.float64)
    q = np.array([c[0] for c in cases], dtype=np.float64)
    w = exact_w(q, v, f)
    assert np.abs(w - np.array([c[1] for c in cases])).max() < 1e-9, (name, w)


def test_exact_mode_bound_is_small():
    """The bound DESIGN.md derives for exact mode stays below 1e-4 on meshes of up to 2e4 faces for queries at least
    5e-3 of the mesh's extent from the surface (it grows as 1 / distance near an edge, where w itself jumps)."""
    from test_closest_points import restate
    v, f = icosphere(5, 0.01, 3)                           # 20 480 faces
    _, b = exact_w(queries(v, f, 100, 4), v, f, bound=True)
    assert b.max() <= 1e-4, b.max()
    for name, make in ALL_MESHES.items():
        v, f = make(np.float64)
        q = queries(v, f, 300, 5)
        _, b = exact_w(q, v, f, bound=True)
        scale = float((v.max(0) - v.min(0)).max())
        away = restate(q, v, f)[0] >= 5e-3 * scale
        assert away.mean() > 0.5 and b[away].max() <= 1e-4, (name, b[away].max())


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _sets(vdtype):
    for name, make in ALL_MESHES.items():
        v, f = make(vdtype)
        yield name, v, f, queries(v, f, 1000, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_exact_mode_within_the_bound(pcu, vdtype):
    for name, v, f, p in _sets(vdtype):
        ref, b = exact_w(p, v, f, bound=True)
        for fdt in FDTYPES:
            w = wn_device(pcu, v, f.astype(fdt), p, float("inf"))
            assert w.dtype == vdtype
            err = np.abs(w.astype(np.float64) - ref)
            assert (err <= b).all(), "%s %s: %d rows outside the bound, worst %.3g (bound %.3g)" % (
                name, fdt.__name__, int((err > b).sum()), err.max(), b[np.argmax(err - b)])


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_public_mode_against_the_exact_sum(pcu, vdtype):
    worst = 0.0
    for name, v, f, p in _sets(vdtype):
        ref = exact_w(p, v, f)
        w = pcu.triangle_soup_fast_winding_number(v, f, p).astype(np.float64)
        err = np.abs(w - ref).max()
        worst = max(worst, err)
        assert err <= PUBLIC_TOL, (name, err)
        clear = np.abs(np.abs(ref) - 0.5) >= 0.1
        assert np.array_equal(np.abs(w[clear]) > 0.5, np.abs(ref[clear]) > 0.5), name
    print("max |w(beta = 2) - w(exact)| %s: %.3g" % (np.dtype(vdtype).name, worst))
    for name, make in CLOSED.items():
        (v, f), cases = make(vdtype)
        q = np.array([c[0] for c in cases], dtype=vdtype)
        w = pcu.triangle_soup_fast_winding_number(v, f, q)
        assert np.abs(w - np.array([c[1] for c in cases])).max() <= PUBLIC_TOL, (name, w)
    # a face list concatenated with itself doubles w
    v, f = icosphere(3, 0.01, 1, vdtype)
    p = queries(v, f, 1000, 9)
    one = pcu.triangle_soup_fast_winding_number(v, f, p).astype(np.float64)
    two = pcu.triangle_soup_fast_winding_number(v, np.concatenate([f, f]), p).astype(np.float64)
    assert np.abs(two - 2 * one).max() <= 2 * PUBLIC_TOL


@pytest.mark.gpu
def test_far_field_error_falls_with_beta(pcu):
    """The expansion is of order 2, so its truncation error falls about as beta^-3: against exact mode (which evaluates
    the same leaves with the same bits), each doubling of beta must divide the largest error by at least 4."""
    for name in ("torus", "icosphere", "nested"):
        v, f = ALL_MESHES[name](np.float32)
        p = queries(v, f, 1000, 6)
        exact = wn_device(pcu, v, f, p, float("inf")).astype(np.float64)
        errs = [np.abs(wn_device(pcu, v, f, p, beta).astype(np.float64) - exact).max() for beta in (2.0, 4.0, 8.0)]
        print("%s: max |w(beta) - w(exact)| at beta 2, 4, 8: %.3g %.3g %.3g" % (name, *errs))
        assert errs[0] <= PUBLIC_TOL and errs[1] <= errs[0] / 4 and errs[2] <= errs[1] / 4, (name, errs)


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
@pytest.mark.parametrize("scale", [2.0 ** 20, 2.0 ** -14])
def test_scale_does_not_matter(pcu, vdtype, scale):
    """A mesh and its queries scaled by a power of two (exact in every precision) of about 1e6 or 1e-4 give the unit-scale
    winding numbers, and finite signed distances."""
    for name in ("torus", "doubled", "nested-opposite"):
        v, f = ALL_MESHES[name](vdtype)
        p = queries(v, f, 1000, 8)
        w = pcu.triangle_soup_fast_winding_number(v, f, p).astype(np.float64)
        ws = pcu.triangle_soup_fast_winding_number(v * vdtype(scale), f, p * vdtype(scale)).astype(np.float64)
        assert np.isfinite(ws).all(), name
        assert np.abs(ws - w).max() <= PUBLIC_TOL, (name, np.abs(ws - w).max())
        s, fi, _ = pcu.signed_distance_to_mesh(p * vdtype(scale), v * vdtype(scale), f)
        s1, fi1, _ = pcu.signed_distance_to_mesh(p, v, f)
        assert np.isfinite(s).all() and np.array_equal(fi, fi1), name
        assert np.array_equal(np.sign(s), np.sign(s1)), name


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_determinism(pcu, vdtype):
    v, f = torus(40, 20, 0.4, vdtype)
    p = queries(v, f, 3000, 11)
    w = pcu.triangle_soup_fast_winding_number(v, f, p)
    assert_bits(pcu.triangle_soup_fast_winding_number(v, f, p), w, "second call")
    perm = np.random.default_rng(2).permutation(len(p))
    assert_bits(pcu.triangle_soup_fast_winding_number(v, f, p[perm]), w[perm], "permuted queries")
    for fdt in FDTYPES:
        assert_bits(pcu.triangle_soup_fast_winding_number(v, f.astype(fdt), p), w, fdt.__name__)


def sd_from_public(pcu, p, v, f):
    """(s, fi, bc) from closest_points_on_mesh and triangle_soup_fast_winding_number: s = fl(fl(1 - 2|w|) d)."""
    d, fi, bc = pcu.closest_points_on_mesh(p, v, f)
    w = pcu.triangle_soup_fast_winding_number(v, f, p)
    sigma = (1.0 - 2.0 * np.abs(w.astype(np.float64))).astype(p.dtype)
    return sigma * d, fi.astype(np.int32), bc


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_signed_distance_bit_for_bit(pcu, vdtype):
    for name, v, f, p in _sets(vdtype):
        ref = sd_from_public(pcu, p, v, f)
        for fdt in FDTYPES:
            s, fi, bc = pcu.signed_distance_to_mesh(p, v, f.astype(fdt))
            assert fi.dtype == np.int32 and s.dtype == vdtype and bc.dtype == vdtype
            assert_bits(s, ref[0], "%s s %s" % (name, fdt.__name__))
            assert np.array_equal(fi, ref[1]), name
            assert_bits(bc, ref[2], "%s bc %s" % (name, fdt.__name__))
    v, f = icosphere(3, 0.0, 0, vdtype)
    s, _, _ = pcu.signed_distance_to_mesh(np.array([[0, 0, 0], [0, 0, 3]], dtype=vdtype), v, f)
    assert s[0] < 0 and s[1] > 0


def band(lower, upper, dt):
    lo, hi = dt(np.float32(lower)), dt(np.float32(upper))
    big = lambda a, b: b if a < b else a          # noqa: E731
    with np.errstate(invalid="ignore", over="ignore"):
        max_abs = big(-lo, hi)
        return max_abs * max_abs, big(max_abs - (hi - lo), dt(0)) ** 2


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_band(pcu, vdtype):
    dt = np.dtype(vdtype).type
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=vdtype)
    f = np.array([[0, 1, 2]], dtype=np.int32)
    q = np.array([[0, 0, 0.5]], dtype=vdtype)                        # d^2 = 0.25 exactly, at the corner (0, 0, 0)
    s, fi, bc = pcu.signed_distance_to_mesh(q, v, f, -0.5, 0.5)       # up = 0.25: out of the band
    assert np.isnan(s[0]) and fi[0] == len(f) + 1 and np.isnan(bc).all()
    s, fi, bc = pcu.signed_distance_to_mesh(q, v, f, -0.5, float(np.nextafter(np.float32(0.5), np.float32(1))))
    assert_bits(s, sd_from_public(pcu, q, v, f)[0], "nudged bound")          # back in the band: sigma * 0.5
    assert fi[0] == 0 and np.array_equal(bc, [[1, 0, 0]])
    q = np.array([[0.2, 0.2, 0.1], [0.2, 0.2, 0.5], [0.2, 0.2, -2.0]], dtype=vdtype)
    s, fi, bc = pcu.signed_distance_to_mesh(q, v, f, 0.2, 1.0)        # low = (1 - 0.8)^2, up = 1
    assert np.isnan(s[0]) and fi[0] == 2 and not np.isnan(s[1]) and fi[1] == 0 and np.isnan(s[2]) and fi[2] == 2
    # the band of random bounds against its restatement; outside it, NaN; inside, the unbanded result
    v, f = icosphere(3, 0.01, 1, vdtype)
    p = queries(v, f, 1000, 13)
    full = pcu.signed_distance_to_mesh(p, v, f)
    assert not np.isnan(full[0]).any()                               # the defaults give no band
    d, _, _ = pcu.closest_points_on_mesh(p, v, f)
    sq = d.astype(np.float64) ** 2                  # d^2 up to rounding: rows near a band edge are left out below
    for lower, upper in ((-0.3, 0.3), (0.05, 0.5), (-2.0, 0.1), (-np.inf, 0.2), (0.1, np.inf), (0.3, 0.2)):   # (0.3, 0.2): all out
        up, low = band(lower, upper, dt)
        got = pcu.signed_distance_to_mesh(p, v, f, lower, upper)
        out = np.isnan(got[0])
        edge = (np.abs(sq - float(up)) < 1e-5) | (np.abs(sq - float(low)) < 1e-5)
        with np.errstate(invalid="ignore"):
            expect = (sq >= float(up)) | (sq < float(low))
        assert np.array_equal(out[~edge], expect[~edge]), (lower, upper)
        assert (got[1][out] == len(f) + 1).all() and np.isnan(got[2][out]).all()
        if (~out).any():
            assert_bits(got[0][~out], full[0][~out], "in band")
            assert np.array_equal(got[1][~out], full[1][~out])


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_full_size(pcu, vdtype):
    import torch
    v, f = icosphere(8, 1e-4, 5, vdtype)                 # 1 310 720 faces
    f = f.astype(np.int32)
    rng = np.random.default_rng(8)
    n = 10 ** 6
    fi = rng.integers(0, len(f), n)
    r = rng.random((n, 2))
    s = np.sqrt(r[:, :1])
    bc = np.concatenate([1 - s, s * (1 - r[:, 1:]), s * r[:, 1:]], 1)
    p = ((v.astype(np.float64)[f[fi]] * bc[:, :, None]).sum(1) + 1e-3 * rng.standard_normal((n, 3))).astype(vdtype)
    pt, vt, ft = (torch.from_numpy(x).cuda() for x in (p, v, f))
    w = pcu.triangle_soup_fast_winding_number(vt, ft, pt)
    assert w.is_cuda and w.dtype == pt.dtype
    rows = torch.from_numpy(rng.choice(n, 1000, replace=False)).cuda()
    ref = exact_w(pt[rows], vt, ft, chunk=8)
    err = float((w[rows].double() - ref).abs().max())
    print("full size max |w(beta = 2) - w(exact)| %s: %.3g" % (np.dtype(vdtype).name, err))
    assert err <= PUBLIC_TOL
    s, sfi, sbc = pcu.signed_distance_to_mesh(pt, vt, ft)
    d, cfi, cbc = pcu.closest_points_on_mesh(pt, vt, ft)
    sigma = (1.0 - 2.0 * w.double().abs()).to(pt.dtype)
    assert sfi.dtype == torch.int32 and torch.equal(sfi, cfi)
    assert torch.equal(sbc, cbc)
    assert torch.equal(s, sigma * d)


@pytest.mark.gpu
def test_input_forms_and_device(pcu):
    import torch
    v, f = icosphere(3, 0.02, 7, np.float32)
    p = queries(v, f, 500, 1)
    w = pcu.triangle_soup_fast_winding_number(v, f, p)
    sd = pcu.signed_distance_to_mesh(p, v, f)
    assert isinstance(w, np.ndarray) and w.dtype == np.float32 and all(isinstance(x, np.ndarray) for x in sd)
    cuda = [torch.from_numpy(x).cuda() for x in (v, f, p)]
    wt = pcu.triangle_soup_fast_winding_number(*cuda)
    sdt = pcu.signed_distance_to_mesh(cuda[2], cuda[0], cuda[1])
    assert wt.is_cuda and all(t.is_cuda for t in sdt) and sdt[1].dtype == torch.int32
    cpu = [torch.from_numpy(x) for x in (v, f, p)]
    wc = pcu.triangle_soup_fast_winding_number(*cpu)
    sdc = pcu.signed_distance_to_mesh(cpu[2], cpu[0], cpu[1])
    assert not wc.is_cuda and all(isinstance(t, torch.Tensor) and not t.is_cuda for t in sdc)
    wd = pcu.triangle_soup_fast_winding_number(v, f, p, device="cuda:0")
    sdd = pcu.signed_distance_to_mesh(p, v, f, device="cuda:0")
    for x in (wt.cpu().numpy(), wc.numpy(), wd):
        assert_bits(x, w, "winding number forms")
    for i in range(3):
        for y in (sdt[i].cpu().numpy(), sdc[i].numpy(), sdd[i]):
            assert np.array_equal(y.view(np.uint8), sd[i].view(np.uint8))


@pytest.mark.gpu
def test_bad_indices_raise_without_a_fault(pcu):
    v, f = icosphere(2)
    p = queries(v, f, 100, 2)
    g = f.astype(np.uint64)
    g[[3, 7], 1] = len(v)
    g[9, 2] = 2 ** 63 + 5
    h = f.astype(np.int32)
    h[[0, 1], 0] = -1
    for bad, count in ((g, 3), (h, 2)):
        with pytest.raises(ValueError, match=r"Invalid face indices: %d faces have a corner outside \[0, #v\)" % count):
            pcu.triangle_soup_fast_winding_number(v, bad, p)
        with pytest.raises(ValueError, match=r"Invalid face indices: %d faces have a corner outside \[0, #v\)" % count):
            pcu.signed_distance_to_mesh(p, v, bad)
    w = pcu.triangle_soup_fast_winding_number(v, f, p)    # the device is fine afterwards
    assert np.abs(w - exact_w(p, v, f)).max() <= PUBLIC_TOL
