"""mesh_face_areas, estimate_mesh_face_normals and estimate_mesh_vertex_normals: the results of DESIGN.md §3 restated
with vectorised numpy; the area restatement pinned bit for bit to a literal scalar transcription of the reference's
loop (src/face_areas.cpp:54-70) in float32 and float64; the argument errors in the reference's order; on the GPU, the
three functions against the restatements (bit for bit, the angle weights within 1e-13 in float64 and 1 ulp in
float32, or 1e-13 where a component's ulp is finer) over every dtype and input form, the squeezed shapes, degenerate and
repeated-corner faces, isolated vertices, a fan of 10^5 faces around one vertex (whose pole sums 10^5 angles and is held
to 1e-10) and a 1.3 * 10^6-face icosphere."""
import numpy as np
import pytest

from meshes import icosphere, to_form, to_numpy

IDX = [np.int32, np.int64, np.uint32, np.uint64]
DBL_MAX = np.finfo(np.float64).max


# ---- the restatements -----------------------------------------------------------------------------------------------
def restate_areas(v, f):
    """Heron's formula in v's precision, operation for operation as src/face_areas.cpp computes it."""
    T = v.dtype.type
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]

    def norm(d):
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])

    a, b, c = norm(p1 - p0), norm(p2 - p1), norm(p0 - p2)
    p = ((a + b) + c) * T(0.5)

    def mx(x):
        return np.where(x < 0, T(0), x)

    return np.sqrt(((p * mx(p - a)) * mx(p - b)) * mx(p - c))


def literal_areas(v, f):
    """src/face_areas.cpp:54-70, one face at a time with numpy scalars of v's type (0.5 is a double in the C++)."""
    R = v.dtype.type
    areas = np.zeros(f.shape[0], v.dtype)
    for i in range(f.shape[0]):
        v1, v2, v3 = v[f[i, 0]], v[f[i, 1]], v[f[i, 2]]

        def nrm(d):
            return R(np.sqrt(R(R(d[0] * d[0]) + R(d[1] * d[1])) + R(d[2] * d[2])))

        a, b, c = nrm(v2 - v1), nrm(v3 - v2), nrm(v1 - v3)
        p = R(np.float64(0.5) * np.float64(R(R(a + b) + c)))
        mx = lambda x: R(0.0) if x < R(0.0) else x   # std::max(x, 0): (x < 0) ? 0 : x
        areas[i] = R(np.sqrt(R(R(R(p * mx(R(p - a))) * mx(R(p - b))) * mx(R(p - c)))))
    return areas


def cross(a, b, c):
    """(b - a) x (c - a) and its norm sqrt((x x + y y) + z z), fp64 (the order of face_area in csrc/meshsample.cuh)."""
    e1, e2 = b - a, c - a
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    return n, np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])


def face_area(a, b, c):
    """face_area of csrc/meshsample.cuh: |(b - a) x (c - a)|, 0 where it is not finite."""
    A = cross(a, b, c)[1]
    return np.where((A >= 0) & (A <= DBL_MAX), A, 0.0)


def corner_dot(a, b, c):
    d1, d2 = b - a, c - a
    return (d1[:, 0] * d2[:, 0] + d1[:, 1] * d2[:, 1]) + d1[:, 2] * d2[:, 2]


def unit_rows(n, ln):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ln[:, None] == 0, 0.0, n / ln[:, None])


def restate_face_normals_f64(v, f):
    p = v.astype(np.float64)
    return unit_rows(*cross(p[f[:, 0]], p[f[:, 1]], p[f[:, 2]]))


def restate_face_normals(v, f):
    return restate_face_normals_f64(v, f).astype(v.dtype)


def corner_weights(v, f, weighting):
    """(m, 3) weights of the corners: |e1 x e2| ('area') or atan2(|e1 x e2|, e1 . e2) ('angle')."""
    p = v.astype(np.float64)
    q = [p[f[:, 0]], p[f[:, 1]], p[f[:, 2]]]
    if weighting == "area":
        return np.repeat(face_area(*q)[:, None], 3, 1)
    return np.stack([np.arctan2(face_area(q[k], q[(k + 1) % 3], q[(k + 2) % 3]), corner_dot(q[k], q[(k + 1) % 3], q[(k + 2) % 3]))
                     for k in range(3)], 1)


def restate_vertex_normals(v, f, weighting="uniform"):
    """Sum of w n_f over every vertex's corners in ascending (face, corner) order (np.add.at is a sequential loop over
    its indices), normalised; fp64, rounded once."""
    nf = restate_face_normals_f64(v, f)
    contrib = np.repeat(nf, 3, 0)
    if weighting != "uniform":
        contrib = corner_weights(v, f, weighting).reshape(-1, 1) * contrib
    N = np.zeros((v.shape[0], 3))
    np.add.at(N, f.astype(np.int64).ravel(), contrib)
    ln = np.sqrt((N[:, 0] * N[:, 0] + N[:, 1] * N[:, 1]) + N[:, 2] * N[:, 2])
    return unit_rows(N, ln).astype(v.dtype)


# ---- meshes ---------------------------------------------------------------------------------------------------------
def random_mesh(rng, nv, m, vdt, idt):
    v = (rng.standard_normal((nv, 3)) * rng.choice([1e-3, 1.0, 1e3])).astype(vdt)
    f = rng.integers(0, nv, (m, 3)).astype(idt)
    return v, f


def fan(n):
    """n faces around vertex 0 (a pole), each with two rim vertices of its own ring."""
    ang = np.linspace(0.0, 2 * np.pi, n, endpoint=False)
    rim = np.stack([np.cos(ang), np.sin(ang), 0.1 * np.sin(7 * ang)], 1)
    v = np.concatenate([[[0.0, 0.0, 1.0]], rim])
    i = np.arange(n)
    f = np.stack([np.zeros(n, np.int64), 1 + i, 1 + (i + 1) % n], 1)
    return v, f


# ---- the CPU --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
def test_areas_restatement_is_the_reference_loop(vdt):
    rng = np.random.default_rng(1)
    for nv, m in ((5, 40), (50, 300), (200, 200)):
        v, f = random_mesh(rng, nv, m, vdt, np.int64)
        f[:5, 1] = f[:5, 0]                                  # repeated corners
        v[-1] = v[-2] + (v[-2] - v[-3])                      # collinear
        f[5] = [nv - 3, nv - 2, nv - 1]
        r, lit = restate_areas(v, f), literal_areas(v, f)
        assert r.dtype == lit.dtype == vdt
        assert np.array_equal(r.view(np.uint8), lit.view(np.uint8))


def test_unit_right_triangle():
    v = np.array([[0.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
    f = np.array([[0, 1, 2]])
    a = restate_areas(v, f)[0]
    assert a == literal_areas(v, f)[0] and abs(a - 0.5) < 1e-15     # Heron's formula rounds: 0.49999999999999983
    a32 = restate_areas(v.astype(np.float32), f)[0]
    assert a32 == literal_areas(v.astype(np.float32), f)[0] and abs(a32 - 0.5) < 1e-6


def test_normals_restatement_basics():
    v = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [5.0, 5.0, 5.0]])
    f = np.array([[0, 1, 2], [0, 0, 1], [3, 3, 3]])
    n = restate_face_normals(v, f)
    assert np.array_equal(n, [[0, 0, 1], [0, 0, 0], [0, 0, 0]])
    vn = restate_vertex_normals(v, f, "angle")
    assert np.array_equal(vn[3], [0, 0, 0]) and np.allclose(vn[:3], [[0, 0, 1]] * 3)
    w = corner_weights(v, f[:1], "angle")
    assert np.allclose(w[0], [np.pi / 2, np.pi / 4, np.pi / 4])


def test_argument_errors(pcu):
    mg = pcu
    v = np.zeros((4, 3))
    f = np.array([[0, 1, 2]], np.int64)
    for fn in (mg.mesh_face_areas, mg.estimate_mesh_face_normals, mg.estimate_mesh_vertex_normals):
        cases = [
            ((v.astype(np.int32), f), "Invalid scalar type (int32) for argument 'v'"),
            ((v, f.astype(np.float32)), "Invalid scalar type (float32) for argument 'f'"),
            ((v, f.astype(np.int32).astype(np.float32)[:0]), "Invalid scalar type"),
            ((v[:0], f), "Invalid input mesh with zero elements"),
            ((v, f[:0]), "Invalid input mesh with zero elements"),
            ((v[:, :2], f), "Only 3D inputs are supported"),
            ((v, f[:, :2]), "Only 3D inputs are supported"),
            ((v[0], f), "Only 3D inputs are supported"),
            ((list(v), f), "Invalid type for v"),
            ((v, list(f)), "Invalid type for f"),
            ((v.astype(np.int32), f.astype(np.float32)), "for argument 'v'"),   # the reference's order: v first
        ]
        for args, msg in cases:
            with pytest.raises(ValueError) as e:
                fn(*args)
            assert msg in str(e.value), (fn.__name__, msg, str(e.value))
        with pytest.raises(TypeError):
            fn(v, f, "uniform", None)                                          # device= is keyword only
    with pytest.raises(ValueError, match="for argument 'f'. Expected one of \\['int32', 'int64'\\]"):
        mg.mesh_face_areas(v, f.astype(np.uint32))
    with pytest.raises(ValueError, match="Invalid weighting_type must be one of 'uniform', 'angle', or 'area', but got 'cot'"):
        mg.estimate_mesh_vertex_normals(v, f, "cot")
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):   # the mesh before the weighting
        mg.estimate_mesh_vertex_normals(v, f[:0], "cot")


# ---- the GPU --------------------------------------------------------------------------------------------------------
def same(got, want):
    got = to_numpy(got)
    return got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8))


def close_angle(got, want, tol=1e-13):
    """Within tol per component in float64; in float32 within 1 ulp of the restatement, or within tol where a
    component is so close to 0 that its ulp is finer than tol."""
    got = to_numpy(got)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    if want.dtype == np.float64:
        return diff.max(initial=0.0) <= tol
    return bool(np.all(diff <= np.maximum(np.spacing(np.abs(want)).astype(np.float64), tol)))


def check_all(pcu, v, f, areas=True, angle=True):
    if areas:
        assert same(pcu.mesh_face_areas(v, f), restate_areas(v, f)), "areas"
    assert same(pcu.estimate_mesh_face_normals(v, f), restate_face_normals(v, f)), "face normals"
    for w in ("uniform", "area"):
        assert same(pcu.estimate_mesh_vertex_normals(v, f, w), restate_vertex_normals(v, f, w)), w
    if angle:
        assert close_angle(pcu.estimate_mesh_vertex_normals(v, f, "angle"), restate_vertex_normals(v, f, "angle")), "angle"


@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", IDX)
def test_every_dtype(pcu, vdt, idt):
    rng = np.random.default_rng(2)
    for nv, m in ((300, 500), (5000, 9000), (40, 3)):
        v, f = random_mesh(rng, nv, m, vdt, idt)
        f[:7, 2] = f[:7, 1]                                  # repeated corners
        f[-1] = [0, 0, 0]
        check_all(pcu, v, f, areas=idt in (np.int32, np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms(pcu, form):
    import torch
    rng = np.random.default_rng(3)
    v, f = random_mesh(rng, 400, 600, np.float32, np.int64)
    kind = np.ndarray if form == "numpy" else torch.Tensor
    outs = [pcu.mesh_face_areas(to_form(form, v), to_form(form, f)), pcu.estimate_mesh_face_normals(to_form(form, v), to_form(form, f)),
            pcu.estimate_mesh_vertex_normals(to_form(form, v), to_form(form, f), "area")]
    assert all(isinstance(o, kind) and (form == "numpy" or o.is_cuda == (form == "cuda")) for o in outs)
    assert same(outs[0], restate_areas(v, f))
    assert same(outs[1], restate_face_normals(v, f))
    assert same(outs[2], restate_vertex_normals(v, f, "area"))


@pytest.mark.gpu
def test_shapes_degenerate_and_isolated(pcu):
    v = np.array([[0.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [3.0, 3.0, 3.0]])
    f = np.array([[0, 1, 2]])
    a = pcu.mesh_face_areas(v, f)
    assert a.shape == () and abs(float(a) - 0.5) < 1e-15
    n = pcu.estimate_mesh_face_normals(v, f)
    assert n.shape == (3,) and np.array_equal(n, [0.0, 0.0, -1.0])
    vn = pcu.estimate_mesh_vertex_normals(v, f)
    assert vn.shape == (4, 3) and np.array_equal(vn[3], [0.0, 0.0, 0.0])   # the isolated vertex
    vn = pcu.estimate_mesh_vertex_normals(v[:1], np.array([[0, 0, 0]], np.uint32))
    assert vn.shape == (3,) and np.array_equal(vn, [0.0, 0.0, 0.0])
    fd = np.array([[0, 1, 2], [0, 0, 1], [1, 2, 2], [3, 3, 3], [0, 2, 1]])      # degenerate, repeated, opposite
    check_all(pcu, v, fd)
    check_all(pcu, v.astype(np.float32), fd.astype(np.int32))


@pytest.mark.gpu
def test_fan_around_one_vertex(pcu):
    v, f = fan(100000)
    for vdt in (np.float64, np.float32):
        v = v.astype(vdt)
        check_all(pcu, v, f, angle=False)
        got, want = to_numpy(pcu.estimate_mesh_vertex_normals(v, f, "angle")), restate_vertex_normals(v, f, "angle")
        assert close_angle(got[1:], want[1:])
        # the pole sums 10^5 angles, each within an ulp or so of numpy's arctan2: the tolerance grows with the count
        assert close_angle(got[:1], want[:1], 1e5 * 1e-15)


@pytest.mark.gpu
def test_large_icosphere(pcu):
    v, f = icosphere(8)
    v = v * (1.0 + 0.01 * np.random.default_rng(4).standard_normal((len(v), 1)))
    for vdt in (np.float64, np.float32):
        check_all(pcu, v.astype(vdt), f)
    again = pcu.estimate_mesh_vertex_normals(v, f, "angle")
    assert same(again, to_numpy(pcu.estimate_mesh_vertex_normals(v, f, "angle")))


@pytest.mark.gpu
def test_corner_errors(pcu):
    v = np.zeros((5, 3))
    for f in (np.array([[0, 1, 5], [0, 1, 2], [-1, 0, 0]], np.int64), np.array([[0, 1, 7], [0, 1, -1]], np.int32)):
        for fn in (pcu.mesh_face_areas, pcu.estimate_mesh_face_normals, pcu.estimate_mesh_vertex_normals):
            with pytest.raises(ValueError, match="Invalid face indices: 2 faces have a corner outside"):
                fn(v, f)
    with pytest.raises(ValueError, match="Invalid face indices: 1 faces"):
        pcu.estimate_mesh_vertex_normals(v, np.array([[0, 1, 2 ** 32 - 1]], np.uint32))
