"""pointcloud_sphere_geometry: the reference's make_sphere_geometry of DESIGN.md §3 restated with numpy (a cos / sin
table from the C library, then every fp64 product and sum rounded on its own) and pinned to a literal transcription of
its loops at 1 to 3 stacks and slices; the argument errors and the signature; on the GPU, vertices and faces bit for
bit equal to the restatement over both dtypes, every radius form and input form, stacks x slices in {1, 2, 3, 16} x
{1, 2, 3, 32}, one point, zero points, 2 * 10^4 points at 16 x 32, a sample of 10^6 points at 8 x 8, and the int32
bound."""
import inspect
import math

import numpy as np
import pytest

from meshes import to_form, to_numpy

STACKS = [1, 2, 3, 16]
SLICES = [1, 2, 3, 32]


# ---- the restatement ------------------------------------------------------------------------------------------------
def table(stacks, slices):
    """cos and sin of the reference's stack angles pi / 2 - a (pi / stacks) and sector angles b (2 pi / slices), in
    fp64, from the C library (Python's math module calls it)."""
    sa = [math.pi / 2 - a * (math.pi / stacks) for a in range(stacks + 1)]
    sb = [b * (2 * math.pi / slices) for b in range(slices + 1)]
    return tuple(np.array([fn(x) for x in xs]) for xs in (sa, sb) for fn in (math.cos, math.sin))


def face_template(stacks, slices):
    """One sphere's faces (0-based) in the reference's loop order: per stack a and sector j, (k1, k2, k1 + 1) unless
    a = 0, then (k1 + 1, k2, k2 + 1) unless a = stacks - 1."""
    k1 = np.arange(stacks)[:, None] * (slices + 1) + np.arange(slices)[None, :]
    k2 = k1 + slices + 1
    both = np.stack([np.stack([k1, k2, k1 + 1], -1), np.stack([k1 + 1, k2, k2 + 1], -1)], 2)   # (stacks, slices, 2, 3)
    keep = np.ones((stacks, slices, 2), bool)
    keep[0, :, 0] = False
    keep[-1, :, 1] = False
    return both[keep]


def restate(p, r, stacks, slices):
    """(vertices (#p V, 3) in p's dtype, faces (#p F, 3) int32); r already in p's dtype."""
    p = np.asarray(p)
    T = p.dtype
    cs, ss, cb, sb = table(stacks, slices)
    r64 = np.asarray(r, T).astype(np.float64)[:, None, None]
    xy, z = r64 * cs[None, :, None], r64 * ss[None, :, None]        # (n, stacks + 1, 1)
    x, y = xy * cb[None, None, :], xy * sb[None, None, :]           # (n, stacks + 1, slices + 1)
    z = np.broadcast_to(z, x.shape)
    p64 = p.astype(np.float64)
    v = np.stack([p64[:, 0, None, None] + x, p64[:, 1, None, None] + y, p64[:, 2, None, None] + z], -1).astype(T)
    V = (stacks + 1) * (slices + 1)
    f = face_template(stacks, slices)[None] + (np.arange(len(p)) * V)[:, None, None]
    return v.reshape(-1, 3), f.reshape(-1, 3).astype(np.int32)


def literal(p, r, stacks, slices):
    """generate_splat_geometry ("sphere") with make_sphere_geometry, loop by loop in Python floats (fp64)."""
    T = np.asarray(p).dtype.type
    V, F = (stacks + 1) * (slices + 1), (stacks - 1) * slices * 2
    out_v = np.zeros((len(p) * V, 3), T)
    out_f = np.zeros((len(p) * F, 3), np.int32)
    for i in range(len(p)):
        radius = float(T(r[i]))
        base_x, base_y, base_z = (float(T(c)) for c in p[i])
        sector_step, stack_step = 2 * math.pi / slices, math.pi / stacks
        cur = i * V
        for a in range(stacks + 1):
            stack_angle = math.pi / 2 - a * stack_step
            xy = radius * math.cos(stack_angle)
            z = radius * math.sin(stack_angle)
            for b in range(slices + 1):
                sector_angle = b * sector_step
                x = xy * math.cos(sector_angle)
                y = xy * math.sin(sector_angle)
                out_v[cur] = (T(base_x + x), T(base_y + y), T(base_z + z))
                cur += 1
        idx = i * F
        for a in range(stacks):
            k1 = a * (slices + 1)
            k2 = k1 + slices + 1
            for _ in range(slices):
                if a != 0:
                    out_f[idx] = (i * V + k1, i * V + k2, i * V + k1 + 1)
                    idx += 1
                if a != stacks - 1:
                    out_f[idx] = (i * V + k1 + 1, i * V + k2, i * V + k2 + 1)
                    idx += 1
                k1 += 1
                k2 += 1
    return out_v, out_f


def cloud(seed, m, dtype):
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((m, 3)) * 10.0 ** rng.integers(-3, 4, (m, 1))
    r = 10.0 ** rng.uniform(-4, 1, m)
    return p.astype(dtype), r.astype(dtype)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("stacks", [1, 2, 3])
@pytest.mark.parametrize("slices", [1, 2, 3])
def test_restatement_equals_literal(dtype, stacks, slices):
    p, r = cloud(stacks * 7 + slices, 5, dtype)
    v, f = restate(p, r, stacks, slices)
    lv, lf = literal(p, r, stacks, slices)
    assert bits_equal(v, lv) and bits_equal(f, lf)
    assert v.shape == (5 * (stacks + 1) * (slices + 1), 3) and f.shape == (5 * 2 * (stacks - 1) * slices, 3)


def test_restatement_shape():
    """A unit sphere at the origin: the poles, the equator and the seam duplicated as the reference has them."""
    v, f = restate(np.zeros((1, 3)), np.ones(1), 2, 4)
    assert v.shape == (15, 3) and f.shape == (8, 3)
    assert np.allclose(v[:5], [0, 0, 1]) and np.allclose(v[10:], [0, 0, -1])
    assert np.allclose(v[5], v[9]) and np.allclose(v[5], [1, 0, 0], atol=1e-15)
    assert f[:4].tolist() == [[1, 5, 6], [2, 6, 7], [3, 7, 8], [4, 8, 9]]
    assert f[4:].tolist() == [[5, 10, 6], [6, 11, 7], [7, 12, 8], [8, 13, 9]]


# ---- CPU: interface and argument errors ---------------------------------------------------------------------------
def test_signature(pcu):
    ps = list(inspect.signature(pcu.pointcloud_sphere_geometry).parameters.values())
    assert [q.name for q in ps] == ["p", "r", "num_stacks", "num_slices", "device"]
    assert all(q.kind == inspect.Parameter.POSITIONAL_OR_KEYWORD and q.default is inspect.Parameter.empty for q in ps[:4])
    assert ps[4].kind == inspect.Parameter.KEYWORD_ONLY and ps[4].default is None
    assert "pointcloud_sphere_geometry" in pcu.__all__


def test_argument_errors(pcu):
    p = np.random.default_rng(0).random((4, 3))
    sg = pcu.pointcloud_sphere_geometry
    cases = [
        ((p, None, 4, 4), "Argument r must be a scalar or numpy array with the same number of rows as p"),
        ((p, np.ones(3), 4, 4), "Argument r have the same number of rows as p"),
        ((p, np.ones((4, 2)), 4, 4), "Invalid shape for argument r, must have shape (N,) or (N, 1)"),
        ((p.astype(np.int64), None, 4, 4), "Argument r must be a scalar"),                # r is checked first
        ((p.astype(np.int64), 0.1, 4, 4), "Invalid scalar type (int64) for argument 'v'. Expected one of ['float32', 'float64']."),
        ((p[:, :2], 0.1, 4, 4), "Only 3D inputs are supported: p must have shape (n, 3)"),
        ((p.ravel()[:4], 0.1, 4, 4), "Only 3D inputs are supported"),
        ((p, 0.1, 0, 4), "num_stacks and num_slices must be at least 1, got 0 and 4"),
        ((p, 0.1, 4, 0), "num_stacks and num_slices must be at least 1, got 4 and 0"),
        ((p, 0.1, -1, -1), "must be at least 1"),
        ((p[:1], 0.1, 46340, 46340), "int32 faces index at most 2^31 - 2 vertices"),      # V = 46341^2 > 2^31
        ((p, 0.1, 23170, 23170), "int32 faces index at most 2^31 - 2 vertices"),          # 4 V > 2^31
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            sg(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        sg(p, 0.1, 4, 4, None)                                  # device= is keyword only


def test_zero_points_without_a_device(pcu):
    for dt in (np.float32, np.float64):
        v, f = pcu.pointcloud_sphere_geometry(np.zeros((0, 3), dt), 0.5, 8, 8)
        assert v.shape == (0, 3) and v.dtype == dt and f.shape == (0, 3) and f.dtype == np.int32


# ---- GPU ------------------------------------------------------------------------------------------------------------
def r_form(r, k):
    """Scalar, (N,), (N, 1), list; k = 0 takes r[0] for every point."""
    return [float(r[0]), r, r[:, None], list(r)][k % 4]


def r_value(r, k, dtype):
    return np.full(len(r), float(r[0])).astype(dtype) if k % 4 == 0 else np.asarray(r).astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("stacks", STACKS)
def test_bits(pcu, dtype, stacks):
    p, r = cloud(stacks, 37, dtype)
    for k, slices in enumerate(SLICES):
        for rk in range(4):
            v, f = pcu.pointcloud_sphere_geometry(p, r_form(r, rk), stacks, slices)
            wv, wf = restate(p, r_value(r, rk, dtype), stacks, slices)
            assert bits_equal(v, wv), (stacks, slices, rk)
            assert bits_equal(f, wf), (stacks, slices, rk)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms(pcu, form):
    import torch
    for dtype in (np.float32, np.float64):
        p, r = cloud(5, 19, dtype)
        for rk, rr in enumerate([0.25, r, r[:, None], list(r), to_form(form, r) if form != "numpy" else r]):
            v, f = pcu.pointcloud_sphere_geometry(to_form(form, p), rr, 3, 5)
            if form != "numpy":
                assert isinstance(v, torch.Tensor) and v.is_cuda == (form == "cuda") and f.dtype == torch.int32
            wv, wf = restate(p, (np.full(19, 0.25) if rk == 0 else r).astype(dtype), 3, 5)
            assert bits_equal(to_numpy(v), wv) and bits_equal(to_numpy(f), wf)


@pytest.mark.gpu
def test_one_and_zero_points(pcu):
    import torch
    p = np.array([[1.5, -2.0, 0.25]], np.float32)
    v, f = pcu.pointcloud_sphere_geometry(p, 0.75, 16, 32)
    wv, wf = restate(p, np.array([0.75], np.float32), 16, 32)
    assert bits_equal(v, wv) and bits_equal(f, wf)
    assert np.allclose(np.linalg.norm(v.astype(np.float64) - p, axis=1), 0.75, rtol=1e-6)
    v, f = pcu.pointcloud_sphere_geometry(torch.zeros((0, 3), dtype=torch.float64, device="cuda"), 0.5, 8, 8)
    assert v.shape == (0, 3) and v.is_cuda and v.dtype == torch.float64 and f.shape == (0, 3) and f.dtype == torch.int32
    v, f = pcu.pointcloud_sphere_geometry(np.zeros((0, 3), np.float32), np.zeros(0), 8, 8)
    assert v.shape == (0, 3) and f.shape == (0, 3)


@pytest.mark.gpu
def test_many_points(pcu):
    for dtype in (np.float32, np.float64):
        p, r = cloud(11, 20000, dtype)
        v, f = pcu.pointcloud_sphere_geometry(p, r, 16, 32)
        wv, wf = restate(p, r, 16, 32)
        assert bits_equal(v, wv) and bits_equal(f, wf)


@pytest.mark.gpu
def test_million_points_sampled(pcu):
    import torch
    p, r = cloud(12, 1_000_000, np.float32)
    V, F = 81, 112
    v, f = pcu.pointcloud_sphere_geometry(torch.from_numpy(p).cuda(), torch.from_numpy(r).cuda(), 8, 8)
    assert v.shape == (1_000_000 * V, 3) and f.shape == (1_000_000 * F, 3)
    pick = np.sort(np.random.default_rng(13).choice(1_000_000, 2000, replace=False))
    pick[-1] = 999_999
    sel = torch.from_numpy(pick).cuda()
    gv = v.view(-1, V, 3)[sel].cpu().numpy().reshape(-1, 3)
    gf = f.view(-1, F, 3)[sel].cpu().numpy()
    wv, _ = restate(p[pick], r[pick], 8, 8)
    wf = face_template(8, 8)[None] + (pick * V)[:, None, None]
    assert bits_equal(gv, wv) and np.array_equal(gf, wf)
    assert int(f.max()) == 1_000_000 * V - 2 and int(f.min()) == 1     # the last seam vertex and the first north pole are never named


@pytest.mark.gpu
def test_int32_bound(pcu):
    import torch
    p = torch.zeros((26512, 3), dtype=torch.float32, device="cuda")      # 26512 * 284 * 286 > 2^31 - 1
    with pytest.raises(ValueError, match="int32 faces index at most 2\\^31 - 2 vertices"):
        pcu.pointcloud_sphere_geometry(p, 0.1, 283, 285)
