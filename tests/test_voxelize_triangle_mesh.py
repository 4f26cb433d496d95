"""voxelize_triangle_mesh: the result of DESIGN.md §3 restated with numpy (fp64, one rounding per operation, in the
reference's order) and pinned to the reference's own triBoxOverlap through oracle/_ref where it is built; the
reference's x loop against the full one; the argument errors; on the GPU, the function bit for bit against the
restatement over every dtype, input form and load shape, and the mesh -> solid pipeline with flood_fill_3d."""
import math

import numpy as np
import pytest

from meshes import to_form, to_numpy

INDEX_DTYPES = [np.int32, np.int64, np.uint32, np.uint64]


# ---- the restatement -----------------------------------------------------------------------------------------------
def _reject(pa, pb, rad):
    lt = pa < pb
    mn, mx = np.where(lt, pa, pb), np.where(lt, pb, pa)
    return (mn > rad) | (mx < -rad)


def _px(a, b, v):
    return a * v[:, 1] - b * v[:, 2]


def _py(a, b, v):
    return (-a) * v[:, 0] + b * v[:, 2]


def _pz(a, b, v):
    return a * v[:, 0] - b * v[:, 1]


def tri_box(c, h, a, b, d):
    """The reference's triBoxOverlap (src/common/tribox.h) over rows: box centres c (K, 3), half size h (3,), corners
    a, b, d (K, 3); fp64, each operation rounded on its own (numpy neither fuses nor reorders)."""
    v0, v1, v2 = a - c, b - c, d - c
    e0, e1, e2 = v1 - v0, v2 - v1, v0 - v2
    rej = np.zeros(len(c), bool)
    for e, second, third in ((e0, (v0, v2), (v2, v1)), (e1, (v0, v2), (v0, v1)), (e2, (v0, v1), (v2, v1))):
        fx, fy, fz = np.abs(e[:, 0]), np.abs(e[:, 1]), np.abs(e[:, 2])
        rej |= _reject(_px(e[:, 2], e[:, 1], second[0]), _px(e[:, 2], e[:, 1], second[1]), fz * h[1] + fy * h[2])
        rej |= _reject(_py(e[:, 2], e[:, 0], second[0]), _py(e[:, 2], e[:, 0], second[1]), fz * h[0] + fx * h[2])
        rej |= _reject(_pz(e[:, 1], e[:, 0], third[0]), _pz(e[:, 1], e[:, 0], third[1]), fy * h[0] + fx * h[1])
    for k in range(3):
        x0, x1, x2 = v0[:, k], v1[:, k], v2[:, k]
        mn, mx = x0.copy(), x0.copy()
        mn = np.where(x1 < mn, x1, mn)
        mx = np.where(x1 > mx, x1, mx)
        mn = np.where(x2 < mn, x2, mn)
        mx = np.where(x2 > mx, x2, mx)
        rej |= (mn > h[k]) | (mx < -h[k])
    n = np.stack([e0[:, 1] * e1[:, 2] - e0[:, 2] * e1[:, 1], e0[:, 2] * e1[:, 0] - e0[:, 0] * e1[:, 2],
                  e0[:, 0] * e1[:, 1] - e0[:, 1] * e1[:, 0]], 1)
    pos = n > 0.0
    vmin = np.where(pos, -h - v0, h - v0)
    vmax = np.where(pos, h - v0, -h - v0)
    dmin = n[:, 0] * vmin[:, 0] + n[:, 1] * vmin[:, 1] + n[:, 2] * vmin[:, 2]
    dmax = n[:, 0] * vmax[:, 0] + n[:, 1] * vmax[:, 1] + n[:, 2] * vmax[:, 2]
    return ~rej & ~(dmin > 0.0) & (dmax >= 0.0)


def accepted(v, f, size, origin, full_x=True, chunk=1 << 21):
    """Every accepted (i, j, k), face by face (candidates z fastest); the faces must be valid."""
    v = np.asarray(v).astype(np.float64)
    f = np.asarray(f).astype(np.int64)
    size, origin = np.asarray(size, np.float64), np.asarray(origin, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    mn = np.minimum(a, np.minimum(b, c))
    mx = np.maximum(a, np.maximum(b, c))
    lo = np.floor((mn - origin) / size).astype(np.int64)
    hi = np.ceil((mx - origin) / size).astype(np.int64)
    ext = hi - lo + 1
    if not full_x:
        ext[:, 0] = 1
    counts = ext.prod(1)
    starts = np.concatenate([[0], np.cumsum(counts)])
    out = []
    for c0 in range(0, int(starts[-1]), chunk):
        q = np.arange(c0, min(c0 + chunk, int(starts[-1])), dtype=np.int64)
        t = np.searchsorted(starts, q, side="right") - 1
        r = q - starts[t]
        nz, ny = ext[t, 2], ext[t, 1]
        ijk = lo[t] + np.stack([r // (nz * ny), (r // nz) % ny, r % nz], 1)
        ctr = origin + ijk.astype(np.float64) * size
        keep = tri_box(ctr, size / 2, a[t], b[t], c[t])
        out.append(ijk[keep].astype(np.int32))
    return np.concatenate(out) if out else np.zeros((0, 3), np.int32)


def restate(v, f, size, origin, oracle, full_x=True):
    """morton_decode(np.unique(morton_encode(accepted))): the reference wrapper's pipeline."""
    ijk = accepted(v, f, size, origin, full_x)
    return oracle.morton_decode(np.unique(oracle.morton_encode(ijk)))


# ---- meshes ----------------------------------------------------------------------------------------------------------
def random_mesh(rng, nv=60, nf=120, scale=4.0, dtype=np.float64):
    v = (rng.standard_normal((nv, 3)) * scale).astype(dtype)
    f = rng.integers(0, nv, (nf, 3))
    f[:5, 1] = f[:5, 0]                                   # zero-area faces: a repeated corner
    v[f[5, 2]] = (v[f[5, 0]].astype(np.float64) * 0.25 + v[f[5, 1]].astype(np.float64) * 0.75).astype(dtype)   # collinear
    return v, f


def on_faces_mesh(rng, size, origin, n=40):
    """Vertices exactly on voxel faces: o + (i + 1/2) s."""
    i = rng.integers(-6, 6, (3 * n, 3)).astype(np.float64)
    v = origin + (i + 0.5) * size
    return v, np.arange(3 * n).reshape(n, 3)


def tilted_cube(k, voxel=1.0):
    """A cube of side k voxels, rotated so its faces cut the grid obliquely: 12 large triangles."""
    c = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64) - 0.5
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                  [0, 6, 4], [1, 5, 7], [1, 7, 3]])
    ax, ay = 0.5, 0.3
    rx = np.array([[1, 0, 0], [0, math.cos(ax), -math.sin(ax)], [0, math.sin(ax), math.cos(ax)]])
    ry = np.array([[math.cos(ay), 0, math.sin(ay)], [0, 1, 0], [-math.sin(ay), 0, math.cos(ay)]])
    return (c @ rx.T @ ry.T) * (k * voxel) + 0.123, f


def sphere_mesh(n_lat=48, n_lon=96, r=1.0):
    """A closed, outward-oriented UV sphere."""
    th = np.linspace(0, math.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * math.pi, n_lon, endpoint=False)
    ring = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.sin(th), np.sin(ph)),
                     np.repeat(np.cos(th)[:, None], n_lon, 1)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], ring, [[0, 0, -1]]]) * r
    f = []
    for j in range(n_lon):
        jn = (j + 1) % n_lon
        f.append([0, 1 + j, 1 + jn])
        for i in range(n_lat - 2):
            a, b = 1 + i * n_lon + j, 1 + i * n_lon + jn
            c, d = a + n_lon, b + n_lon
            f += [[a, c, d], [a, d, b]]
        base = 1 + (n_lat - 2) * n_lon
        f.append([base + j, len(v) - 1, base + jn])
    return v, np.array(f, np.int64)


# ---- restatement against the reference's own test (CPU) -------------------------------------------------------------
@pytest.fixture(scope="module")
def ref(oracle):
    """oracle/voxelize_ref.py: the reference's own triBoxOverlap behind the candidate loop."""
    from oracle import voxelize_ref
    voxelize_ref.build()
    if not voxelize_ref.available():
        pytest.skip("oracle/_ref/libpcu_ref_voxelize.so is built only where a checkout of the reference is present")
    return voxelize_ref


@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", INDEX_DTYPES)
def test_restatement_equals_reference_test(oracle, ref, vdt, idt):
    rng = np.random.default_rng(11)
    v, f = random_mesh(rng, dtype=vdt)
    f = f.astype(idt)
    for size, origin in [((0.7, 0.7, 0.7), (0.0, 0.0, 0.0)), ((0.31, 1.7, 0.9), (-3.3, 0.123, 5.5)), ((2.5, 0.25, 1.0), (1e-3, -7.0, 0.5))]:
        want = ref.voxelize_triangle_mesh(v, f, size, origin, full_x=True)
        got = restate(v, f, size, origin, oracle)
        assert got.dtype == np.int32 and np.array_equal(got, want)


def test_restatement_on_voxel_faces_and_aliasing(oracle, ref):
    rng = np.random.default_rng(3)
    size, origin = np.array([0.5, 0.75, 0.4]), np.array([0.1, -0.2, 0.3])
    v, f = on_faces_mesh(rng, size, origin)
    assert np.array_equal(restate(v, f, size, origin, oracle), ref.voxelize_triangle_mesh(v, f, size, origin))
    # coordinates beyond +-2^20 voxels: the 21-bit Morton fields alias, as in the reference's pipeline
    for shift in (2.0 ** 20 + 3.0, -(2.0 ** 21) - 5.0, 2.0 ** 22):
        v2, f2 = random_mesh(rng, nv=20, nf=30, scale=1.5)
        v2 = v2 + shift
        got = restate(v2, f2, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), oracle)
        assert np.array_equal(got, ref.voxelize_triangle_mesh(v2, f2, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0)))
        assert np.abs(got).max() < 2 ** 21                # decoded codes: 21-bit two's complement


def test_reference_x_loop_is_a_subset(oracle, ref):
    rng = np.random.default_rng(5)
    v, f = random_mesh(rng)
    size, origin = (0.6, 0.45, 0.8), (0.2, 0.1, -0.3)
    full = ref.voxelize_triangle_mesh(v, f, size, origin, full_x=True)
    first_slab = ref.voxelize_triangle_mesh(v, f, size, origin, full_x=False)
    as_set = lambda a: {tuple(r) for r in a}          # noqa: E731
    assert as_set(first_slab) < as_set(full)              # strictly fewer voxels on a random mesh
    assert np.array_equal(restate(v, f, size, origin, oracle, full_x=False), first_slab)


def test_reference_x_loop_equal_on_quarter_offset_planes(oracle, ref):
    """Planes of constant x a quarter voxel past a voxel centre lie within the x extent of their voxel inix: there the
    reference's loop and the full one agree."""
    rng = np.random.default_rng(9)
    size, origin = np.array([0.5, 0.3, 0.7]), np.array([0.05, -0.1, 0.2])
    vs, fs = [], []
    for i, x_idx in enumerate(range(-3, 4)):
        x = origin[0] + (x_idx + 0.25) * size[0]
        yz = rng.uniform(-2, 2, (30, 2))
        vs.append(np.column_stack([np.full(30, x), yz]))
        fs.append(rng.integers(0, 30, (40, 3)) + 30 * i)
    v, f = np.concatenate(vs), np.concatenate(fs)
    full = ref.voxelize_triangle_mesh(v, f, size, origin, full_x=True)
    assert np.array_equal(full, ref.voxelize_triangle_mesh(v, f, size, origin, full_x=False))
    assert np.array_equal(full, restate(v, f, size, origin, oracle))


def test_restatement_without_reference(oracle):
    """Where oracle/_ref is absent: hand-checked voxels of one triangle."""
    v = np.array([[0.1, 0.1, 0.1], [0.2, 0.1, 0.1], [0.1, 0.2, 0.1]])
    f = np.array([[0, 1, 2]])
    assert np.array_equal(restate(v, f, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), oracle), [[0, 0, 0]])
    # the box of voxel 0 is centred at the origin: a triangle at x in [0.6, 0.9] lies in voxel 1 only
    v = np.array([[0.6, 0.0, 0.0], [0.9, 0.0, 0.0], [0.6, 0.1, 0.0]])
    assert np.array_equal(restate(v, f, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), oracle), [[1, 0, 0]])


# ---- argument errors (CPU: raised before any device call) -----------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    v = np.random.default_rng(0).random((10, 3))
    f = np.array([[0, 1, 2], [3, 4, 5]])
    vox = pcu.voxelize_triangle_mesh
    cases = [
        ((v, f, 1.0, (0, 0)), "expected 3D coordinate"),
        ((v, f, 1.0, 0.0), "expected 3D coordinate"),
        ((v, f, (1.0, 1.0), (0, 0, 0)), "expected 3D coordinate"),
        ((v, f, np.float32(1.0), (0, 0, 0)), "expected 3D coordinate"),   # not a Python float: the reference's rule
        ((v.astype(np.int32), f, 1.0, (0, 0, 0)), "Invalid scalar type (int32) for argument 'v'"),
        ((v, f.astype(np.float32), 1.0, (0, 0, 0)), "Invalid scalar type (float32) for argument 'f'"),
        ((v[:0], f, 1.0, (0, 0, 0)), "Invalid input mesh with zero elements"),
        ((v, f[:0], 1.0, (0, 0, 0)), "Invalid input mesh with zero elements"),
        ((v[:, :2], f, 1.0, (0, 0, 0)), "Only 3D inputs are supported"),
        ((v, f, 0.0, (0, 0, 0)), "Invalid voxel size"),
        ((v, f, (1.0, -1.0, 1.0), (0, 0, 0)), "Invalid voxel size"),
        ((list(v), f, 1.0, (0, 0, 0)), "Invalid type for v"),
        # the reference's order: the coordinates are converted before the arrays are looked at
        ((v.astype(np.int32), f, 1.0, (0, 0)), "expected 3D coordinate"),
        ((v[:0], f, 0.0, (0, 0, 0)), "Invalid input mesh with zero elements"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            vox(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        vox(v, f, 1.0, (0, 0, 0), None)                   # device= is keyword only


# ---- the GPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", INDEX_DTYPES)
def test_equals_restatement_every_dtype(pcu, oracle, vdt, idt):
    rng = np.random.default_rng(21)
    v, f = random_mesh(rng, nv=200, nf=300, scale=2.0, dtype=vdt)
    for size, origin in [(0.5, (0.0, 0.0, 0.0)), ((0.31, 1.7, 0.9), (-3.3, 0.123, 5.5))]:
        got = pcu.voxelize_triangle_mesh(v, f.astype(idt), size, origin)
        s3 = np.array([size] * 3 if np.isscalar(size) else size)
        want = restate(v, f, s3, origin, oracle)
        assert got.dtype == np.int32 and np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms(pcu, oracle, form):
    import torch
    rng = np.random.default_rng(4)
    v, f = random_mesh(rng, nv=200, nf=500, scale=2.0, dtype=np.float32)
    got = pcu.voxelize_triangle_mesh(to_form(form, v), to_form(form, f), (0.4, 0.6, 0.5), (0.1, 0.2, 0.3))
    if form == "cuda":
        assert isinstance(got, torch.Tensor) and got.is_cuda and got.dtype == torch.int32
    elif form == "cpu":
        assert isinstance(got, torch.Tensor) and not got.is_cuda
    assert np.array_equal(to_numpy(got), restate(v, f, (0.4, 0.6, 0.5), (0.1, 0.2, 0.3), oracle))


@pytest.mark.gpu
def test_voxel_faces_degenerate_and_aliasing(pcu, oracle):
    rng = np.random.default_rng(8)
    size, origin = np.array([0.5, 0.75, 0.4]), np.array([0.1, -0.2, 0.3])
    v, f = on_faces_mesh(rng, size, origin, n=300)
    assert np.array_equal(pcu.voxelize_triangle_mesh(v, f, size, origin), restate(v, f, size, origin, oracle))
    for shift in (2.0 ** 20 + 3.0, -(2.0 ** 21) - 5.0, 2.0 ** 22, 1.5e9):
        v2, f2 = random_mesh(rng, nv=100, nf=200, scale=2.0)
        v2 = v2 + shift
        got = pcu.voxelize_triangle_mesh(v2, f2, 1.0, (0.0, 0.0, 0.0))
        assert np.array_equal(got, restate(v2, f2, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), oracle))


@pytest.mark.gpu
def test_tilted_cube_large_faces(pcu, oracle):
    """12 faces of about 10^6 candidates each: every face spans many CTAs' slices."""
    v, f = tilted_cube(100)
    got = pcu.voxelize_triangle_mesh(v, f, 1.0, (0.0, 0.0, 0.0))
    assert np.array_equal(got, restate(v, f, (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), oracle))


@pytest.mark.gpu
def test_million_faces(pcu, oracle):
    v, f = sphere_mesh(708, 708)                          # 10^6 faces
    assert len(f) >= 10 ** 6
    for vdt in (np.float32, np.float64):
        size = 1.0 / 128
        got = pcu.voxelize_triangle_mesh(v.astype(vdt), f, size, (0.0, 0.0, 0.0))
        assert np.array_equal(got, restate(v.astype(vdt), f, (size,) * 3, (0.0, 0.0, 0.0), oracle))


@pytest.mark.gpu
def test_device_errors(pcu):
    v = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    with pytest.raises(ValueError, match="faces have a corner outside"):
        pcu.voxelize_triangle_mesh(v, np.array([[0, 1, 3]]), 1.0, (0, 0, 0))
    with pytest.raises(ValueError, match="non-finite vertex or voxel index bounds"):
        pcu.voxelize_triangle_mesh(np.where(v == 1.0, np.inf, v), np.array([[0, 1, 2]]), 1.0, (0, 0, 0))
    with pytest.raises(ValueError, match="non-finite vertex or voxel index bounds"):   # ceil = INT32_MAX: the reference never ends
        pcu.voxelize_triangle_mesh(v + 2147483646.5, np.array([[0, 1, 2]]), 1.0, (0, 0, 0))
    with pytest.raises(ValueError, match="overflow a 64-bit count"):
        big = np.array([[-1e9, -1e9, -1e9], [1e9, 1e9, 1e9], [1e9, -1e9, 0.0]])
        pcu.voxelize_triangle_mesh(big, np.array([[0, 1, 2]]), 0.5, (0, 0, 0))


@pytest.mark.gpu
def test_mesh_to_solid_pipeline(pcu):
    """Voxelize a closed sphere, flood the exterior of a grid padded by one voxel from a corner, and check the solid with
    winding numbers and the sphere's volume."""
    v, f = sphere_mesh(64, 128, r=1.0)
    s = 1.0 / 24
    ijk = pcu.voxelize_triangle_mesh(v, f, s, (0.0, 0.0, 0.0))
    lo = ijk.min(0) - 1
    shape = tuple(ijk.max(0) - lo + 2)
    grid = np.zeros(shape, np.int32)
    grid[tuple((ijk - lo).T)] = 1                         # surface voxels
    filled = pcu.flood_fill_3d(grid, (0, 0, 0), 2)
    assert filled[0, 0, 0] == 2 and (filled[grid == 1] == 1).all()
    centres = (np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), -1).reshape(-1, 3) + lo) * s
    wn = pcu.triangle_soup_fast_winding_number(v, f, centres).reshape(shape)
    assert (wn[filled == 2] < 0.5).all()
    assert (wn[filled == 0] > 0.5).all()
    solid = int((filled != 2).sum())
    exact = 4.0 / 3.0 * math.pi / s ** 3
    shell = 2.0 * 4.0 * math.pi / s ** 2                  # tolerance: two voxel layers of the sphere's surface
    assert abs(solid - exact) <= shell, (solid, exact)
