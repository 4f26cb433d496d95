"""sparse_voxel_grid_from_pointcloud, dilate_sparse_voxel_grid, erode_sparse_voxel_grid and
sparse_voxel_grid_to_hex_mesh: numpy restatements of the definitions in DESIGN.md §3 (built on the oracle's Morton
functions, the reference's own MortonCode64 where oracle/_ref was built), pinned to loop-by-loop transcriptions of the
reference's bindings (src/sparse_voxel_grid.cpp:78-460, with its literal 26-entry table and its 0.5 * gx) and to
set-based definitions; argument errors; on the GPU, the functions against the restatements in every form, at scale,
and the points -> grid -> dilate -> hex mesh -> SDF -> marching cubes pipeline."""
import bisect

import numpy as np
import pytest

from meshes import to_form, to_numpy
from oracle import oracle as O

OVERFLOW = "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small."
OFF26 = [(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
# the reference's table (src/sparse_voxel_grid.cpp:171-200 and :256-285), repeats included
REF26 = [(-1, -1, -1), (-1, -1, 0), (-1, -1, 1), (-1, 0, -1), (-1, 0, 0), (-1, 0, 1), (-1, 1, -1), (-1, 1, 0), (-1, 0, 1),
         (0, -1, -1), (0, -1, 0), (0, -1, 1), (0, 0, -1), (0, 0, 1), (0, 1, -1), (0, 1, 0), (0, 0, 1),
         (1, -1, -1), (1, -1, 0), (1, -1, 1), (1, 0, -1), (1, 0, 0), (1, 0, 1), (1, 1, -1), (1, 1, 0), (1, 0, 1)]
NEVER = [(-1, 1, 1), (0, 1, 1), (1, 1, 1)]     # the offsets the reference's table never visits
CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]


# ---- Morton codes through the oracle --------------------------------------------------------------------------------
def enc(g):
    return O.morton_encode(np.asarray(g, np.int64).reshape(-1, 3))


def add(codes, off):
    codes = np.asarray(codes, np.uint64)
    return O.morton_add(codes, np.repeat(enc([off]), len(codes)))


def dec(codes):
    return O.morton_decode(np.asarray(codes, np.uint64)) if len(codes) else np.zeros((0, 3), np.int32)


def c_round(v):
    """C's round(): half away from zero, exactly (np.round rounds half to even; floor(v + 0.5) misrounds
    0.49999999999999994)."""
    t = np.trunc(v)
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(v - t) >= 0.5, t + np.sign(v), t)


# ---- restatements of DESIGN.md §3 -----------------------------------------------------------------------------------
def from_points(p, size, origin):
    with np.errstate(invalid="ignore"):
        r = c_round((p.astype(np.float64) - np.asarray(origin, np.float64)) / np.asarray(size, np.float64))
        if (r > 2147483646.0).any() or (r < -2147483647.0).any():
            raise ValueError(OVERFLOW)
    idx = np.where(np.isnan(r), -(2 ** 31), np.nan_to_num(r)).astype(np.int64)
    codes = enc(idx)
    uniq = np.unique(codes)
    return dec(uniq), np.searchsorted(uniq, codes).astype(np.int64)


def check_range(g):
    g = np.asarray(g)
    if g.dtype.kind == "u" or (g > 2 ** 31 - 2).any() or (g < -(2 ** 31) + 1).any():
        raise ValueError(OVERFLOW)


def dilate_once(g):
    check_range(g)
    codes = enc(g)
    cand = np.unique(np.concatenate([add(codes, o) for o in OFF26]))
    new = cand[~np.isin(cand, codes)]
    return np.concatenate([g, dec(new).astype(g.dtype)])


def erode_once(g):
    check_range(g)
    codes = enc(g)
    keep = np.ones(len(g), bool)
    for o in OFF26:
        keep &= np.isin(add(codes, o), codes)
    return g[keep]


def hex_mesh(g, size=(1.0, 1.0, 1.0), origin=(0.0, 0.0, 0.0)):
    check_range(g)
    codes = enc(g)
    corners = np.stack([add(codes, c) for c in CORNERS], 1)
    uniq = np.unique(corners)
    c = dec(uniq).astype(np.float64)
    s, o = np.asarray(size, np.float64), np.asarray(origin, np.float64)
    return (c * s + o) - 0.5 * s, np.searchsorted(uniq, corners).astype(np.int64)


# ---- loop-by-loop transcriptions of the reference's bindings -------------------------------------------------------
M64 = (1 << 64) - 1
SIGNS, XM = 0x7000000000000000, 0x1249249249249249


def _split(x):
    r = x & M64
    for s, m in ((32, 0x1f00000000ffff), (16, 0x1f0000ff0000ff), (8, 0x100f00f00f00f00f), (4, 0x10c30c30c30c30c3),
                 (2, 0x1249249249249249)):
        r = (r | (r << s)) & m
    return r


def code1(x, y, z):
    """MortonCode64(x, y, z) (morton_code.cpp:48-63) of int32 values."""
    v = []
    for c in (x, y, z):
        u = c & 0xffffffff
        q = ((u & 0x80000000) >> 11) | (u & 0x0fffff)
        v.append(_split(q))
    return (v[0] | v[1] << 1 | v[2] << 2) ^ SIGNS


def add1(a, b):
    c1, c2 = a ^ SIGNS, b ^ SIGNS
    out = 0
    for m in (XM, XM << 1, XM << 2):
        out |= ((c1 | (~m & M64)) + (c2 & m)) & m
    return out ^ SIGNS


def safe_cast(x):
    if x > 2 ** 31 - 2 or x < -(2 ** 31) + 1:
        raise ValueError(OVERFLOW)
    return int(x)


def binsearch(needle, hay):
    i = bisect.bisect_left(hay, needle)
    return -1 if i == len(hay) or needle < hay[i] else i


def ref_codes(g):
    return sorted(code1(*(safe_cast(v) for v in row)) for row in g.tolist())


def ref_dilate(g):
    voxel_codes = ref_codes(g)
    offsets = [code1(*o) for o in REF26]
    new = []
    for row in g.tolist():
        vc = code1(*(safe_cast(v) for v in row))
        for off in offsets:
            t = add1(vc, off)
            if binsearch(t, voxel_codes) < 0:
                new.append(t)
    new = sorted(set(new))
    return np.concatenate([g, dec(np.array(new, np.uint64)).astype(g.dtype)])


def ref_erode(g):
    voxel_codes = ref_codes(g)
    offsets = [code1(*o) for o in REF26]
    keep = []
    for i, row in enumerate(g.tolist()):
        vc = code1(*(safe_cast(v) for v in row))
        if all(binsearch(add1(vc, off), voxel_codes) >= 0 for off in offsets):
            keep.append(i)
    return g[keep]


def ref_hex(g, gx, gy, gz, ox, oy, oz):
    offsets = [code1(*c) for c in CORNERS]
    vertex_codes = []
    for row in g.tolist():
        cc = code1(*(safe_cast(v) for v in row))
        vertex_codes += [add1(cc, off) for off in offsets]
    vertex_codes = sorted(set(vertex_codes))
    cubes = np.array([[binsearch(add1(code1(*row), off), vertex_codes) for off in offsets] for row in g.tolist()], np.int64)
    xyz = dec(np.array(vertex_codes, np.uint64)).tolist()
    v = np.array([[float(x) * gx + ox - 0.5 * gx, float(y) * gy + oy - 0.5 * gx, float(z) * gz + oz - 0.5 * gx] for x, y, z in xyz])
    return v, cubes


def ref_from_points(p, gx, gy, gz, ox, oy, oz):
    import math

    def rnd(v):                                              # C round, on a Python float
        if v != v:
            return v
        t = math.trunc(v) if math.isfinite(v) else v
        return t + math.copysign(1.0, v) if math.isfinite(v) and abs(v - t) >= 0.5 else t

    def cast(v):
        if v > 2147483646.0 or v < -2147483647.0:
            raise ValueError(OVERFLOW)
        return -(2 ** 31) if v != v else int(v)

    codes = [code1(cast(rnd((float(a) - ox) / gx)), cast(rnd((float(b) - oy) / gy)), cast(rnd((float(c) - oz) / gz)))
             for a, b, c in p.tolist()]
    uniq = sorted(set(codes))
    return dec(np.array(uniq, np.uint64)), np.array([binsearch(c, uniq) for c in codes], np.int64)


# ---- inputs ---------------------------------------------------------------------------------------------------------
def block(k, origin=(0, 0, 0), dtype=np.int32):
    a = np.arange(k)
    z, y, x = np.meshgrid(a, a, a, indexing="ij")
    return (np.stack([x.ravel(), y.ravel(), z.ravel()], 1) + np.array(origin)).astype(dtype)


def small_grids(count=60, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(count):
        n = int(rng.integers(1, 40))
        g = rng.integers(-4, 4, (n, 3))
        if t % 4 == 1:
            g = np.concatenate([g, g[rng.integers(0, n, 5)]])                         # duplicates
        if t % 4 == 2:
            g = g + rng.choice([2 ** 20 - 2, -(2 ** 20) + 1, 2 ** 21, -(2 ** 21)], (1, 3))  # wrap at +-2^20, alias at 2^21
        if t % 4 == 3:
            g = np.concatenate([g, [[2 ** 31 - 2, 0, 0], [-(2 ** 31) + 1, 5, -7]]])   # int32 extremes
        out.append(g.astype(np.int64 if t % 2 else np.int32))
    out.append(block(4))
    out.append(np.concatenate([block(3), block(3, (1, 1, 1))]))
    return out


def as_set(g):
    return {tuple(r) for r in np.asarray(g).tolist()}


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_transcription_codes_are_the_oracles():
    g = np.concatenate(small_grids(20))
    assert np.array_equal(np.array([code1(*r) for r in g.tolist()], np.uint64), enc(g))
    a, b = enc(g[:50]), enc(g[50:100])
    assert [add1(int(x), int(y)) for x, y in zip(a, b)] == O.morton_add(a, b).tolist()


def test_dilation_against_the_reference_transcription():
    for g in small_grids():
        ours, ref = dilate_once(g), ref_dilate(g)
        n = len(g)
        assert np.array_equal(ours[:n], g) and np.array_equal(ref[:n], g)
        assert ours.dtype == g.dtype
        new, rnew = enc(ours[n:]), enc(ref[n:])
        assert (np.diff(new.astype(np.float64)) >= 0).all() and len(np.unique(new)) == len(new)
        assert set(rnew.tolist()) <= set(new.tolist())                   # a superset of the reference's
        extra = set(new.tolist()) - set(rnew.tolist())
        through = set(np.concatenate([add(enc(g), o) for o in NEVER]).tolist())
        assert extra <= through                                          # only through the three offsets it misses
        if not extra:
            assert np.array_equal(ours, ref)


def test_erosion_against_the_reference_transcription():
    for g in small_grids():
        ours, ref = erode_once(g), ref_erode(g)
        assert as_set(ours) <= as_set(ref)                               # a subset of the reference's
        codes = enc(g)
        lost = [i for i, r in enumerate(g.tolist()) if tuple(r) in as_set(ref) - as_set(ours)]
        for i in lost:                                                   # removed only for one of the three offsets
            assert not all(np.isin(add(codes[[i]], o), codes)[0] for o in NEVER)
        if not lost:
            assert np.array_equal(ours, ref)
    b = block(5)
    assert np.array_equal(erode_once(b), ref_erode(b)) and len(erode_once(b)) == 27


def test_hex_mesh_against_the_reference_transcription():
    rng = np.random.default_rng(3)
    for g in small_grids(40):
        for size, origin in (((1.0,) * 3, (0.0,) * 3), ((0.37,) * 3, (1.5, -2.25, 1e-3)), ((0.1, 0.3, 2.0), (0.2, 0.0, -1.0))):
            v, c = hex_mesh(g, size, origin)
            rv, rc = ref_hex(g, *size, *origin)
            assert np.array_equal(c, rc)
            if size[0] == size[1] == size[2]:
                assert np.array_equal(v, rv)
            else:
                assert np.array_equal(v[:, 0], rv[:, 0])
    g = rng.integers(-50, 50, (200, 3)).astype(np.int32)
    assert np.array_equal(hex_mesh(g, (0.25,) * 3, (3.0, 2.0, 1.0))[0], ref_hex(g, 0.25, 0.25, 0.25, 3.0, 2.0, 1.0)[0])


def test_from_points_against_the_reference_transcription():
    rng = np.random.default_rng(5)
    for t in range(30):
        p = rng.normal(0, 3, (int(rng.integers(1, 300)), 3))
        p = p.astype(np.float32) if t % 2 else p
        size = tuple(rng.uniform(0.05, 2.0, 3)) if t % 3 else (0.5,) * 3
        origin = tuple(rng.normal(0, 1, 3))
        g, idx = from_points(p, size, origin)
        rg, ridx = ref_from_points(p, *size, *origin)
        assert np.array_equal(g, rg) and np.array_equal(idx, ridx)


def test_set_definitions():
    rng = np.random.default_rng(8)
    for t in range(20):
        g = rng.integers(-6, 6, (int(rng.integers(1, 80)), 3)).astype(np.int32)
        s = as_set(g)
        minkowski = {(a + x, b + y, c + z) for a, b, c in s for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)}
        assert as_set(dilate_once(g)) == minkowski
        assert as_set(erode_once(g)) == {v for v in s if all((v[0] + x, v[1] + y, v[2] + z) in s for x, y, z in OFF26)}
        v, cubes = hex_mesh(g, (0.5,) * 3, (1.0, 2.0, 3.0))
        assert len(np.unique(v, axis=0)) == len(v)
        for i, r in enumerate(g.tolist()):
            for k, c in enumerate(CORNERS):
                assert tuple(v[cubes[i, k]]) == tuple((r[a] + c[a]) * 0.5 + (1.0, 2.0, 3.0)[a] - 0.25 for a in range(3))


def test_rounding_and_non_finite_points():
    from decimal import ROUND_HALF_UP, Decimal
    rng = np.random.default_rng(9)
    v = np.concatenate([[2.5, -2.5, 0.49999999999999994, -0.49999999999999994, 0.5, -0.5, 1.5, -1.5, 3.0, 2 ** 52 + 1.0],
                        rng.integers(-20, 20, 200) + 0.5, rng.normal(0, 30, 2000)])
    want = [float(Decimal(x).quantize(Decimal(1), rounding=ROUND_HALF_UP)) for x in v.tolist()]   # half away from zero
    assert c_round(v).tolist() == want
    assert c_round(v)[:4].tolist() == [3.0, -3.0, 0.0, -0.0]
    g = 0.1
    p = np.array([[2.5 * g, -2.5 * g, 0.49999999999999994 * g], [np.nan, 0.0, 1.0]])
    grid, idx = from_points(p, (g,) * 3, (0.0,) * 3)
    q = p[0] / g
    row0 = tuple(int(Decimal(x).quantize(Decimal(1), rounding=ROUND_HALF_UP)) for x in q.tolist())
    assert as_set(grid) == {row0, (-(2 ** 20), 0, 10)}                 # a NaN axis lands at -2^20
    for bad in (np.inf, -np.inf, 3e9):
        with pytest.raises(ValueError, match="overflow"):
            from_points(np.array([[0.0, bad, 0.0]]), (1.0,) * 3, (0.0,) * 3)


def test_argument_errors():
    import pcu_b200 as pcu
    g = block(3)
    p = np.random.default_rng(0).random((10, 3))
    with pytest.raises(ValueError, match="voxel_size must be a scalar or an array/tuple/list of length 3"):
        pcu.sparse_voxel_grid_from_pointcloud(p.astype(np.int32), (1.0, 1.0))     # the wrapper checks first
    with pytest.raises(ValueError, match="voxel_size must have a real numeric type"):
        pcu.sparse_voxel_grid_from_pointcloud(p, 1j)
    with pytest.raises(ValueError, match="origin must be an array/tuple/list of length 3"):
        pcu.sparse_voxel_grid_from_pointcloud(p, 1.0, (0.0, 0.0))
    with pytest.raises(ValueError, match="origin must have a real numeric type"):
        pcu.sparse_voxel_grid_from_pointcloud(p, 1.0, (0.0, 1j, 0.0))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'points'"):
        pcu.sparse_voxel_grid_from_pointcloud(p.astype(np.int32), 1.0)
    with pytest.raises(ValueError, match="Invalid points has zero rows!"):
        pcu.sparse_voxel_grid_from_pointcloud(p[:0], 1.0)
    with pytest.raises(ValueError, match=r"Invalid shape for points must have shape \(N, 3\) but got \(10, 2\)"):
        pcu.sparse_voxel_grid_from_pointcloud(p[:, :2], 1.0)
    for fn in (pcu.dilate_sparse_voxel_grid, pcu.erode_sparse_voxel_grid,
               lambda x: pcu.sparse_voxel_grid_to_hex_mesh(x, 0.5)):
        with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'grid_coordinates'"):
            fn(g.astype(np.float64))
        with pytest.raises(ValueError, match=r"Invalid shape for grid_coordinates must have shape \(N, 3\) but got \(27, 2\)"):
            fn(g[:, :2])
        for dt in (np.uint32, np.uint64):
            with pytest.raises(ValueError) as e:
                fn(g.astype(dt))
            assert str(e.value) == OVERFLOW
    for fn in (pcu.dilate_sparse_voxel_grid, pcu.erode_sparse_voxel_grid):
        with pytest.raises(ValueError, match="Invalid grid_coordinates has zero rows!"):
            fn(g[:0])
        assert fn(g.astype(np.float64), 0) is not None                  # count <= 0: returned unchecked
        x = g.astype(np.uint64)
        assert fn(x, -1) is x
    with pytest.raises(ValueError, match="voxel_size must be a scalar"):
        pcu.sparse_voxel_grid_to_hex_mesh(g.astype(np.float64), (1.0, 1.0))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\)"):
        pcu.sparse_voxel_grid_to_hex_mesh(g[:0].astype(np.float64))
    v, c = pcu.sparse_voxel_grid_to_hex_mesh(g[:0], dtype=np.float32)   # the reference's binding never validates
    assert v.shape == (0, 3) and v.dtype == np.float32 and c.shape == (0, 8) and c.dtype == np.int64


def test_signatures():
    import inspect
    import pcu_b200 as pcu
    for fn, names in ((pcu.sparse_voxel_grid_from_pointcloud, ["points", "voxel_size", "origin", "device"]),
                      (pcu.dilate_sparse_voxel_grid, ["grid_coordinates", "count", "device"]),
                      (pcu.erode_sparse_voxel_grid, ["grid_coordinates", "count", "device"]),
                      (pcu.sparse_voxel_grid_to_hex_mesh, ["grid_coordinates", "voxel_size", "origin", "dtype", "device"])):
        sig = inspect.signature(fn)
        assert list(sig.parameters) == names
        assert sig.parameters["device"].kind == inspect.Parameter.KEYWORD_ONLY
    sig = inspect.signature(pcu.sparse_voxel_grid_to_hex_mesh)
    assert sig.parameters["voxel_size"].default == 1.0 and sig.parameters["dtype"].default is np.float64
    assert inspect.signature(pcu.dilate_sparse_voxel_grid).parameters["count"].default == 1
    assert "sparse_voxel_grid_to_hex_mesh" in pcu.__all__


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _same(got, want):
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(got, want, equal_nan=got.dtype.kind == "f")


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_from_points_equals_restatement(form):
    import pcu_b200 as pcu
    rng = np.random.default_rng(1)
    ties = np.array([[2.5 * 0.1, -2.5 * 0.1, 0.49999999999999994 * 0.1], [np.nan, 0.0, 1.0], [0.0, 0.0, 0.0]])
    for p in (rng.normal(0, 2, (5000, 3)), rng.random((10 ** 5, 3)), ties, rng.random((1, 3))):
        for dt in (np.float32, np.float64):
            for size, origin in ((0.1, (0.0, 0.0, 0.0)), ((0.05, 0.2, 0.3), (0.5, -0.25, 1.0))):
                pp = p.astype(dt)
                g, idx = pcu.sparse_voxel_grid_from_pointcloud(to_form(form, pp), size, origin)
                wg, widx = from_points(pp, np.broadcast_to(size, 3), origin)
                _same(to_numpy(g, form), wg.squeeze())
                _same(to_numpy(idx, form), widx.squeeze())
    for bad in (np.inf, -np.inf, 1e10):
        with pytest.raises(ValueError) as e:
            pcu.sparse_voxel_grid_from_pointcloud(to_form(form, np.array([[0.0, 0.0, 0.0], [0.0, bad, 0.0]])), 1.0)
        assert str(e.value) == OVERFLOW


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_dilate_erode_hex_equal_restatement(form):
    import pcu_b200 as pcu
    grids = small_grids(24, seed=4) + [block(6, (-3, 0, 2)), np.array([[1, 2, 3]], np.int32)]
    for g in grids:
        for dt in (np.int32, np.int64):
            gg = g.astype(dt)
            for count in (0, 1, 3):
                want = gg
                for _ in range(count):
                    want = dilate_once(want)
                _same(to_numpy(pcu.dilate_sparse_voxel_grid(to_form(form, gg), count), form), want if count == 0 else want.squeeze())
            e = erode_once(gg)
            _same(to_numpy(pcu.erode_sparse_voxel_grid(to_form(form, gg)), form), e.squeeze() if len(e) else e)
            for hdt in (np.float32, np.float64, np.float16):
                v, c = pcu.sparse_voxel_grid_to_hex_mesh(to_form(form, gg), (0.3, 0.25, 0.5), (1.0, -2.0, 0.125), hdt)
                wv, wc = hex_mesh(gg, (0.3, 0.25, 0.5), (1.0, -2.0, 0.125))
                _same(to_numpy(v, form), wv.astype(hdt))
                _same(to_numpy(c, form), wc.squeeze())
    b = block(9)
    want = b
    for _ in range(3):
        want = erode_once(want)
    got = pcu.erode_sparse_voxel_grid(to_form(form, b), 3)                 # 9^3 -> 7^3 -> 5^3 -> 3^3
    _same(to_numpy(got, form), want)
    assert len(want) == 27
    one = pcu.erode_sparse_voxel_grid(to_form(form, b), 4)                  # -> the single centre voxel, squeezed
    _same(to_numpy(one, form), np.array([4, 4, 4], np.int32))
    empty = pcu.erode_sparse_voxel_grid(to_form(form, block(2)))
    assert to_numpy(empty, form).shape == (0, 3)
    with pytest.raises(ValueError, match="Invalid grid_coordinates has zero rows!"):
        pcu.erode_sparse_voxel_grid(to_form(form, block(2)), 2)            # a round on the empty result, as in the reference
    with pytest.raises(ValueError, match=r"but got \(3, 1\)"):
        pcu.erode_sparse_voxel_grid(to_form(form, b), 5)                   # the squeezed one-row result, as in the reference


@pytest.mark.gpu
def test_range_check():
    import pcu_b200 as pcu
    for bad in ([2 ** 31 - 1, 0, 0], [0, -(2 ** 31), 0], [0, 0, 2 ** 33]):
        g = np.concatenate([block(3, dtype=np.int64), np.array([bad], np.int64)])
        for fn in (pcu.dilate_sparse_voxel_grid, pcu.erode_sparse_voxel_grid, pcu.sparse_voxel_grid_to_hex_mesh):
            for form in ("numpy", "cuda"):
                with pytest.raises(ValueError) as e:
                    fn(to_form(form, g))
                assert str(e.value) == OVERFLOW


@pytest.mark.gpu
def test_at_scale():
    import torch
    import pcu_b200 as pcu
    rng = np.random.default_rng(2)
    p = rng.normal(0, 1, (10 ** 7, 3)).astype(np.float32)
    g, idx = pcu.sparse_voxel_grid_from_pointcloud(torch.from_numpy(p).cuda(), 0.01)
    wg, widx = from_points(p, (0.01,) * 3, (0.0,) * 3)
    _same(g.cpu().numpy(), wg)
    _same(idx.cpu().numpy(), widx)

    b = torch.from_numpy(block(200, (-100, 3, 7), np.int64)).cuda()
    bn = b.cpu().numpy()
    d = pcu.dilate_sparse_voxel_grid(b)
    big = block(202, (-101, 2, 6), np.int64)                     # the 3 x 3 x 3 Minkowski sum of the block
    ring = big[~((big >= bn.min(0)) & (big <= bn.max(0))).all(1)]
    _same(d.cpu().numpy(), np.concatenate([bn, ring[np.argsort(enc(ring), kind="stable")]]))
    e = pcu.erode_sparse_voxel_grid(b)
    _same(e.cpu().numpy(), bn[((bn > bn.min(0)) & (bn < bn.max(0))).all(1)])
    assert len(e) == 198 ** 3

    shell = _sphere_points(4 * 10 ** 6, 1.0, rng)
    sg, _ = pcu.sparse_voxel_grid_from_pointcloud(shell, 0.0018)
    assert len(sg) > 10 ** 6
    v, c = pcu.sparse_voxel_grid_to_hex_mesh(torch.from_numpy(sg).cuda(), 0.0018)
    wv, wc = hex_mesh(sg, (0.0018,) * 3)
    _same(v.cpu().numpy(), wv)
    _same(c.cpu().numpy(), wc)


def _sphere_points(n, r, rng):
    d = rng.normal(0, 1, (n, 3))
    return r * d / np.linalg.norm(d, axis=1, keepdims=True)


@pytest.mark.gpu
def test_pipeline_points_to_surface():
    import pcu_b200 as pcu
    rng = np.random.default_rng(6)
    r, s = 1.0, 0.02
    centre = np.array([0.013, -0.021, 0.007])
    p = _sphere_points(400000, r, rng) + centre
    g, _ = pcu.sparse_voxel_grid_from_pointcloud(p, s)
    band = pcu.dilate_sparse_voxel_grid(g, 2)
    v, cubes = pcu.sparse_voxel_grid_to_hex_mesh(band, s)
    sdf = np.linalg.norm(v - centre, axis=1) - r                   # the sphere's exact signed distance
    mv, mf = pcu.marching_cubes_sparse_voxel_grid(sdf, v, cubes, 0.0)
    dist = np.abs(np.linalg.norm(mv - centre, axis=1) - r)
    assert dist.max() <= s * (1 + 1e-9)                            # within one voxel edge of the sphere
    e = np.sort(np.concatenate([mf[:, [0, 1]], mf[:, [1, 2]], mf[:, [2, 0]]]), axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    assert (counts == 2).all()                                     # closed: the hex mesh welds shared corners
