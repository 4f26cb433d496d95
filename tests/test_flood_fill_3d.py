"""flood_fill_3d: the result of DESIGN.md §3 restated with scipy's connected components over the reference's
linear-offset graph, pinned to a literal restatement of the reference's queue loop at small sizes; the argument errors;
on the GPU, the function bit for bit against the restatement over every dtype and input form, a serpentine of depth
about 10^6, a grid of 2^27 voxels, the wraps, a NaN seed and a fill equal to the seed's value."""
from collections import deque

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

from meshes import to_form, to_numpy

DTYPES = [np.int32, np.int64, np.float32, np.float64]


# ---- the restatement -----------------------------------------------------------------------------------------------
def cast_fill(fill, dtype):
    """(T)(double)fill as the reference's x86 build converts it: cvttsd2si for the integers (NaN and out-of-range
    truncations give INT_MIN), round to nearest for float32."""
    fill = float(fill)
    if dtype == np.int32:
        return np.int32(int(fill)) if -2147483649.0 < fill < 2147483648.0 else np.int32(-2 ** 31)
    if dtype == np.int64:
        return np.int64(int(fill)) if -2.0 ** 63 <= fill < 2.0 ** 63 else np.int64(-2 ** 63)
    with np.errstate(over="ignore"):
        return np.array(fill).astype(dtype)[()]


def restate(grid, seed, fill):
    """The seed's component among the voxels equal to its value, in the graph where linear index o is adjacent to
    o + 1, o + d and o + h d when those are in range; the component gets the converted fill."""
    grid = np.ascontiguousarray(grid)
    w, h, d = grid.shape
    flat = grid.ravel()
    n = flat.size
    o = (seed[0] * h + seed[1]) * d + seed[2]
    sv = flat[o]
    fv = cast_fill(fill, grid.dtype.type)
    out = flat.copy()
    eq = flat == sv
    if not eq[o] or fv == sv:
        return out.reshape(grid.shape)
    rows, cols = [], []
    for step in (1, d, h * d):
        a = np.arange(n - step)
        keep = eq[a] & eq[a + step]
        rows.append(a[keep])
        cols.append(a[keep] + step)
    r, c = np.concatenate(rows), np.concatenate(cols)
    g = scipy.sparse.coo_matrix((np.ones(len(r), np.int8), (r, c)), shape=(n, n))
    _, lab = scipy.sparse.csgraph.connected_components(g, directed=False)
    out[eq & (lab == lab[o])] = fv
    return out.reshape(grid.shape)


def literal_bfs(grid, seed, fill):
    """The reference's loop (src/flood_fill_3d.cpp:11-51) line by line; needs fill != the seed's value."""
    g = np.ascontiguousarray(grid).ravel().copy()
    w, h, d = grid.shape
    fv = cast_fill(fill, grid.dtype.type)
    start = seed[0] * h * d + seed[1] * d + seed[2]
    sv = g[start]
    q = deque([start])
    while q:
        off = q.popleft()
        x = off // (h * d)
        y = (off - x * h * d) // d
        z = off - x * h * d - y * d
        if 0 <= off < g.size and g[off] == sv:
            g[off] = fv
            for dx, dy, dz in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
                q.append((x + dx) * h * d + (y + dy) * d + (z + dz))
    return g.reshape(grid.shape)


def same(a, b):
    """Bit for bit (NaN payloads included: both sides copy or write the same values)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def random_grid(rng, shape, dtype, levels=2):
    g = rng.integers(0, levels, shape)
    return g.astype(dtype)


def serpentine(X, Y, Z):
    """A one-voxel corridor through a (2X+1) x (2Y+1) x (2Z+1) grid of walls, visiting X Y Z cells in boustrophedon
    order: a path of depth about 2 X Y Z from one end to the other."""
    g = np.ones((2 * X + 1, 2 * Y + 1, 2 * Z + 1), np.int32)
    xs, ys, zs = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
    ys = np.where(xs % 2 == 1, Y - 1 - ys, ys)
    row = xs * Y + np.arange(Y)[None, :, None]
    zs = np.where(row % 2 == 1, Z - 1 - zs, zs)
    cells = np.stack([xs, ys, zs], -1).reshape(-1, 3) * 2 + 1
    g[tuple(cells.T)] = 0
    mid = (cells[1:] + cells[:-1]) // 2
    g[tuple(mid.T)] = 0
    return g, tuple(cells[0]), tuple(cells[-1])


# ---- the restatement against the literal loop (CPU) -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_restatement_equals_literal_loop(dtype):
    rng = np.random.default_rng(1)
    for shape in [(5, 4, 3), (3, 7, 2), (1, 1, 9), (6, 1, 1), (4, 5, 6)]:
        for trial in range(6):
            g = random_grid(rng, shape, dtype, levels=2 + trial % 2)
            seed = tuple(int(rng.integers(0, s)) for s in shape)
            fill = 7.9 if trial % 2 else -3.5
            assert same(restate(g, seed, fill), literal_bfs(g, seed, fill))


def test_wraps():
    """A region touching z = d - 1 continues at z = 0 of the next row, and one touching y = h - 1 at y = 0 of the next
    slab, as in the reference."""
    g = np.ones((3, 3, 4), np.int32)
    g[0, 0, 3] = 0                                         # z wrap: (0, 0, 3) -> (0, 1, 0)
    g[0, 1, 0] = 0
    g[0, 2, 2] = 0                                         # y wrap: (0, 2, 2) -> (1, 0, 2)
    g[1, 0, 2] = 0
    for seed in [(0, 0, 3), (0, 2, 2)]:
        want = literal_bfs(g, seed, 5)
        assert same(restate(g, seed, 5), want)
        assert (want == 5).sum() == 2
    assert same(restate(g, (0, 0, 3), 5), literal_bfs(g, (0, 0, 3), 5))


def test_nan_seed_and_signed_zero():
    g = np.array([[[0.0, -0.0, np.nan], [np.nan, 0.0, 1.0]]], np.float64)
    assert same(restate(g, (0, 0, 2), 3.0), literal_bfs(g, (0, 0, 2), 3.0))   # NaN seed: nothing
    assert same(restate(g, (0, 0, 2), 3.0), g)
    out = restate(g, (0, 0, 0), 3.0)                                           # -0.0 matches 0.0
    assert same(out, literal_bfs(g, (0, 0, 0), 3.0))
    assert out[0, 0, 1] == 3.0 and out[0, 1, 1] == 3.0
    assert same(restate(g, (0, 0, 0), -0.0), g)            # fill == seed (IEEE): an unchanged copy


def test_integer_fills():
    for fill, want32, want64 in [(7.9, 7, 7), (-7.9, -7, -7), (2.0 ** 31, -2 ** 31, 2 ** 31), (-2.0 ** 31 - 0.5, -2 ** 31, -2 ** 31),
                                 (2147483647.9, 2147483647, 2147483647), (float("nan"), -2 ** 31, -2 ** 63),
                                 (1e19, -2 ** 31, -2 ** 63), (-1e300, -2 ** 31, -2 ** 63), (float("inf"), -2 ** 31, -2 ** 63)]:
        assert cast_fill(fill, np.int32) == want32 and cast_fill(fill, np.int64) == want64, fill
        g = np.zeros((2, 2, 2), np.int32)
        assert same(restate(g, (0, 0, 0), fill), literal_bfs(g, (0, 0, 0), fill))
    assert cast_fill(1e40, np.float32) == np.float32(np.inf)
    assert cast_fill(0.1, np.float32) == np.float32(0.1)


# ---- argument errors (CPU: raised before any device call) -----------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    g = np.zeros((3, 4, 5), np.int32)
    ff = pcu.flood_fill_3d
    cases = [
        ((g, (0, 0), 1), "expected 3D coordinate"),
        ((g, 0, 1), "expected 3D coordinate"),
        ((g[0], (0, 0, 0), 1), "grid must have shape [w, h, d]"),
        ((g[0], (0, 0), 1), "expected 3D coordinate"),   # the reference's order: the seed is converted first
        ((g.astype(np.uint8), (0, 0, 0), 1), "Invalid scalar type (uint8) for argument 'grid'. Expected one of "
                                             "['int32', 'int64', 'float32', 'float64']."),
        ((g, (3, 0, 0), 1), "seed point must be inside grid"),
        ((g, (0, -1, 0), 1), "seed point must be inside grid"),
        ((g, (0, 0, 5), 1), "seed point must be inside grid"),
        ((g.astype(np.uint8), (3, 0, 0), 1), "Invalid scalar type (uint8)"),
        ((np.zeros((0, 4, 5), np.float32), (0, 0, 0), 1), "seed point must be inside grid"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            ff(*args)
        assert msg in str(e.value), (msg, str(e.value))
    big = np.lib.stride_tricks.as_strided(np.zeros(1, np.int32), (2048, 1024, 1024), (0, 0, 0))
    with pytest.raises(ValueError, match="at most 2\\^31 - 1 voxels"):
        ff(big, (0, 0, 0), 1)
    with pytest.raises(TypeError):
        ff(g, (0, 0, 0), 1, None)                          # device= is keyword only


# ---- the GPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_equals_restatement(pcu, dtype, form):
    import torch
    rng = np.random.default_rng(2)
    for shape in [(37, 29, 41), (1, 1, 50), (70, 3, 1), (64, 64, 64), (5, 300, 7)]:
        g = random_grid(rng, shape, dtype, levels=2)
        seed = tuple(int(rng.integers(0, s)) for s in shape)
        got = pcu.flood_fill_3d(to_form(form, g), seed, -2.5)
        if form == "cuda":
            assert isinstance(got, torch.Tensor) and got.is_cuda
        assert same(to_numpy(got), restate(g, seed, -2.5)), shape


@pytest.mark.gpu
def test_wraps_nan_and_fill_equal_to_seed(pcu):
    rng = np.random.default_rng(6)
    g = np.ones((20, 9, 13), np.float32)
    g[:, :, 12] = 0                                        # every z = d - 1 voxel: connected only through the z wrap
    g[:, 8, :] = 0                                         # and the y = h - 1 rows, through the y wrap
    g[3, 4, 5] = 0                                         # isolated
    for seed in [(0, 0, 12), (7, 8, 3), (3, 4, 5)]:
        assert same(pcu.flood_fill_3d(g, seed, 2.0), restate(g, seed, 2.0))
    h = rng.integers(0, 2, (30, 31, 32)).astype(np.float64)
    h[rng.random(h.shape) < 0.1] = np.nan
    h[rng.random(h.shape) < 0.2] = -0.0
    nan_seed = tuple(int(i[0]) for i in np.nonzero(np.isnan(h)))
    assert same(pcu.flood_fill_3d(h, nan_seed, 5.0), h)
    zero_seed = tuple(int(i[0]) for i in np.nonzero(h == 0))
    assert same(pcu.flood_fill_3d(h, zero_seed, 5.0), restate(h, zero_seed, 5.0))
    assert same(pcu.flood_fill_3d(h, zero_seed, -0.0), h)  # fill == seed value: an unchanged copy
    i32 = rng.integers(-3, 3, (40, 40, 40)).astype(np.int32)
    for fill in (2.0 ** 31, float("nan"), -7.9):
        seed = (1, 2, 3)
        assert same(pcu.flood_fill_3d(i32, seed, fill), restate(i32, seed, fill))
    sv = int(i32[1, 2, 3])
    assert same(pcu.flood_fill_3d(i32, (1, 2, 3), sv + (0.5 if sv >= 0 else -0.5)), i32)   # truncates to the seed's value


@pytest.mark.gpu
def test_serpentine(pcu):
    g, a, b = serpentine(80, 80, 80)                       # a corridor of about 10^6 voxels, 161^3 grid
    out = pcu.flood_fill_3d(g, a, 7)
    assert out[b] == 7 and (out == 7).sum() == (g == 0).sum()
    assert same(out, restate(g, a, 7))


@pytest.mark.gpu
def test_large_grid(pcu):
    """2^27 voxels; the y and z faces are walls, so the wraps connect nothing and scipy.ndimage.label restates it."""
    import scipy.ndimage
    import torch
    rng = np.random.default_rng(12)
    g = (rng.random((512, 512, 512)) < 0.6).astype(np.int32)   # above the percolation threshold: one giant component
    g[:, 0, :] = g[:, -1, :] = 2
    g[:, :, 0] = g[:, :, -1] = 2
    seed = tuple(int(i[0]) for i in np.nonzero(g[:, 1:-1, 1:-1] == 1))
    seed = (seed[0], seed[1] + 1, seed[2] + 1)
    out = pcu.flood_fill_3d(torch.from_numpy(g).cuda(), seed, 9).cpu().numpy()
    lab, _ = scipy.ndimage.label(g == 1)
    want = g.copy()
    want[lab == lab[seed]] = 9
    assert same(out, want)
