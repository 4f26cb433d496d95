"""sparse_voxel_grid_boundary: the reference's algorithm (src/sparse_voxel_grid.cpp:463-522) restated with numpy --
its Morton codes checked against the oracle's (the reference's own MortonCode64 where oracle/_ref was built) -- and
against a set-based neighbour test; argument errors; on the GPU, the function against the restatement in every form."""
import numpy as np
import pytest

from meshes import to_form, to_numpy
from oracle import oracle as O

X = np.uint64(0x1249249249249249)
SIGNS = np.uint64(0x7000000000000000)
OVERFLOW = "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small."


def _split21(x):
    r = x.astype(np.int64).astype(np.uint64)               # sign-extended, as `uint64_t r = x` does
    for s, m in ((32, 0x1f00000000ffff), (16, 0x1f0000ff0000ff), (8, 0x100f00f00f00f00f), (4, 0x10c30c30c30c30c3),
                 (2, 0x1249249249249249)):
        r = (r | (r << np.uint64(s))) & np.uint64(m)
    return r


def encode(p):
    """MortonCode64(x, y, z) of int32 coordinates."""
    p = p.astype(np.int32).view(np.uint32)
    q = ((p & np.uint32(0x80000000)) >> np.uint32(11)) | (p & np.uint32(0x0fffff))
    q = q.view(np.int32)
    return (_split21(q[:, 0]) | (_split21(q[:, 1]) << np.uint64(1)) | (_split21(q[:, 2]) << np.uint64(2))) ^ SIGNS


def add(a, b):
    c1, c2 = a ^ SIGNS, b ^ SIGNS
    out = np.zeros_like(a)
    for m in (X, X << np.uint64(1), X << np.uint64(2)):
        out |= ((c1 | ~m) + (c2 & m)) & m
    return out ^ SIGNS


OFFSETS = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.int32)


def restate(g):
    """The boundary rows (int64, ascending) of int32 / int64 voxels whose coordinates passed the range check."""
    codes = encode(g)
    srt = np.sort(codes)
    boundary = np.zeros(len(g), bool)
    with np.errstate(over="ignore"):
        for off in encode(OFFSETS):
            q = add(codes, np.full_like(codes, off))
            pos = np.searchsorted(srt, q)
            found = (pos < len(srt)) & (srt[np.minimum(pos, len(srt) - 1)] == q)
            boundary |= ~found
    return np.nonzero(boundary)[0].astype(np.int64)


def brute(g):
    s = {tuple(r) for r in g.tolist()}
    return np.array([i for i, r in enumerate(g.tolist())
                     if any((r[0] + o[0], r[1] + o[1], r[2] + o[2]) not in s for o in OFFSETS.tolist())], np.int64)


def block(k, origin=(0, 0, 0), dtype=np.int32):
    a = np.arange(k)
    z, y, x = np.meshgrid(a, a, a, indexing="ij")
    return (np.stack([x.ravel(), y.ravel(), z.ravel()], 1) + np.array(origin)).astype(dtype)


def cases():
    rng = np.random.default_rng(0)
    two_blocks = np.concatenate([block(5), block(4, (7, -3, 2))])
    dup = np.concatenate([block(3), block(3)[[0, 4, 13, 13]]])
    alias = np.array([[2 ** 20 - 1, 0, 0], [-(2 ** 20), 0, 0], [0, 2 ** 20 - 1, 5], [0, -(2 ** 20), 5],
                      [2 ** 21, 3, 3], [0, 3, 3], [2 ** 21 + 1, 3, 3]], np.int32)     # +-2^20 wraps; 2^21 aliases 0
    rnd = rng.integers(-40, 40, (3000, 3)).astype(np.int64)
    big = np.array([[2 ** 31 - 2, -(2 ** 31) + 1, 0], [2 ** 31 - 3, -(2 ** 31) + 1, 0]], np.int64)
    return {"two blocks": two_blocks, "duplicates": dup, "aliasing": alias, "random": rnd, "int32 extremes": big}


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_codes_are_the_oracles():
    for name, g in cases().items():
        codes = encode(g)
        assert np.array_equal(codes, O.morton_encode(g.astype(np.int32))), name
        for off in OFFSETS:
            want = O.morton_add(codes, np.repeat(O.morton_encode(off[None, :]), len(codes)))
            with np.errstate(over="ignore"):
                assert np.array_equal(add(codes, np.full_like(codes, encode(off[None, :])[0])), want), name


def test_restatement_against_neighbour_sets():
    for name in ("two blocks", "duplicates", "random"):
        g = cases()[name]
        assert np.array_equal(restate(g), brute(g)), name
    b = block(6)
    inner = ((b > 0) & (b < 5)).all(1)
    assert np.array_equal(restate(b), np.nonzero(~inner)[0])     # a dense block's interior is not boundary
    alias = cases()["aliasing"]
    assert encode(alias[[4]])[0] == encode(alias[[5]])[0]          # 2^21 aliases 0
    with np.errstate(over="ignore"):                              # 2^20 - 1, plus one, wraps to -2^20
        assert add(encode(alias[[0]]), encode(OFFSETS[[0]]))[0] == encode(alias[[1]])[0]


def test_argument_errors():
    import pcu_b200 as pcu
    g = block(3)
    for dt in (np.uint32, np.uint64):
        with pytest.raises(ValueError) as e:
            pcu.sparse_voxel_grid_boundary(g.astype(dt))
        assert str(e.value) == OVERFLOW
    with pytest.raises(ValueError, match="Invalid grid_coordinates has zero rows!"):
        pcu.sparse_voxel_grid_boundary(g[:0])
    with pytest.raises(ValueError, match=r"Invalid shape for grid_coordinates must have shape \(N, 3\) but got \(27, 2\)"):
        pcu.sparse_voxel_grid_boundary(g[:, :2])
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'grid_coordinates'"):
        pcu.sparse_voxel_grid_boundary(g.astype(np.float64))


# ---- GPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_equals_restatement(form):
    import pcu_b200 as pcu
    rng = np.random.default_rng(11)
    sets = dict(cases())
    sets["random 10^6"] = rng.integers(-60, 60, (10 ** 6, 3)).astype(np.int32)
    sets["block 200^3"] = block(200, (-100, 3, 7), np.int64)
    for name, g in sets.items():
        for dt in (np.int32, np.int64):
            gg = g.astype(dt)
            got = pcu.sparse_voxel_grid_boundary(to_form(form, gg))
            if form != "numpy":
                assert got.is_cuda == (form == "cuda")
            assert to_numpy(got).dtype == np.int64
            assert np.array_equal(to_numpy(got), restate(gg)), (name, dt)


@pytest.mark.gpu
def test_range_check_and_shapes():
    import pcu_b200 as pcu
    for bad in ([2 ** 31 - 1, 0, 0], [0, -(2 ** 31), 0], [0, 0, 2 ** 33]):
        g = np.concatenate([block(3, dtype=np.int64), np.array([bad], np.int64)])
        for form in ("numpy", "cuda"):
            with pytest.raises(ValueError) as e:
                pcu.sparse_voxel_grid_boundary(to_form(form, g))
            assert str(e.value) == OVERFLOW
        if bad[2] != 2 ** 33:
            with pytest.raises(ValueError, match="overflow"):
                pcu.sparse_voxel_grid_boundary(g.astype(np.int32))
    one = pcu.sparse_voxel_grid_boundary(np.array([[1, 2, 3]], np.int32))
    assert one.shape == () and int(one) == 0                      # (1, 1) squeezed
    assert pcu.sparse_voxel_grid_boundary(block(3)).shape == (26,)
