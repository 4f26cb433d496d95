"""remove_mesh_vertices and remove_unreferenced_mesh_vertices: the results of DESIGN.md §3 restated with np.flatnonzero
and fancy indexing, pinned to literal transcriptions of the reference's mask loop (src/remove_mesh_vertices.cpp:41-66)
and of libigl's remove_unreferenced (mark, number, remap) on many small random inputs; the argument errors in the
reference's order; on the GPU, both functions bit for bit (dtype, shape, values) against the restatements over every
dtype and input form, the squeezed shapes, all-false and all-true masks, the unsigned -1 of corr_f and a
1.3 * 10^6-face icosphere."""
import numpy as np
import pytest

from meshes import icosphere, to_form

IDX = [np.int32, np.int64, np.uint32, np.uint64]


# ---- the restatements -----------------------------------------------------------------------------------------------
def restate_mask(v, f, mask):
    """(v_out, f_out), squeezed: the kept vertices, and the faces whose corners are all kept, re-indexed."""
    mask = np.asarray(mask).reshape(-1)
    keep = np.flatnonzero(mask)
    remap = np.full(len(v), -1, np.int64)
    remap[keep] = np.arange(len(keep))
    fk = f[mask[f].all(axis=1)]
    return np.squeeze(v[keep]), np.squeeze(remap[fk].astype(f.dtype).reshape(-1, 3))


def restate_unref(v, f):
    """(v_out, f_out, J, I), squeezed: J the referenced vertices ascending, I[J] = arange, -1 elsewhere, f_out = I[f]."""
    used = np.zeros(len(v), bool)
    used[f.ravel()] = True
    J = np.flatnonzero(used)
    I = np.full(len(v), -1, np.int64)
    I[J] = np.arange(len(J))
    return tuple(np.squeeze(x) for x in (v[J], I[f].astype(f.dtype), J.astype(f.dtype), I.astype(f.dtype)))


def literal_mask(v, f, mask):
    """src/remove_mesh_vertices.cpp:37-70 line by line."""
    v_out = np.zeros_like(v)
    f_out = np.zeros((f.shape[0], v.shape[1]), f.dtype)
    u2m = np.zeros(len(v), np.int32)
    nv = 0
    for i in range(mask.size):
        if mask.reshape(-1)[i]:
            u2m[i] = nv
            v_out[u2m[i]] = v[i]
            nv += 1
        else:
            u2m[i] = -1
    nf = 0
    for i in range(f.shape[0]):
        keep = True
        for j in range(f.shape[1]):
            if u2m[f[i, j]] == -1:
                keep = False
                break
        if keep:
            for j in range(f.shape[1]):
                f_out[nf, j] = u2m[f[i, j]]
            nf += 1
    return np.squeeze(v_out[:nv]), np.squeeze(f_out[:nf])


def literal_unref(v, f):
    """igl::remove_unreferenced(V, F, NV, NF, I, J) line by line (mark, count, number, remap), returned as the
    reference's binding returns it: (NV, NF, J, I)."""
    n = v.shape[0]
    mark = np.zeros(n, np.int64)
    for i in range(f.shape[0]):
        for j in range(f.shape[1]):
            mark[f[i, j]] = 1
    newsize = int(mark.sum())
    I = np.zeros(n, np.int64)
    J = np.zeros(newsize, np.int64)
    count = 0
    for i in range(n):
        if mark[i] == 1:
            I[i] = count
            J[count] = i
            count += 1
        else:
            I[i] = -1
    NF = f.astype(np.int64).copy()
    for i in range(f.shape[0]):
        for j in range(f.shape[1]):
            NF[i, j] = I[f[i, j]]
    NV = np.zeros((newsize, v.shape[1]), v.dtype)
    for i in range(newsize):
        NV[i] = v[J[i]]
    return tuple(np.squeeze(x) for x in (NV, NF.astype(f.dtype), J.astype(f.dtype), I.astype(f.dtype)))


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def all_same(got, want):
    return len(got) == len(want) and all(same(g if isinstance(g, np.ndarray) else g.cpu().numpy(), w) for g, w in zip(got, want))


def random_mesh(rng, nv, m, vdt, idt, hi=None):
    v = rng.standard_normal((nv, 3)).astype(vdt)
    f = rng.integers(0, nv if hi is None else hi, (m, 3))
    if m > 2:
        f[1] = f[0, 0]                                      # repeated corners
    return v, f.astype(idt)


# ---- the restatements against the literal loops (CPU) ----------------------------------------------------------------
@pytest.mark.parametrize("idt", [np.int32, np.int64])
def test_mask_restatement_equals_literal_loop(idt):
    rng = np.random.default_rng(7)
    for trial in range(80):
        nv = int(rng.integers(1, 15))
        v, f = random_mesh(rng, nv, int(rng.integers(1, 12)), np.float64, idt)
        mask = rng.random(nv) < (0.2, 0.5, 0.9, 1.0, 0.0)[trial % 5]
        if trial % 3 == 0:
            mask = mask[:, None]
        assert all_same(restate_mask(v, f, mask), literal_mask(v, f, mask)), (v, f, mask)


@pytest.mark.parametrize("idt", IDX)
def test_unreferenced_restatement_equals_literal_loop(idt):
    rng = np.random.default_rng(8)
    for trial in range(80):
        nv = int(rng.integers(1, 20))
        hi = max(1, nv // (1 + trial % 3))                    # gaps: the last vertices are often unreferenced
        v, f = random_mesh(rng, nv, int(rng.integers(1, 8)), np.float32, idt, hi)
        assert all_same(restate_unref(v, f), literal_unref(v, f)), (v, f)
    v = np.arange(12.0).reshape(4, 3)
    got = restate_unref(v, np.array([[3, 1, 3]], np.uint32))
    assert got[3].dtype == np.uint32 and list(got[3]) == [2 ** 32 - 1, 0, 2 ** 32 - 1, 1] and list(got[2]) == [1, 3]


# ---- argument errors (CPU: raised before any device call) -------------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    v = np.random.default_rng(0).random((6, 3))
    f = np.array([[0, 1, 2], [3, 4, 5]])
    m = np.ones(6, bool)
    rmv = pcu.remove_mesh_vertices
    cases = [
        ((v.astype(np.int32), f, m), "Invalid scalar type (int32) for argument 'v'"),
        ((v, f.astype(np.uint32), m), "Invalid scalar type (uint32) for argument 'f'"),
        ((v, f, m.astype(np.uint8)), "Invalid scalar type (uint8) for argument 'mask'"),
        ((v[:0], f, m), "Invalid input mesh with zero elements"),
        ((v, f[:0], m), "Invalid input mesh with zero elements"),
        ((v[:, :2], f, m), "Only 3D inputs are supported"),
        ((v, f[:, :2], m), "Only 3D inputs are supported"),
        ((v, f, m[:5]), "mask should have the same number of rows as v"),
        ((v, f, np.ones((6, 2), bool)), "mask should have only one column"),
        ((v, f, np.ones((5, 2), bool)), "mask should have the same number of rows as v"),   # rows first
        ((v[:0], f, m[:3]), "Invalid input mesh with zero elements"),                      # validate_mesh first
        ((v, f.astype(np.float32), m.astype(np.uint8)), "for argument 'f'"),               # dtypes in argument order
        ((list(v), f, m), "Invalid type for v"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            rmv(*args)
        assert msg in str(e.value), (msg, str(e.value))
    rur = pcu.remove_unreferenced_mesh_vertices
    cases = [
        ((v.astype(np.int32), f), "Invalid scalar type (int32) for argument 'v'"),
        ((v, f.astype(np.float64)), "Invalid scalar type (float64) for argument 'f'"),
        ((v[:0], f), "Invalid input mesh with zero elements"),
        ((v, f[:, :2]), "Only 3D inputs are supported"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            rur(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        rmv(v, f, m, None)                                   # device= is keyword only
    with pytest.raises(TypeError):
        rur(v, f, None)


# ---- the GPU --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", [np.int32, np.int64])
def test_mask_every_dtype(pcu, vdt, idt):
    rng = np.random.default_rng(21)
    for nv, m, p in ((300, 500, 0.7), (5000, 9000, 0.95), (40, 30, 0.3)):
        v, f = random_mesh(rng, nv, m, vdt, idt)
        mask = rng.random(nv) < p
        assert all_same(pcu.remove_mesh_vertices(v, f, mask), restate_mask(v, f, mask))
        assert all_same(pcu.remove_mesh_vertices(v, f, mask[:, None]), restate_mask(v, f, mask))


@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", IDX)
def test_unreferenced_every_dtype(pcu, vdt, idt):
    rng = np.random.default_rng(22)
    for nv, m, hi in ((300, 200, 250), (5000, 900, 5000), (40, 3, 40)):
        v, f = random_mesh(rng, nv, m, vdt, idt, hi)
        got = pcu.remove_unreferenced_mesh_vertices(v, f)
        assert all_same(got, restate_unref(v, f))
        if idt in (np.uint32, np.uint64):
            assert (got[3] == np.iinfo(idt).max).any()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms(pcu, form):
    import torch
    rng = np.random.default_rng(23)
    v, f = random_mesh(rng, 400, 600, np.float32, np.int64)
    mask = rng.random(400) < 0.8
    got = pcu.remove_mesh_vertices(to_form(form, v), to_form(form, f), to_form(form, mask))
    kinds = {"numpy": np.ndarray, "cuda": torch.Tensor, "cpu": torch.Tensor}
    assert all(isinstance(g, kinds[form]) and (form == "numpy" or g.is_cuda == (form == "cuda")) for g in got)
    assert all_same(got, restate_mask(v, f, mask))
    for idt in (np.int32, np.uint32, np.uint64):
        fu = f.astype(idt)
        got = pcu.remove_unreferenced_mesh_vertices(to_form(form, v), to_form(form, fu))
        assert all(isinstance(g, kinds[form]) for g in got)
        assert all_same(got, restate_unref(v, fu))


@pytest.mark.gpu
def test_shapes_and_edge_masks(pcu):
    v = np.arange(15.0).reshape(5, 3)
    f = np.array([[0, 1, 2], [2, 3, 4]], np.int32)
    v2, f2 = pcu.remove_mesh_vertices(v, f, np.zeros(5, bool))                 # all false
    assert v2.shape == (0, 3) and f2.shape == (0, 3) and f2.dtype == np.int32
    got = pcu.remove_mesh_vertices(v, f, np.ones(5, bool))                     # all true
    assert all_same(got, (v, f))
    v2, f2 = pcu.remove_mesh_vertices(v, f, np.array([0, 0, 1, 0, 0], bool))  # one vertex: a (3,) row, no faces
    assert v2.shape == (3,) and np.array_equal(v2, v[2]) and f2.shape == (0, 3)
    v2, f2 = pcu.remove_mesh_vertices(v, f, np.array([1, 1, 1, 0, 1], bool))  # one face: (3,)
    assert f2.shape == (3,) and list(f2) == [0, 1, 2]
    got = pcu.remove_unreferenced_mesh_vertices(v, np.array([[3, 3, 3]], np.uint64))   # one referenced vertex
    assert all_same(got, restate_unref(v, np.array([[3, 3, 3]], np.uint64)))
    assert got[0].shape == (3,) and got[1].shape == (3,) and got[2].shape == () and got[3].shape == (5,)
    assert list(got[3]) == [2 ** 64 - 1] * 3 + [0, 2 ** 64 - 1]
    got = pcu.remove_unreferenced_mesh_vertices(v[:1], np.array([[0, 0, 0]], np.int64))  # one vertex: 0-d I
    assert got[3].shape == () and int(got[3]) == 0


@pytest.mark.gpu
def test_corner_errors(pcu):
    v = np.zeros((5, 3))
    for f in (np.array([[0, 1, 5], [0, 1, 2], [-1, 0, 0]], np.int64), np.array([[0, 1, 7], [0, 1, -1]], np.int32)):
        with pytest.raises(ValueError, match="Invalid face indices: 2 faces have a corner outside"):
            pcu.remove_mesh_vertices(v, f, np.ones(5, bool))
        with pytest.raises(ValueError, match="Invalid face indices: 2 faces have a corner outside"):
            pcu.remove_unreferenced_mesh_vertices(v, f)
    with pytest.raises(ValueError, match="Invalid face indices: 1 faces"):
        pcu.remove_unreferenced_mesh_vertices(v, np.array([[0, 1, 2 ** 32 - 1]], np.uint32))


@pytest.mark.gpu
def test_large_icosphere(pcu):
    v, f = icosphere(8)
    rng = np.random.default_rng(24)
    mask = v[:, 2] > -0.3
    assert all_same(pcu.remove_mesh_vertices(v, f, mask), restate_mask(v, f, mask))
    fh = f[rng.random(len(f)) < 0.5].astype(np.int32)
    got = pcu.remove_unreferenced_mesh_vertices(v.astype(np.float32), fh)
    assert all_same(got, restate_unref(v.astype(np.float32), fh))
    again = pcu.remove_unreferenced_mesh_vertices(v.astype(np.float32), fh)
    assert all_same(again, got)
