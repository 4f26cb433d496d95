"""connected_components: the result of DESIGN.md §3 restated with scipy's connected components over the consecutive
corner pairs, relabelled by each component's smallest vertex, and pinned to a literal transcription of the reference's
BFS over libigl's all-pairs adjacency on many small random inputs; the argument errors; on the GPU, the function bit for
bit (dtype, shape, values) against the restatement over every dtype and input form, the squeezed shapes, a permuted
icosphere of 1.3 * 10^6 faces, 10^6 disjoint triangles, a numbered strip of 10^6 faces, a marching-cubes mesh with
thousands of components, the reference's own test and the keep-the-largest-component pipeline."""
from collections import deque

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

from meshes import icosphere, to_form, to_numpy

IDX = [np.int32, np.int64, np.uint32, np.uint64]


# ---- the restatement ------------------------------------------------------------------------------------------------
def _rows(f):
    f = np.asarray(f)
    return f.reshape(len(f), -1).astype(np.int64)


def restate(f):
    """(cv, nv, cf, nf) in f's dtype, squeezed: components of [0, max(f) + 1) under the edges f[i, j] -- f[i, j + 1],
    numbered in ascending order of their smallest vertex; cf[i] = cv[f[i, 0]]."""
    F = _rows(f)
    n = int(F.max()) + 1
    a, b = F[:, :-1].ravel(), F[:, 1:].ravel()
    g = scipy.sparse.coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(n, n))
    k, lab = scipy.sparse.csgraph.connected_components(g, directed=False)
    first = np.full(k, n, np.int64)
    np.minimum.at(first, lab, np.arange(n))
    rank = np.empty(k, np.int64)
    rank[np.argsort(first)] = np.arange(k)
    cv = rank[lab]
    cf = cv[F[:, 0]]
    out = (cv, np.bincount(cv, minlength=k), cf, np.bincount(cf, minlength=k))
    return tuple(np.squeeze(x.astype(np.asarray(f).dtype)) for x in out)


def literal(f):
    """src/connected_components.cpp:23-64 and :98-107 line by line, over igl::adjacency_matrix (every pair of corners of
    a row, both directions, n = max(f) + 1), rows iterated in ascending column order as Eigen's InnerIterator does."""
    F = _rows(f)
    n = int(F.max()) + 1
    adj = [set() for _ in range(n)]
    for row in F:
        for j in range(len(row)):
            for k in range(j + 1, len(row)):
                adj[row[j]].add(int(row[k]))
                adj[row[k]].add(int(row[j]))
    comp = [n] * n
    counts = []
    for s in range(n):
        current = len(counts)
        num = 0
        if comp[s] < n:
            continue
        q = deque([s])
        while q:
            g = q.popleft()
            if comp[g] < n:
                continue
            comp[g] = current
            num += 1
            for nb in sorted(adj[g]):
                if comp[nb] < n:
                    continue
                q.append(nb)
        counts.append(num)
    cf = [comp[F[i, 0]] for i in range(len(F))]
    fc = [0] * len(counts)
    for c in cf:
        fc[c] += 1
    dt = np.asarray(f).dtype
    return tuple(np.squeeze(np.array(x, dtype=np.int64).reshape(-1, 1).astype(dt)) for x in (comp, counts, cf, fc))


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def random_faces(rng, m, c, hi, dtype):
    """Random rows with repeated corners and gaps in the index range (hi may exceed the indices used)."""
    f = rng.integers(0, hi, (m, c))
    if m > 2:
        f[rng.integers(0, m), :] = f[0, 0]                   # a row of one repeated corner
    return f.astype(dtype)


# ---- the restatement against the literal loops (CPU) ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", IDX)
def test_restatement_equals_literal_bfs(dtype):
    rng = np.random.default_rng(3)
    for trial in range(60):
        c = 1 + trial % 4
        m = int(rng.integers(1, 12))
        hi = int(rng.integers(1, 30))
        f = random_faces(rng, m, c, hi, dtype)
        got, want = restate(f), literal(f)
        assert all(same(a, b) for a, b in zip(got, want)), (f, got, want)
    # isolated vertices below max(f): each a component of one
    f = np.array([[9, 7, 8], [0, 2, 2]], dtype)
    assert all(same(a, b) for a, b in zip(restate(f), literal(f)))
    cv, nv, cf, nf = restate(f)
    assert list(cv) == [0, 1, 0, 2, 3, 4, 5, 6, 6, 6] and list(nv) == [2, 1, 1, 1, 1, 1, 3]
    assert list(cf) == [6, 0] and list(nf) == [1, 0, 0, 0, 0, 0, 1]


def test_restatement_shapes():
    cv, nv, cf, nf = restate(np.array([[0, 1, 2]], np.int32))
    assert cv.shape == (3,) and nv.shape == () and cf.shape == () and nf.shape == ()
    cv, nv, cf, nf = restate(np.array([[0]], np.int64))
    assert cv.shape == () and nv.shape == () and int(nv) == 1


# ---- argument errors (CPU: raised before any device call) -------------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    v = np.random.default_rng(0).random((10, 3))
    f = np.array([[0, 1, 2], [3, 4, 5]])
    cc = pcu.connected_components
    cases = [
        ((v.astype(np.int32), f), "Invalid scalar type (int32) for argument 'v'"),
        ((v, f.astype(np.float32)), "Invalid scalar type (float32) for argument 'f'"),
        ((v, f.astype(np.int16)), "Invalid scalar type (int16) for argument 'f'"),
        ((v, f[:0]), "f must have at least one row and one column"),
        ((v, f[:, :0]), "f must have at least one row and one column"),
        ((v, f.reshape(1, 2, 3)), "f must be a 1-D or 2-D array"),
        ((list(v), f), "Invalid type for v"),
        ((v, list(f)), "Invalid type for f"),
        ((v.astype(np.int32), f.astype(np.float32)), "for argument 'v'"),     # the reference's order: v first
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            cc(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        cc(v, f, None)                                       # device= is keyword only


# ---- meshes ---------------------------------------------------------------------------------------------------------
def lattice(k, lo=-1.0, hi=1.0):
    """(coordinates (k^3, 3), cubes ((k-1)^3, 8) int64) of a k^3 lattice, x fastest."""
    ax = np.linspace(lo, hi, k)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    gc = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    idx = np.arange(k ** 3).reshape(k, k, k)
    b = idx[:-1, :-1, :-1].ravel()
    off = [0, 1, 1 + k, k, k * k, 1 + k * k, 1 + k + k * k, k + k * k]
    return gc, b[:, None] + np.array(off)[None, :]


def noisy_mc_mesh(pcu, k=96, seed=5):
    """Marching cubes of a box-smoothed noise field: thousands of small closed blobs."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((k, k, k))
    for ax in range(3):
        g = (g + np.roll(g, 1, ax) + np.roll(g, -1, ax)) / 3.0
    gc, ci = lattice(k)
    return pcu.marching_cubes_sparse_voxel_grid(g.ravel() - 0.4, gc, ci, 0.0)


def two_spheres(pcu, k=64):
    gc, ci = lattice(k, -1.5, 1.5)
    s = np.minimum(np.linalg.norm(gc - [-0.7, 0, 0], axis=1) - 0.6, np.linalg.norm(gc - [0.8, 0, 0], axis=1) - 0.4)
    return pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.0)


# ---- the GPU --------------------------------------------------------------------------------------------------------
def check(got, f):
    want = restate(f)
    assert len(got) == 4
    for g, w in zip(got, want):
        g = to_numpy(g)
        assert same(g, w), (g.dtype, g.shape, w.dtype, w.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", IDX)
def test_every_dtype(pcu, vdt, idt):
    rng = np.random.default_rng(11)
    v = rng.random((50, 3)).astype(vdt)
    for c in (1, 2, 3, 4):
        f = random_faces(rng, 40, c, 70, idt)
        check(pcu.connected_components(v, f), f)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
@pytest.mark.parametrize("idt", IDX)
def test_forms(pcu, form, idt):
    import torch
    v, f = icosphere(2)
    f = np.concatenate([f, f + len(v) + 5]).astype(idt)
    got = pcu.connected_components(to_form(form, v), to_form(form, f))
    kinds = {"numpy": np.ndarray, "cuda": torch.Tensor, "cpu": torch.Tensor}
    for g in got:
        assert isinstance(g, kinds[form])
        if form != "numpy":
            assert g.is_cuda == (form == "cuda")
    check(got, f)


@pytest.mark.gpu
def test_vertex_range_and_shapes(pcu):
    v = np.random.default_rng(0).random((20, 3))
    f = np.array([[0, 1, 2], [3, 4, 5]], np.int64)           # max(f) + 1 = 6 < #v
    check(pcu.connected_components(v, f), f)
    assert to_numpy(pcu.connected_components(v, f)[0]).shape == (6,)
    f = np.array([[0, 1, 2], [30, 4, 25]], np.int32)          # max(f) + 1 = 31 > #v
    check(pcu.connected_components(v, f), f)
    cv, nv, cf, nf = pcu.connected_components(v, np.array([[2, 0, 1]], np.int32))   # one face, one component
    assert cv.shape == (3,) and nv.shape == () and cf.shape == () and nf.shape == ()
    assert int(nv) == 3 and int(cf) == 0 and int(nf) == 1
    cv, nv, cf, nf = pcu.connected_components(v, np.array([[0, 1, 2], [5, 6, 7]], np.uint64))
    assert cf.shape == (2,) and nv.shape == (4,) and cf.dtype == np.uint64 and list(nv) == [3, 1, 1, 3]
    cv, nv, cf, nf = pcu.connected_components(v, np.array([[0]], np.int64))          # n = 1
    assert cv.shape == () and nv.shape == () and int(nv) == 1
    v2, f2 = icosphere(1)
    cv, nv, cf, nf = pcu.connected_components(v2, f2)                                  # one component
    assert nv.shape == () and nf.shape == () and int(nv) == len(v2) and int(nf) == len(f2)


@pytest.mark.gpu
def test_index_errors(pcu):
    v = np.random.default_rng(0).random((10, 3))
    for f in (np.array([[0, -1, 2]], np.int32), np.array([[0, 1, -5]], np.int64), np.array([[0, 2 ** 31 - 1, 1]], np.int64),
              np.array([[0, 2 ** 31 - 1, 1]], np.uint32), np.array([[2 ** 63, 1, 1]], np.uint64)):
        with pytest.raises(ValueError, match="face indices are negative or above 2"):
            pcu.connected_components(v, f)


@pytest.mark.gpu
def test_permuted_icosphere(pcu):
    v, f = icosphere(8)                                       # 1 310 720 faces
    assert len(f) == 1310720
    perm = np.random.default_rng(2).permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    fp = inv[f].astype(np.int32)
    got = pcu.connected_components(v[perm], fp)
    check(got, fp)
    assert got[1].shape == () and int(got[1]) == len(v)


@pytest.mark.gpu
def test_disjoint_triangles(pcu):
    m = 10 ** 6
    f = np.random.default_rng(4).permutation(3 * m).reshape(m, 3).astype(np.int64)
    got = pcu.connected_components(np.zeros((3 * m, 3)), f)
    check(got, f)
    assert len(got[1]) == m and (got[1] == 3).all() and (got[3] == 1).all()


@pytest.mark.gpu
def test_numbered_strip(pcu):
    m = 10 ** 6
    i = np.arange(m)
    f = np.stack([i, i + 1, i + 2], 1).astype(np.int32)
    got = pcu.connected_components(np.zeros((m + 2, 3), np.float32), f)
    check(got, f)
    fr = f[::-1].copy()                                       # the same strip, faces in reverse order
    check(pcu.connected_components(np.zeros((m + 2, 3), np.float32), fr), fr)


@pytest.mark.gpu
def test_marching_cubes_components(pcu):
    v, f = noisy_mc_mesh(pcu)
    got = pcu.connected_components(v, f)
    check(got, f)
    assert len(got[1]) > 1000


@pytest.mark.gpu
def test_reference_example_and_repeatability(pcu):
    """tests/test_examples.py:719-730 of the reference, on a generated mesh: two shifted copies."""
    v, f = icosphere(4)
    f = np.concatenate([f, f + v.shape[0]])
    v = np.concatenate([v, v + 1.0])
    cv, nv, cf, nf = pcu.connected_components(v, f)
    assert nv.sum() == v.shape[0] and nf.sum() == f.shape[0] and len(nv) == 2
    again = pcu.connected_components(v, f)
    assert all(same(a, b) for a, b in zip((cv, nv, cf, nf), again))


@pytest.mark.gpu
def test_keep_largest_component(pcu):
    v, f = two_spheres(pcu)
    cv, nv, cf, nf = pcu.connected_components(v, f)
    assert len(nv) == 2
    keep = cv == nv.argmax()
    v2, f2 = pcu.remove_mesh_vertices(v, f, keep)
    assert np.array_equal(v2, v[keep]) and v2[:, 0].max() < 0.0          # the larger sphere, at x = -0.7
    remap = np.cumsum(keep) - 1
    assert np.array_equal(f2, remap[f[keep[f].all(1)]].astype(f.dtype))
    assert len(f2) == nf.max()
    c2 = pcu.connected_components(v2, f2)
    assert c2[1].shape == () and int(c2[1]) == len(v2)
