"""orient_mesh_faces: the result of DESIGN.md §3 restated (the parity of regular pairs through a connected-components
pass over doubled faces, plus a literal bfs_orient replay on collapsed patches only) and pinned to a literal
transcription of libigl's orientable_patches + vertex_components + bfs_orient on many small random soups and on
constructed meshes; the argument errors; on the GPU, the function bit for bit (dtype, shape, values) against the
restatement over every dtype and input form, a permuted, half-reversed icosphere of 1.3 * 10^6 faces, 10^6 disjoint
triangles, a marching-cubes mesh with thousands of components, a large Moebius strip and a welded mesh with degenerate
faces, the reference's own test, winding numbers before and after, and a call that never synchronises the host."""
import os
import time
from collections import deque

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

from meshes import icosphere, to_form, to_numpy

IDX = [np.int32, np.int64, np.uint32, np.uint64]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def same_pair(got, want):
    return len(got) == 2 and all(same(to_numpy(g), w) for g, w in zip(got, want))


# ---- the literal transcription of libigl ----------------------------------------------------------------------------
def literal(f):
    """orientable_patches, vertex_components and bfs_orient as DESIGN.md §3 reads them, step by step: half-edge blocks
    (F1, F2), (F2, F0), (F0, F1); sorted rows made unique; uE2FT from summed triplets of 1; columns with more than two
    stored entries set to 0 but kept stored; A = uE2FT uE2FT^T with entries above 1 set to 1; components by a BFS from
    faces in ascending order over nonzero entries; then per patch a FIFO (with repeat pushes) from its smallest face,
    every neighbour n != f with A(f, n) != 0 in ascending order compared edge by edge with the current rows, a row
    reversed on every match."""
    a = np.asarray(f)
    dt = a.dtype
    F = [[int(x) for x in row] for row in a.reshape(len(a), -1)]
    m = len(F)
    E = [(F[i][1], F[i][2]) for i in range(m)] + [(F[i][2], F[i][0]) for i in range(m)] + [(F[i][0], F[i][1]) for i in range(m)]
    sE = [tuple(sorted(e)) for e in E]
    uE = sorted(set(sE))
    emap = {e: i for i, e in enumerate(uE)}
    cols = [dict() for _ in uE]                     # uE2FT, column-major: edge -> {face: value}
    for e in range(3 * m):
        col = cols[emap[sE[e]]]
        col[e % m] = col.get(e % m, 0) + 1
    for col in cols:
        if len(col) > 2:
            for k in col:
                col[k] = 0                          # the values go, the entries stay stored
    A = [dict() for _ in range(m)]
    for col in cols:
        for p, vp in col.items():
            for q, vq in col.items():
                A[p][q] = A[p].get(q, 0) + vp * vq
    for row in A:
        for q in row:
            if row[q] > 1:
                row[q] = 1
    C = [-1] * m
    count = 0
    for s in range(m):
        if C[s] >= 0:
            continue
        Q = deque([s])
        while Q:
            g = Q.popleft()
            if C[g] >= 0:
                continue
            C[g] = count
            for n in sorted(A[g]):
                if C[n] < 0 and A[g][n] != 0:
                    Q.append(n)
        count += 1
    FF = [list(r) for r in F]
    seen = [False] * m
    ES = ((1, 2), (2, 0), (0, 1))
    for c in range(count):
        Q = deque([next(f for f in range(m) if C[f] == c)])
        while Q:
            f = Q.popleft()
            if seen[f]:
                continue
            seen[f] = True
            for n in sorted(A[f]):
                if A[f][n] != 0 and n != f:
                    for efi in range(3):
                        ef = (FF[f][ES[efi][0]], FF[f][ES[efi][1]])
                        for eni in range(3):
                            en = (FF[n][ES[eni][0]], FF[n][ES[eni][1]])
                            if ef == en:
                                FF[n] = FF[n][::-1]
                    Q.append(n)
    return np.squeeze(np.array(FF, dtype=object).astype(dt).reshape(m, 3)), np.squeeze(np.array(C, dtype=np.int64).astype(dt))


# ---- the restatement ------------------------------------------------------------------------------------------------
def _ids(a):
    """Face ids as int64 images that are equal exactly when the ids are."""
    a = a.reshape(len(a), -1)
    return a.view(np.int64) if a.dtype == np.uint64 else a.astype(np.int64)


def pairs(V):
    """(f, g, regular, same_direction) for every edge that exactly two distinct faces f < g share."""
    m = len(V)
    frm = np.concatenate([V[:, 1], V[:, 2], V[:, 0]])
    to = np.concatenate([V[:, 2], V[:, 0], V[:, 1]])
    opp = np.concatenate([V[:, 0], V[:, 1], V[:, 2]])
    face = np.tile(np.arange(m), 3)
    lo, hi = np.minimum(frm, to), np.maximum(frm, to)
    order = np.lexsort((hi, lo))
    head = np.ones(3 * m, bool)
    head[1:] = (lo[order][1:] != lo[order][:-1]) | (hi[order][1:] != hi[order][:-1])
    edge = np.empty(3 * m, np.int64)
    edge[order] = np.cumsum(head) - 1
    ne = int(edge.max()) + 1
    nhalf = np.bincount(edge, minlength=ne)
    ef = np.unique(edge * m + face)
    nfaces = np.bincount(ef // m, minlength=ne)
    pe = ef[nfaces[ef // m] == 2].reshape(-1, 2)
    pedge, pf, pg = pe[:, 0] // m, pe[:, 0] % m, pe[:, 1] % m
    nondeg = (V[:, 0] != V[:, 1]) & (V[:, 1] != V[:, 2]) & (V[:, 0] != V[:, 2])
    h = np.flatnonzero((nfaces[edge] == 2) & (nhalf[edge] == 2))
    h = h[np.lexsort((face[h], edge[h]))].reshape(-1, 2)
    regular, same_dir = np.zeros(ne, bool), np.zeros(ne, bool)
    regular[edge[h[:, 0]]] = nondeg[face[h[:, 0]]] & nondeg[face[h[:, 1]]] & (opp[h[:, 0]] != opp[h[:, 1]])
    same_dir[edge[h[:, 0]]] = frm[h[:, 0]] == frm[h[:, 1]]
    return pf, pg, regular[pedge], same_dir[pedge]


def _labels(n, a, b):
    g = scipy.sparse.coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(n, n))
    return scipy.sparse.csgraph.connected_components(g, directed=False)[1]


def replay(rows, nbrs, s):
    """bfs_orient from s with repeat pushes dropped (the pops keep their order) over rows {face: list}."""
    enq, Q = {s}, deque([s])
    while Q:
        f = Q.popleft()
        a = rows[f]
        ef = ((a[1], a[2]), (a[2], a[0]), (a[0], a[1]))
        for n in nbrs[f]:
            c = rows[n]
            for e in ef:
                for k in range(3):
                    if (c[(k + 1) % 3], c[(k + 2) % 3]) == e:
                        c = c[::-1]
            rows[n] = c
            if n not in enq:
                enq.add(n)
                Q.append(n)


def restate(f):
    """(oriented faces, patch ids) in f's dtype, squeezed: patches are the components of the pair graph, numbered by
    their smallest face s; a patch whose doubled graph keeps 2s and 2s + 1 apart comes out consistent with s (f is
    flipped when 2f joins 2s + 1), a collapsed one is replayed literally."""
    a = np.asarray(f)
    rows = a.reshape(len(a), -1).copy()
    V = _ids(a)
    m = len(V)
    pf, pg, reg, sd = pairs(V)
    patch = _labels(m, pf, pg)
    first = np.full(patch.max() + 1, m, np.int64)
    np.minimum.at(first, patch, np.arange(m))
    s = first[patch]
    rank = np.zeros(m + 1, np.int64)
    rank[np.sort(first)] = np.arange(len(first))
    P2, G2 = 2 * pf, 2 * pg
    par = reg & sd
    keep = reg & ~sd
    da = np.concatenate([P2[keep], P2[keep] + 1, P2[par], P2[par] + 1, P2[~reg], P2[~reg], G2[~reg]])
    db = np.concatenate([G2[keep], G2[keep] + 1, G2[par] + 1, G2[par], P2[~reg] + 1, G2[~reg], G2[~reg] + 1])
    dbl = _labels(2 * m, da, db)
    collapsed = dbl[2 * s] == dbl[2 * s + 1]
    flip = ~collapsed & (dbl[2 * np.arange(m)] != dbl[2 * s])
    rows[flip] = rows[flip][:, ::-1]
    seeds = np.unique(s[collapsed])
    if len(seeds):
        faces = np.flatnonzero(collapsed)
        live = np.zeros(m, bool)
        live[faces] = True
        nbrs = {int(x): set() for x in faces}
        for p, q in zip(pf[live[pf]].tolist(), pg[live[pf]].tolist()):
            nbrs[p].add(q)
            nbrs[q].add(p)
        nbrs = {k: sorted(v) for k, v in nbrs.items()}
        r = {int(x): [int(y) for y in rows[x]] for x in faces}
        for seed in seeds.tolist():
            replay(r, nbrs, seed)
        rows[faces] = np.array([r[x] for x in faces.tolist()], dtype=object).astype(a.dtype)
    return np.squeeze(rows), np.squeeze(rank[s].astype(a.dtype))


# ---- meshes ---------------------------------------------------------------------------------------------------------
def random_soup(rng, m, hi, dtype):
    """Random rows over a few ids, with repeated corners, duplicate and reversed-duplicate faces and edges shared by
    three or more faces all frequent."""
    f = rng.integers(0, hi, (m, 3))
    if m > 3:
        f[rng.integers(0, m)] = f[rng.integers(0, m)]
        f[rng.integers(0, m)] = f[rng.integers(0, m)][::-1]
    return f.astype(dtype)


def grid(k):
    i = np.arange(k * k).reshape(k, k)
    a, b, c, d = i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, 1:].ravel(), i[1:, :-1].ravel()
    return np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)])


def moebius(n):
    """A strip of n quads (2 n faces) closed with a half twist: top i = 2 i, bottom i = 2 i + 1."""
    i = np.arange(n)
    t, b = 2 * i, 2 * i + 1
    tn, bn = np.where(i + 1 < n, t + 2, 1), np.where(i + 1 < n, b + 2, 0)
    f = np.empty((2 * n, 3), np.int64)
    f[0::2] = np.stack([t, b, tn], 1)
    f[1::2] = np.stack([b, bn, tn], 1)
    return f


def klein(p, q):
    """A p x q grid closed into a torus along j and with a reflection j -> -j along i: a Klein bottle."""
    def vid(i, j):
        if i == p:
            i, j = 0, -j
        return i * q + j % q
    f = []
    for i in range(p):
        for j in range(q):
            a, b, c, d = vid(i, j), vid(i + 1, j), vid(i + 1, j + 1), vid(i, j + 1)
            f += [[a, b, c], [a, c, d]]
    return np.array(f, np.int64)


def reverse_some(f, rng, frac=0.5):
    f = f.copy()
    r = rng.random(len(f)) < frac
    f[r] = f[r][:, ::-1]
    return f


def constructed(rng):
    g = grid(6)
    out = {"grid": reverse_some(g, rng), "moebius": reverse_some(moebius(9), rng), "klein": reverse_some(klein(5, 4), rng)}
    # two grids whose shared edge (0, 1) also has a third face: the edge joins nothing, two patches plus one
    g2 = g.copy()
    g2[g2 > 1] += 100
    out["three-face edge"] = reverse_some(np.concatenate([g, g2[::-1], [[1, 0, 500]]]), rng)
    # two fans sharing only vertex 0
    fan = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 4, 1]])
    fan2 = np.where(fan > 0, fan + 10, 0)
    out["bow-tie"] = reverse_some(np.concatenate([fan, fan2]), rng)
    return out


def extreme_ids(f, dtype):
    """f relabelled onto ids at the ends of dtype's range: int64 minimum and uint64 maximum included."""
    u = np.unique(f)
    info = np.iinfo(dtype)
    ids = [int(info.min), int(info.max)] + [int(info.min) + 1 + k for k in range(len(u) - 2)]
    lut = dict(zip(u.tolist(), ids))
    return np.vectorize(lambda x: lut[x], otypes=[object])(f).astype(dtype)


# ---- the restatement against the literal transcription (CPU) --------------------------------------------------------
@pytest.mark.parametrize("dtype", IDX)
def test_restatement_equals_literal_on_random_soups(dtype):
    rng = np.random.default_rng(7)
    for trial in range(300):
        m = int(rng.integers(1, 16))
        hi = int(rng.integers(2, 7))
        f = random_soup(rng, m, hi, dtype)
        got, want = restate(f), literal(f)
        assert same_pair(got, want), (f, got, want)


def test_restatement_equals_literal_on_constructed_meshes():
    rng = np.random.default_rng(8)
    for name, f in constructed(rng).items():
        for dt in IDX:
            fd = f.astype(dt)
            assert same_pair(restate(fd), literal(fd)), name
    for dt in (np.int64, np.uint64, np.int32, np.uint32):
        f = extreme_ids(reverse_some(klein(4, 4), rng), dt)
        assert same_pair(restate(f), literal(f))
        f = extreme_ids(reverse_some(grid(4), rng), dt)
        assert same_pair(restate(f), literal(f))


def test_restatement_on_known_cases():
    rng = np.random.default_rng(9)
    g = grid(5)
    flip = rng.random(len(g)) < 0.5
    for first, want in ((False, g), (True, g[:, ::-1])):   # consistent with face 0, whichever way it points
        flip[0] = first
        r = g.copy()
        r[flip] = r[flip][:, ::-1]
        ff, c = restate(r)
        assert np.array_equal(ff, want) and not c.any()
    fan = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4]])
    ff, c = restate(np.concatenate([fan, np.where(fan > 0, fan + 10, 0)]))
    assert list(c) == [0, 0, 0, 1, 1, 1]                   # a bow-tie vertex joins nothing
    ff, c = restate(np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]]))
    assert list(c) == [0, 1, 2]                            # an edge of three faces joins nothing
    ff, c = restate(np.array([[3, 4, 5]], np.uint32))
    assert ff.shape == (3,) and c.shape == () and c.dtype == np.uint32
    m = moebius(7)
    ff, c = restate(m)
    assert not c.any() and not np.array_equal(ff, m)       # non-orientable: the replay decides


# ---- argument errors (CPU: raised before any device call) -----------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    f = np.array([[0, 1, 2], [2, 1, 3]])
    om = pcu.orient_mesh_faces
    cases = [
        ((f.astype(np.float32),), "Invalid scalar type (float32) for argument 'f'. Expected one of ['int32', 'int64', 'uint32', 'uint64']."),
        ((f.astype(np.int16),), "Invalid scalar type (int16) for argument 'f'"),
        ((f[:0],), "Invalid input faces with zero elements: f must have shape (n, 3) where n > 0. Got f.shape =(0, 3)."),
        ((np.zeros((0, 2), np.int32),), "Invalid input faces with zero elements: f must have shape (n, 3) where n > 0. Got f.shape =(0, 2)."),
        ((f[:, :2],), "Only triangle inputs are supported: f must have shape (n, 3) where n > 0. Got f.shape =(2, 2)."),
        ((f.ravel(),), "Only triangle inputs are supported: f must have shape (n, 3) where n > 0. Got f.shape =(6, 1)."),
        ((np.zeros(0, np.int64),), "Invalid input faces with zero elements"),
        ((f.reshape(1, 2, 3),), "f must be a 1-D or 2-D array"),
        ((list(f),), "Invalid type for f"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            om(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        om(f, "uniform", None)                             # device= is keyword only


# ---- the GPU --------------------------------------------------------------------------------------------------------
def check(pcu, f):
    got = pcu.orient_mesh_faces(f)
    assert same_pair(got, restate(f))
    return got


def welded_sphere(sub):
    """The icosphere with its cap z > 0.8 removed and a degenerate face (a, b, b) welded onto every boundary edge (a, b):
    each such edge then holds three half-edges of two faces, an irregular pair, so the whole mesh is one collapsed patch."""
    v, f = icosphere(sub)
    f = f[~(v[f][:, :, 2] > 0.8).all(1)]
    e = np.concatenate([f[:, [1, 2]], f[:, [2, 0]], f[:, [0, 1]]])
    key = np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1])
    u, cnt = np.unique(key, return_counts=True)
    b = e[np.isin(key, u[cnt == 1])]
    return np.concatenate([f, np.stack([b[:, 0], b[:, 1], b[:, 1]], 1)])


def half_reversed_sphere(sub, seed=2):
    """(v, consistently oriented faces, the same faces half reversed), vertices and faces randomly permuted."""
    v, f = icosphere(sub)
    rng = np.random.default_rng(seed)
    perm = rng.permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    f = inv[f][rng.permutation(len(f))]
    return v[perm], f, reverse_some(f, rng)


@pytest.mark.gpu
@pytest.mark.parametrize("idt", IDX)
def test_every_dtype_on_random_soups(pcu, idt):
    rng = np.random.default_rng(11)
    for trial in range(40):
        f = random_soup(rng, int(rng.integers(1, 60)), int(rng.integers(2, 12)), idt)
        check(pcu, f)
    for f in constructed(rng).values():
        check(pcu, f.astype(idt))
    check(pcu, extreme_ids(reverse_some(klein(6, 5), rng), idt))
    check(pcu, extreme_ids(random_soup(rng, 50, 8, np.int64), idt))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
@pytest.mark.parametrize("idt", IDX)
def test_forms_and_shapes(pcu, form, idt):
    import torch
    rng = np.random.default_rng(12)
    _, _, f = half_reversed_sphere(2)
    f = np.concatenate([f, reverse_some(klein(5, 5), rng) + 500]).astype(idt)
    kinds = {"numpy": np.ndarray, "cuda": torch.Tensor, "cpu": torch.Tensor}
    for x in (f, f[:1], f[1:2], f[:2]):
        got = pcu.orient_mesh_faces(to_form(form, x))
        for g in got:
            assert isinstance(g, kinds[form])
            if form != "numpy":
                assert g.is_cuda == (form == "cuda")
        assert same_pair(got, restate(x))
    ff, c = pcu.orient_mesh_faces(to_form(form, f[:1]), "area")        # weighting_type is ignored
    assert tuple(ff.shape) == (3,) and tuple(c.shape) == () and int(c) == 0


@pytest.mark.gpu
def test_half_reversed_icosphere(pcu):
    v, good, f = half_reversed_sphere(8)                            # 1 310 720 faces
    assert len(f) == 1310720
    want = good if np.array_equal(f[0], good[0]) else good[:, ::-1]
    for dt in (np.int32, np.uint64):
        ff, c = check(pcu, f.astype(dt))
        assert np.array_equal(ff, want.astype(dt)) and not c.any()


@pytest.mark.gpu
def test_disjoint_triangles(pcu):
    m = 10 ** 6
    f = np.random.default_rng(4).permutation(3 * m).reshape(m, 3).astype(np.int64)
    ff, c = check(pcu, f)
    assert np.array_equal(ff, f) and np.array_equal(c, np.arange(m))


def lattice(k, lo=-1.0, hi=1.0):
    ax = np.linspace(lo, hi, k)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    gc = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    idx = np.arange(k ** 3).reshape(k, k, k)
    b = idx[:-1, :-1, :-1].ravel()
    off = [0, 1, 1 + k, k, k * k, 1 + k * k, 1 + k + k * k, k + k * k]
    return gc, b[:, None] + np.array(off)[None, :]


@pytest.mark.gpu
def test_marching_cubes_components(pcu):
    rng = np.random.default_rng(5)
    g = rng.standard_normal((96, 96, 96))
    for ax in range(3):
        g = (g + np.roll(g, 1, ax) + np.roll(g, -1, ax)) / 3.0
    gc, ci = lattice(96)
    v, f = pcu.marching_cubes_sparse_voxel_grid(g.ravel() - 0.4, gc, ci, 0.0)
    f = reverse_some(f, rng)
    ff, c = check(pcu, f)
    assert int(c.max()) > 1000


@pytest.mark.gpu
def test_replay_at_size(pcu):
    rng = np.random.default_rng(6)
    f = reverse_some(moebius(50000), rng)                          # one collapsed patch of 10^5 faces
    ff, c = check(pcu, f)
    assert not c.any()
    wf = reverse_some(welded_sphere(6), rng)                       # one collapsed patch of 74 084 faces
    deg = (wf[:, 0] == wf[:, 1]) | (wf[:, 1] == wf[:, 2]) | (wf[:, 0] == wf[:, 2])
    assert deg.sum() == 216                                        # one per boundary edge
    ff, c = check(pcu, wf.astype(np.int32))
    assert not c.any()
    check(pcu, wf.astype(np.uint64))


@pytest.mark.gpu
def test_reference_example(pcu):
    """tests/test_examples.py:755-763 of the reference: the bunny's faces come back unchanged, all in component 0."""
    f = np.load(os.path.join(GOLDEN, "bunny_faces.npy"))
    ff, c = pcu.orient_mesh_faces(f)
    assert ff.shape == f.shape and np.all(ff == f) and np.all(c == 0)
    assert same_pair((ff, c), restate(f))


@pytest.mark.gpu
def test_winding_numbers_after_orienting(pcu):
    v, good, f = half_reversed_sphere(6)
    ff, _ = pcu.orient_mesh_faces(f)
    sign = 1.0 if np.array_equal(f[0], good[0]) else -1.0          # the icosphere's faces point outwards
    p = np.random.default_rng(3).standard_normal((200, 3)) * 0.2
    w = pcu.triangle_soup_fast_winding_number(v, ff, p)
    assert np.abs(w - sign).max() < 1e-2                          # the fast winding number's far-field error is about 3e-3
    w0 = pcu.triangle_soup_fast_winding_number(v, f, p)
    assert np.abs(np.abs(w0) - 1.0).max() > 0.3


@pytest.mark.gpu
def test_cuda_call_does_not_synchronise(pcu):
    import torch
    _, _, f = half_reversed_sphere(5)
    f = np.concatenate([f, moebius(500) + len(f) * 3])
    ft = torch.from_numpy(f).cuda()
    pcu.orient_mesh_faces(ft)                                      # warm: the workspace exists and is large enough
    spin = 1 << 30                                                 # clock cycles: a good fraction of a second
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    torch.cuda._sleep(spin)
    t1.record()
    t1.synchronize()
    spin_ms = t0.elapsed_time(t1)
    before = pcu.launch_count()
    torch.cuda.set_sync_debug_mode("error")                        # no torch-side synchronisation either
    try:
        torch.cuda._sleep(spin)
        start = time.perf_counter()
        ff, c = pcu.orient_mesh_faces(ft)
        host_ms = 1e3 * (time.perf_counter() - start)
        pending = not torch.cuda.current_stream().query()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # a synchronisation anywhere inside the call would have waited for the spin enqueued just before it
    assert host_ms < spin_ms / 4, (host_ms, spin_ms)
    assert pending, "the call waited for the stream"
    assert pcu.launch_count() > before
    assert same_pair((ff, c), restate(f))
