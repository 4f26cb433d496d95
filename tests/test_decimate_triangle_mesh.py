"""decimate_triangle_mesh: the result of DESIGN.md §3 restated round by round with numpy, its invariants, the
independence of each round's collapses and its quality against a sequential greedy (CPU); the GPU bit for bit against
the restatement, the reference's own test, meshes at scale, stalls and rejected inputs (GPU); the host-side checks."""
import heapq
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from meshes import icosphere, noisy_icosphere

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REJECTED = "produced an empty mesh"


# ---- the restatement of DESIGN.md §3 -------------------------------------------------------------------------------
def adjacency(F, alive, nv):
    """Runs of the directed edges of the alive faces, in (src, dst) order: rs, rd, the opposite vertices o0 and o1 (-1:
    a boundary edge, whose second face is the one on the virtual vertex), the record count of every run, the CSR of
    every vertex's runs and its boundary edges."""
    faces = F[alive]
    src, dst, opp = [], [], []
    for k in range(3):
        u, w, o = faces[:, (k + 1) % 3], faces[:, (k + 2) % 3], faces[:, k]
        src += [u, w]
        dst += [w, u]
        opp += [o, o]
    src, dst, opp = np.concatenate(src), np.concatenate(dst), np.concatenate(opp)
    key = src * nv + dst
    order = np.argsort(key, kind="stable")
    key, opp = key[order], opp[order]
    runs, start, count = np.unique(key, return_index=True, return_counts=True)
    o0 = opp[start]
    o1 = np.where(count >= 2, opp[np.minimum(start + 1, len(opp) - 1)], -1)
    rs, rd = runs // nv, runs % nv
    ids = np.arange(nv)
    beg, end = np.searchsorted(rs, ids, "left"), np.searchsorted(rs, ids, "right")
    nb = np.bincount(rs[o1 < 0], minlength=nv)
    return dict(key=runs, rs=rs, rd=rd, o0=o0, o1=o1, count=count, beg=beg, end=end, nb=nb)


def accepted(F, nv):
    if (F[:, 0] == F[:, 1]).any() or (F[:, 1] == F[:, 2]).any() or (F[:, 0] == F[:, 2]).any():
        return False
    adj = adjacency(F, np.ones(len(F), bool), nv)
    return bool((adj["count"] <= 2).all() and np.isin(adj["nb"], [0, 2]).all())


def validity(adj, nv):
    """Valid flag of every run (False where rs > rd): the link condition on the mesh closed by the virtual vertex."""
    rs, rd, o0, o1, nb, key = adj["rs"], adj["rd"], adj["o0"], adj["o1"], adj["nb"], adj["key"]
    A = sp.csr_matrix((np.ones(len(rs)), (rs, rd)), shape=(nv, nv))
    common = np.asarray((A @ A)[rs, rd]).ravel().astype(np.int64)
    interior = o1 >= 0
    c, d = o0, o1
    ia = np.minimum(np.searchsorted(key, rs * nv + c), len(key) - 1)
    ib = np.minimum(np.searchsorted(key, rd * nv + c), len(key) - 1)
    fold = ((o0[ia] == d) | (o1[ia] == d)) & ((o0[ib] == d) | (o1[ib] == d))
    ok_int = (c != d) & ~((nb[rs] > 0) & (nb[rd] > 0)) & (common == 2) & ~fold
    ok_bnd = (common == 1) & ~((o1[ia] < 0) & (o1[ib] < 0))
    return (rs < rd) & np.where(interior, ok_int, ok_bnd)


def edge_keys(x, a, b):
    d = x[a] - x[b]
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def ragged(beg, end):
    """The concatenated ranges [beg[i], end[i]) and the i each element came from."""
    n = end - beg
    owner = np.repeat(np.arange(len(n)), n)
    return np.repeat(beg, n) + np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n), owner


def one_round(F, alive, x, max_faces):
    """One round in place: returns (valid count, applied (a, b) pairs in rank order, faces removed)."""
    nv = len(x)
    adj = adjacency(F, alive, nv)
    valid = np.nonzero(validity(adj, nv))[0]
    if len(valid) == 0:
        return 0, np.zeros((0, 2), np.int64), 0
    A = int(alive.sum())
    K = A - max_faces
    a, b = adj["rs"][valid], adj["rd"][valid]
    ranked = valid[np.argsort(edge_keys(x, a, b), kind="stable")]   # valid is in run order: ties by (a, b)
    cand = ranked[:K]
    P = len(cand)
    ca, cb = adj["rs"][cand], adj["rd"][cand]
    na, oa = ragged(adj["beg"][ca], adj["end"][ca])
    nbb, ob = ragged(adj["beg"][cb], adj["end"][cb])
    verts = np.concatenate([ca, cb, adj["rd"][na], adj["rd"][nbb]])
    owner = np.concatenate([np.arange(P), np.arange(P), oa, ob])
    stamp = np.full(nv, np.iinfo(np.int64).max)
    np.minimum.at(stamp, verts, owner)
    sel = np.bincount(owner, weights=stamp[verts] != owner, minlength=P) == 0
    rem = sel * np.where(adj["o1"][cand] >= 0, 2, 1)
    applied = sel & (np.cumsum(rem) - rem < K)
    pa, pb = ca[applied], cb[applied]
    collapse(F, alive, x, pa, pb)
    return len(valid), np.stack([pa, pb], 1), int(rem[applied].sum())


def collapse(F, alive, x, pa, pb):
    """b merges into a at the midpoint, every alive face relabelled, faces with a repeated corner die."""
    m = np.arange(len(x))
    m[pb] = pa
    x[pa] = (x[pa] + x[pb]) * 0.5
    F[alive] = m[F[alive]]
    G = F[alive]
    alive[np.nonzero(alive)[0]] = (G[:, 0] != G[:, 1]) & (G[:, 1] != G[:, 2]) & (G[:, 0] != G[:, 2])
    return m


def decimate(v, f, max_faces, rounds_out=None):
    """The restatement: (v_out, f_out, v_corr, f_corr) in the dtypes of the package's result, and the number of rounds
    that collapsed an edge."""
    x = v.astype(np.float64)
    F = f.astype(np.int64)
    assert accepted(F, len(x))
    alive = np.ones(len(F), bool)
    rounds = 0
    while alive.sum() > max_faces:
        nvalid, _, _ = one_round(F, alive, x, max_faces)
        if nvalid == 0:
            break
        rounds += 1
    if rounds_out is not None:
        rounds_out.append(rounds)
    return output(x, F, alive, v.dtype, f.dtype)


def output(x, F, alive, vdtype, fdtype):
    f_corr = np.nonzero(alive)[0]
    fo = F[f_corr]
    v_corr = np.unique(fo)
    return (x[v_corr].astype(vdtype), np.searchsorted(v_corr, fo).astype(fdtype), v_corr.astype(fdtype), f_corr.astype(fdtype))


# ---- meshes --------------------------------------------------------------------------------------------------------
def grid_faces(nu, nv, wrap_u, wrap_v):
    """Two triangles per cell of an nu x nv vertex grid, wrapped along u and / or v."""
    cu, cv = (nu if wrap_u else nu - 1), (nv if wrap_v else nv - 1)
    i, j = np.meshgrid(np.arange(cu), np.arange(cv), indexing="ij")
    i, j = i.ravel(), j.ravel()
    p = lambda a, b: (a % nu) * nv + (b % nv)  # noqa: E731
    q00, q10, q01, q11 = p(i, j), p(i + 1, j), p(i, j + 1), p(i + 1, j + 1)
    return np.concatenate([np.stack([q00, q10, q11], 1), np.stack([q00, q11, q01], 1)]).astype(np.int64)


def torus(nu=40, nv=20, R=1.0, r=0.35):
    u, w = np.meshgrid(np.linspace(0, 2 * np.pi, nu, endpoint=False), np.linspace(0, 2 * np.pi, nv, endpoint=False), indexing="ij")
    v = np.stack([(R + r * np.cos(w)) * np.cos(u), (R + r * np.cos(w)) * np.sin(u), r * np.sin(w)], -1).reshape(-1, 3)
    return v, grid_faces(nu, nv, True, True)


def noisy_disk(n=24, seed=0):
    rng = np.random.default_rng(seed)
    s, t = np.meshgrid(np.linspace(-1, 1, n), np.linspace(-1, 1, n), indexing="ij")
    v = np.stack([s, t, 0.05 * rng.standard_normal(s.shape)], -1).reshape(-1, 3)
    v[:, :2] += 0.01 * rng.standard_normal((len(v), 2))
    return v, grid_faces(n, n, False, False)


def holed_sphere():
    """A level-3 icosphere without the faces of three far-apart vertices: three boundary loops."""
    v, f = icosphere(3)
    holes = [int(np.argmax(v @ d)) for d in ([0, 0, 1], [1, 0, 0], [0, -1, -0.2])]
    return v, f[~np.isin(f, holes).any(1)]


def many_components():
    parts = [icosphere(1), torus(12, 8), noisy_disk(8, 3), icosphere(2), holed_sphere()]
    vs, fs, off = [], [], 0
    for i, (v, f) in enumerate(parts):
        vs.append(v + np.array([3.0 * i, 0, 0]))
        fs.append(f + off)
        off += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def bunny():
    return np.load(os.path.join(GOLDEN, "bunny_vertices.npy")), np.load(os.path.join(GOLDEN, "bunny_faces.npy"))


MESHES = {"icosphere": lambda: icosphere(3), "torus": torus, "disk": noisy_disk, "holed_sphere": holed_sphere,
          "components": many_components, "bunny": bunny}


# ---- invariants ----------------------------------------------------------------------------------------------------
def topology(v_count, f):
    """Per component (labelled by its smallest vertex): Euler characteristic and boundary loops."""
    f = np.asarray(f, np.int64)
    used = np.unique(f)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    ue, cnt = np.unique(e, axis=0, return_counts=True)
    g = sp.coo_matrix((np.ones(len(ue)), (ue[:, 0], ue[:, 1])), shape=(v_count, v_count))
    _, lab = connected_components(g, directed=False)
    out = {}
    bnd = ue[cnt == 1]
    gb = sp.coo_matrix((np.ones(len(bnd)), (bnd[:, 0], bnd[:, 1])), shape=(v_count, v_count))
    _, blab = connected_components(gb, directed=False)
    for c in np.unique(lab[used]):
        verts = used[lab[used] == c]
        nf = int((lab[f[:, 0]] == c).sum())
        ne = int((lab[ue[:, 0]] == c).sum())
        loops = len(np.unique(blab[bnd[lab[bnd[:, 0]] == c][:, 0]])) if len(bnd) else 0
        out[int(verts.min())] = (len(verts) - ne + nf, loops)
    return out


def check_invariants(v, f, max_faces, res, rep=None):
    v_out, f_out, v_corr, f_corr = res
    nf = len(f_out)
    x = np.asarray(v_corr, np.int64)
    assert nf in (max_faces, max_faces - 1) or (nf > max_faces), (nf, max_faces)
    assert np.all(np.diff(x) > 0) and x.min() >= 0 and x.max() < len(v)
    fc = np.asarray(f_corr, np.int64)
    assert np.all(np.diff(fc) > 0) and fc.min() >= 0 and fc.max() < len(f)
    fo = x[np.asarray(f_out, np.int64)]                           # output faces in input vertex ids
    assert accepted(fo, len(v)), "the closed output is not edge-manifold"
    assert len(np.unique(np.sort(fo, 1), axis=0)) == nf, "duplicate face"
    # topology per component, the input's component of each output vertex labelling it
    before, after = topology(len(v), f), topology(len(v), fo)
    g = sp.coo_matrix((np.ones(3 * len(f)), (np.repeat(np.asarray(f, np.int64)[:, 0], 3), np.asarray(f, np.int64).ravel())),
                      shape=(len(v), len(v)))
    _, lab = connected_components(g, directed=False)
    first = {}
    for vid in np.unique(np.asarray(f, np.int64)):
        first.setdefault(lab[vid], vid)
    after_by_input = {first[lab[k]]: val for k, val in after.items()}
    assert after_by_input == before
    if rep is not None:
        assert np.array_equal(fo, rep[np.asarray(f, np.int64)[fc]])


def decimate_traced(v, f, max_faces):
    """The restatement with the composed collapse map of every input vertex."""
    x = v.astype(np.float64)
    F = f.astype(np.int64)
    alive = np.ones(len(F), bool)
    rep = np.arange(len(x))
    while alive.sum() > max_faces:
        nvalid, pairs, _ = one_round(F, alive, x, max_faces)
        if nvalid == 0:
            break
        m = np.arange(len(x))
        m[pairs[:, 1]] = pairs[:, 0]
        rep = m[rep]
    return output(x, F, alive, v.dtype, f.dtype), rep


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("frac", [2, 4, 20])
def test_restatement_invariants(name, frac):
    v, f = MESHES[name]()
    target = max(1, len(f) // frac)
    res, rep = decimate_traced(v, f, target)
    check_invariants(v, f, target, res, rep)
    if name not in ("components",):                               # a lone small part may stall in the mix
        assert len(res[1]) in (target, target - 1)


def test_restatement_stalls_on_tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int64)
    vo, fo, vc, fc = decimate(v, f, 2)
    assert np.array_equal(fo, f) and np.array_equal(vo, v)


@pytest.mark.parametrize("name", ["icosphere", "disk", "holed_sphere", "bunny"])
def test_rounds_are_independent(name):
    """Each round's applied collapses, one by one in shuffled order, each valid at its turn, reach the same state."""
    v, f = MESHES[name]()
    x = v.astype(np.float64)
    F = f.astype(np.int64)
    alive = np.ones(len(F), bool)
    target = len(f) // 10
    rng = np.random.default_rng(7)
    for _ in range(4):
        if alive.sum() <= target:
            break
        x1, F1, al1 = x.copy(), F.copy(), alive.copy()
        before = int(alive.sum())
        nvalid, pairs, removed = one_round(F, alive, x, target)
        assert nvalid > 0 and len(pairs) > 0
        for i in rng.permutation(len(pairs)):
            a, b = pairs[i]
            adj = adjacency(F1, al1, len(x1))
            j = np.searchsorted(adj["key"], a * len(x1) + b)
            assert adj["key"][j] == a * len(x1) + b and validity(adj, len(x1))[j], (a, b)
            collapse(F1, al1, x1, np.array([a]), np.array([b]))
        assert np.array_equal(al1, alive) and np.array_equal(F1[alive], F[alive]) and np.array_equal(x1, x)
        assert before - int(alive.sum()) == removed


# ---- quality against a sequential greedy -----------------------------------------------------------------------------
def greedy(v, f, max_faces):
    """One collapse at a time, the shortest valid edge first (a heap with lazy updates), the same key, validity rule and
    midpoint: the algorithm of the reference's decimation with this package's cost."""
    x = v.astype(np.float64).copy()
    F = [list(r) for r in np.asarray(f, np.int64)]
    alive = [True] * len(F)
    vf = [set() for _ in range(len(x))]
    for t, r in enumerate(F):
        for c in r:
            vf[c].add(t)
    nalive = len(F)

    def nbrs(a):
        return {c for t in vf[a] for c in F[t]} - {a}

    def is_bnd_edge(a, c):
        return len(vf[a] & vf[c]) == 1

    def on_bnd(a):
        return any(is_bnd_edge(a, c) for c in nbrs(a))

    def opp(a, b):
        return [next(c for c in F[t] if c != a and c != b) for t in vf[a] & vf[b]]

    def valid(a, b):
        o = opp(a, b)
        if not o:
            return False
        common = nbrs(a) & nbrs(b)
        if len(o) == 2:
            c, d = o
            if c == d or (on_bnd(a) and on_bnd(b)) or common != {c, d}:
                return False
            return not (vf[a] & vf[c] & vf[d] and vf[b] & vf[c] & vf[d])
        c = o[0]
        return common == {c} and not (is_bnd_edge(a, c) and is_bnd_edge(b, c))

    def key(a, b):
        d = x[a] - x[b]
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]

    heap = []
    for a in range(len(x)):
        for b in nbrs(a):
            if a < b:
                heap.append((key(a, b), a, b))
    heapq.heapify(heap)
    while nalive > max_faces and heap:
        k, a, b = heapq.heappop(heap)
        if not (vf[a] & vf[b]) or k != key(a, b) or not valid(a, b):
            continue
        touched = nbrs(a) | nbrs(b)
        for t in vf[a] & vf[b]:
            alive[t] = False
            nalive -= 1
            for c in F[t]:
                vf[c].discard(t)
        for t in list(vf[b]):
            F[t] = [a if c == b else c for c in F[t]]
            vf[a].add(t)
        vf[b].clear()
        x[a] = (x[a] + x[b]) * 0.5
        for u in touched | {a}:
            for w in nbrs(u):
                heapq.heappush(heap, (key(min(u, w), max(u, w)), min(u, w), max(u, w)))
    return output(x, np.array(F, np.int64), np.array(alive), v.dtype, np.int64)


def point_triangle_distance(p, a, b, c):
    """Distances from points p (n, 3) to triangles (a, b, c) (each (n, 3)), by the regions of Ericson's closest point."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = (ab * ap).sum(1), (ac * ap).sum(1)
    bp = p - b
    d3, d4 = (ab * bp).sum(1), (ac * bp).sum(1)
    cp = p - c
    d5, d6 = (ab * cp).sum(1), (ac * cp).sum(1)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    denom = va + vb + vc
    with np.errstate(divide="ignore", invalid="ignore"):
        v = vb / denom
        w = vc / denom
        q = a + ab * v[:, None] + ac * w[:, None]
        t_ab = d1 / (d1 - d3)
        t_ac = d2 / (d2 - d6)
        t_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    cases = [
        (d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (d6 >= 0) & (d5 <= d6),
        (vc <= 0) & (d1 >= 0) & (d3 <= 0), (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)]
    points = [a, b, c, a + ab * t_ab[:, None], a + ac * t_ac[:, None], b + (c - b) * t_bc[:, None]]
    done = np.zeros(len(p), bool)
    for m, pt in zip(cases, points):
        m = m & ~done
        q[m] = pt[m]
        done |= m
    return np.linalg.norm(p - q, axis=1)


def point_mesh_distance(p, v, f, chunk=64):
    out = np.empty(len(p))
    A, B, C = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    for s in range(0, len(p), chunk):
        q = p[s:s + chunk]
        n = len(q)
        d = point_triangle_distance(np.repeat(q, len(f), 0), np.tile(A, (n, 1)), np.tile(B, (n, 1)), np.tile(C, (n, 1)))
        out[s:s + n] = d.reshape(n, len(f)).min(1)
    return out


def quality(v, f, res):
    vo, fo = res[0].astype(np.float64), np.asarray(res[1], np.int64)
    e = np.sort(np.concatenate([fo[:, [0, 1]], fo[:, [1, 2]], fo[:, [2, 0]]]), 1)
    e = np.unique(e, axis=0)
    mean_edge = np.linalg.norm(vo[e[:, 0]] - vo[e[:, 1]], axis=1).mean()
    v64 = v.astype(np.float64)
    haus = max(point_mesh_distance(vo, v64, np.asarray(f, np.int64)).max(), point_mesh_distance(v64, vo, fo).max())
    return mean_edge, haus


# The rounds against the sequential greedy (same key, validity and placement), mean edge length and the symmetric
# vertex-to-surface Hausdorff distance to the input.  Measured (DESIGN.md §7), rounds over greedy: bunny at f // 4,
# mean edge 0.9993 and Hausdorff 1.000; noisy icosphere at f // 10, 0.9993 and 1.000.  The bounds leave a margin.
@pytest.mark.parametrize("name,frac", [("bunny", 4), ("noisy_icosphere", 10)])
def test_quality_against_sequential_greedy(name, frac):
    v, f = bunny() if name == "bunny" else noisy_icosphere(4, 1, 0.02)
    target = len(f) // frac
    ours, ref = quality(v, f, decimate(v, f, target)), quality(v, f, greedy(v, f, target))
    assert ours[0] <= 1.02 * ref[0], (ours, ref)
    assert ours[1] <= 1.10 * ref[1], (ours, ref)


# ---- host-side checks ----------------------------------------------------------------------------------------------
def test_signature():
    import inspect
    import pcu_b200 as pcu
    sig = inspect.signature(pcu.decimate_triangle_mesh)
    assert list(sig.parameters) == ["v", "f", "max_faces", "decimation_heuristic", "device"]
    assert sig.parameters["decimation_heuristic"].default == "shortest_edge"
    assert sig.parameters["device"].kind == inspect.Parameter.KEYWORD_ONLY
    assert "decimate_triangle_mesh" in pcu.__all__


def test_argument_errors(pcu):
    v = np.random.rand(4, 3)
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.decimate_triangle_mesh(v.astype(np.int64), f, 1)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.decimate_triangle_mesh(v, f.astype(np.float32), 1)
    with pytest.raises(ValueError, match="zero elements"):
        pcu.decimate_triangle_mesh(v[:0], f, 1)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.decimate_triangle_mesh(v[:, :2], f, 1)
    with pytest.raises(ValueError, match="Invalid type"):
        pcu.decimate_triangle_mesh(v.tolist(), f, 1)
    with pytest.raises(ValueError, match=r"max_faces must be greater than 0, got 0\."):
        pcu.decimate_triangle_mesh(v, f, 0)
    with pytest.raises(ValueError, match=r"less than or equal to the number of input faces \(2\), got 3\."):
        pcu.decimate_triangle_mesh(v, f, 3)
    with pytest.raises(ValueError, match="Invalid decimation heuristic"):
        pcu.decimate_triangle_mesh(v, f, 1, "qem")
    with pytest.raises(ValueError, match="Only 3D inputs"):         # the mesh check comes first
        pcu.decimate_triangle_mesh(v[:, :2], f, 0, "qem")


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _same(got, want):
    for g, w in zip(got, want):
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        assert g.dtype == w.dtype and g.shape == w.shape, (g.dtype, w.dtype, g.shape, w.shape)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)) if g.size else True


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MESHES))
def test_gpu_matches_restatement(pcu, name):
    v, f = MESHES[name]()
    for frac in (1, 2, 4, 20, None):
        target = 1 if frac is None else max(1, len(f) // frac)
        want = decimate(v, f, target)
        _same(pcu.decimate_triangle_mesh(v, f, target), want)


@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("fdt", [np.int32, np.int64, np.uint32, np.uint64])
def test_gpu_dtypes_and_forms(pcu, vdt, fdt):
    import torch
    v, f = holed_sphere()
    v, f = v.astype(vdt), f.astype(fdt)
    target = len(f) // 4
    want = decimate(v, f, target)
    _same(pcu.decimate_triangle_mesh(v, f, target), want)
    if fdt in (np.int32, np.int64):
        got = pcu.decimate_triangle_mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), target)
        assert all(g.is_cuda for g in got)
        _same(got, want)
        got = pcu.decimate_triangle_mesh(torch.from_numpy(v), torch.from_numpy(f), target)
        assert all(isinstance(g, torch.Tensor) and not g.is_cuda for g in got)
        _same(got, want)


@pytest.mark.gpu
def test_gpu_device_routing(pcu):
    import torch
    v, f = icosphere(2)
    want = decimate(v, f, 100)
    _same(pcu.decimate_triangle_mesh(v, f, 100, device=0), want)
    _same(pcu.decimate_triangle_mesh(v, f, 100, device="cuda:0"), want)
    with pytest.raises(ValueError, match="out of range"):
        pcu.decimate_triangle_mesh(v, f, 100, device=pcu.device_count())
    if pcu.device_count() > 1:
        with pytest.raises(ValueError, match="contradicts"):
            pcu.decimate_triangle_mesh(torch.from_numpy(v).cuda(0), torch.from_numpy(f).cuda(0), 100, device=1)


@pytest.mark.gpu
def test_gpu_reference_bunny(pcu):
    """tests/test_examples.py:680-691 of the reference."""
    v, f = bunny()
    target = f.shape[0] // 4
    v_d, f_d, v_c, f_c = pcu.decimate_triangle_mesh(v, f, target)
    assert v_c.max() < v.shape[0]
    assert f_c.max() < f.shape[0]
    assert f_d.shape[0] <= target
    assert v_d.dtype == v.dtype and f_d.dtype == f.dtype and v_c.dtype == f.dtype and f_c.dtype == f.dtype
    assert v_c.shape == (v_d.shape[0],) and f_c.shape == (f_d.shape[0],)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["icosphere", "torus"])
def test_gpu_scale(pcu, name):
    import torch
    v, f = icosphere(8) if name == "icosphere" else torus(1000, 650)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    for frac in (4, 100):
        target = len(f) // frac
        res = [r.cpu().numpy() for r in pcu.decimate_triangle_mesh(vt, ft, target)]
        assert len(res[1]) in (target, target - 1)
        check_invariants(v, f, target, res)


@pytest.mark.gpu
def test_gpu_stall_and_determinism(pcu):
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int64)
    vo, fo, vc, fc = pcu.decimate_triangle_mesh(v, f, 2)
    assert np.array_equal(fo, f) and np.array_equal(vo, v) and np.array_equal(vc, np.arange(4)) and np.array_equal(fc, np.arange(4))
    vb, fb = bunny()
    a = pcu.decimate_triangle_mesh(vb, fb, 500)
    b = pcu.decimate_triangle_mesh(vb, fb, 500)
    _same(a, b)


@pytest.mark.gpu
def test_gpu_rejected_inputs(pcu):
    v = np.random.default_rng(0).random((6, 3))
    three = np.array([[0, 1, 2], [0, 1, 3], [0, 1, 4]], np.int64)               # edge (0, 1) in three faces
    bowtie = np.array([[0, 1, 2], [0, 3, 4]], np.int64)                         # vertex 0 with four boundary edges
    degenerate = np.array([[0, 1, 2], [0, 0, 3]], np.int64)
    for f in (three, bowtie, degenerate):
        assert not accepted(f, len(v))
        with pytest.raises(ValueError, match=REJECTED):
            pcu.decimate_triangle_mesh(v, f, 1)
    with pytest.raises(ValueError, match="Invalid face indices"):
        pcu.decimate_triangle_mesh(v, np.array([[0, 1, 6]], np.int64), 1)
    with pytest.raises(ValueError, match="Invalid face indices"):
        pcu.decimate_triangle_mesh(v, np.array([[0, 1, -1]], np.int64), 1)
    bad = v.copy()
    bad[5, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        pcu.decimate_triangle_mesh(bad, np.array([[0, 1, 2]], np.int64), 1)
