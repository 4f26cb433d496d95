"""make_mesh_watertight: the manifold triangulation table (CPU), the result of DESIGN.md §3 restated with numpy and the
package's own voxelizer and closest-point query (GPU, bit for bit), the surface's properties at scale on closed,
open and non-manifold inputs (GPU), and the input forms and errors."""
import os
import sys

import numpy as np
import pytest

from meshes import icosphere, torus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mc_tables  # noqa: E402

CORNERS = np.array(mc_tables.CORNERS)
EDGES = np.array(mc_tables.EDGES)


def _tables(manifold):
    _, tris = mc_tables.tables(manifold=manifold)
    tab = np.full((256, mc_tables.MAX_TRIS, 3), -1, np.int64)
    for c, t in enumerate(tris):
        if t:
            tab[c, :len(t)] = t
    return tab, np.array([len(t) for t in tris])


TAB_M, TRI_CNT = _tables(True)
TAB_OLD, _ = _tables(False)
# per table edge: the axis it runs along and the cube corner it starts from (its lower end)
EDGE_AXIS = np.array([int(np.nonzero(CORNERS[a] != CORNERS[b])[0][0]) for a, b in mc_tables.EDGES])
EDGE_LOW = np.array([CORNERS[a] if CORNERS[a][EDGE_AXIS[e]] < CORNERS[b][EDGE_AXIS[e]] else CORNERS[b]
                     for e, (a, b) in enumerate(mc_tables.EDGES)])


# ---- the restatement of DESIGN.md §3 -------------------------------------------------------------------------------
def exterior(occ):
    """The empty voxels 6-connected to voxel (0, 0, 0)."""
    from scipy import ndimage
    lab, _ = ndimage.label(~occ)
    return lab == lab[0, 0, 0]


def surface(ext, o=(0.0, 0.0, 0.0), s=1.0, tab=TAB_M):
    """Pre-projection vertices (fp64, numbered by (voxel, axis)) and faces (int64) of the exterior's boundary."""
    N = ext.shape[0]
    cross = np.zeros(ext.shape + (3,), bool)
    cross[:-1, :, :, 0] = ext[:-1] != ext[1:]
    cross[:, :-1, :, 1] = ext[:, :-1] != ext[:, 1:]
    cross[:, :, :-1, 2] = ext[:, :, :-1] != ext[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.cumsum(flat) - 1
    idx = np.nonzero(flat)[0]
    ijk = np.stack(np.unravel_index(idx // 3, ext.shape), 1).astype(np.float64)
    coord = ijk + 0.5 + 0.5 * (idx[:, None] % 3 == np.arange(3))
    x = np.asarray(o, np.float64) + coord * np.float64(s)
    M = N - 1
    case = np.zeros((M, M, M), np.int64)
    for k, (dx, dy, dz) in enumerate(CORNERS):
        case |= ext[dx:dx + M, dy:dy + M, dz:dz + M].astype(np.int64) << k
    case = case.reshape(-1)
    cnt = TRI_CNT[case]
    cube = np.repeat(np.arange(len(case)), cnt)
    tt = np.arange(len(cube)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    edges = tab[case[cube], tt]                                        # (nf, 3) table edges
    cijk = np.stack(np.unravel_index(cube, (M, M, M)), 1)
    q = cijk[:, None, :] + EDGE_LOW[edges]                               # the edges' lower voxels
    lin = (q[..., 0] * N + q[..., 1]) * N + q[..., 2]
    return x, vid[3 * lin + EDGE_AXIS[edges]].astype(np.int64)


def _normals(p):
    u, w = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    return np.stack([u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1], u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2],
                     u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]], 1)


def occupied(pcu, v, f, s, origin):
    """voxelize_triangle_mesh's voxels, none when it accepts none (it raises there)."""
    try:
        return pcu.voxelize_triangle_mesh(v, f, s, origin)
    except ValueError as e:
        if "empty array" not in str(e):
            raise
        return np.zeros((0, 3), np.int32)


def restate(pcu, v, f, resolution):
    """(vw in fp64, fw, depth) of DESIGN.md §3."""
    vv = v.astype(np.float64)
    lo, hi = vv.min(0), vv.max(0)
    c = (lo + hi) / 2
    L = 1.4 * np.max(hi - lo)
    o = c - L / 2
    for d in range(3, 11):
        s = L / 2 ** d
        ijk = occupied(pcu, v, f, s, o + s / 2)
        if len(ijk) >= resolution or d == 10:
            break
    N = 2 ** d
    occ = np.zeros((N, N, N), bool)
    occ[ijk[:, 0], ijk[:, 1], ijk[:, 2]] = True
    x0, F = surface(exterior(occ), o, s)
    x, alpha = x0.copy(), np.ones(len(x0))
    n0 = _normals(x0[F])
    fi64 = f.astype(np.int64)
    for _ in range(10):
        _, fi, bc = pcu.closest_points_on_mesh(x, vv, f)
        A, B, C = (vv[fi64[fi, k]] for k in range(3))
        t = (bc[:, 0:1] * A + bc[:, 1:2] * B) + bc[:, 2:3] * C
        y = x + alpha[:, None] * (t - x)
        rev = np.zeros(len(x), np.int64)
        p = 1
        while True:
            back = (rev != 0) & (rev < p)
            n = _normals(np.where(back[:, None], x, y)[F])
            flip = ~(((n0[:, 0] * n[:, 0] + n0[:, 1] * n[:, 1]) + n0[:, 2] * n[:, 2]) > 0)
            if not flip.any():
                break
            vs = np.unique(F[flip])
            rev[vs[rev[vs] == 0]] = p
            p += 1
        x = np.where(rev[:, None] != 0, x, y)
        alpha = np.where(rev != 0, alpha * 0.5, alpha)
    return x, F, d


# ---- closed 2-manifold checks ---------------------------------------------------------------------------------------
def manifold_problems(F, nv):
    """Why F (faces over nv vertices) is not a closed, consistently oriented 2-manifold ([] when it is)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    F = np.asarray(F, np.int64)
    out = []
    if len(F) == 0:
        return ["no faces"]
    if np.any((F[:, 0] == F[:, 1]) | (F[:, 1] == F[:, 2]) | (F[:, 2] == F[:, 0])):
        out.append("degenerate face")
    if len(np.unique(F)) != nv:
        out.append("unreferenced vertex")
    a = F.reshape(-1)
    b = F[:, [1, 2, 0]].reshape(-1)
    key, rkey = a * nv + b, b * nv + a
    skey = np.sort(key)
    if np.any(skey[1:] == skey[:-1]):
        out.append("directed edge used twice")
    if not np.array_equal(skey, np.sort(rkey)):
        out.append("directed edge without its reverse")
    if out:
        return out
    # corner (face t, slot j) at vertex a = F[t, j]: the next corner around a is the one whose outgoing edge is the
    # reverse of the corner's incoming edge; a vertex link is one cycle when its corners form one component
    order = np.argsort(key)
    prev = F[:, [2, 0, 1]].reshape(-1)                                 # incoming edge prev -> a of every corner
    nxt = order[np.searchsorted(skey, a * nv + prev)]
    m = len(a)
    g = coo_matrix((np.ones(m, np.int8), (np.arange(m), nxt)), shape=(m, m))
    ncomp, _ = connected_components(g, directed=False)
    if ncomp != nv:
        out.append("vertex link of more than one cycle")
    return out


def signed_volume(v, F):
    p = v[F].astype(np.float64)
    return np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0


# ---- CPU: the table and the restatement ---------------------------------------------------------------------------
def test_manifold_table_properties():
    """Same masks, cycles and counts as kMcTris; no chord joins two edges on a common cube face; 20 cycles move."""
    assert mc_tables.check_manifold_table() == 20
    masks, tris = mc_tables.tables()
    masks_m, tris_m = mc_tables.tables(manifold=True)
    assert masks == masks_m
    for case in range(256):
        cycles = mc_tables.case_cycles(case)
        assert sorted(map(sorted, tris_m[case])) != [] or not cycles
        assert {frozenset(t) for t in tris_m[case]} <= {frozenset(t) for c in cycles for t in
                                                       [(c[i], c[j], c[k]) for i in range(len(c)) for j in range(len(c))
                                                        for k in range(len(c))]}


def test_header_holds_both_tables_and_kmctris_is_unchanged():
    """kMcTris is still the fan from each cycle's lowest edge; the header is what the generator writes."""
    with open(mc_tables.HEADER) as fh:
        text = fh.read()
    assert text == mc_tables.render()
    assert "kMcTrisManifold[256][3 * kMcMaxTris]" in text
    _, tris = mc_tables.tables()
    for case in range(256):
        want = [(c[0], c[i], c[i + 1]) for c in mc_tables.case_cycles(case) for i in range(1, len(c) - 1)]
        assert tris[case] == want
    body = text.split("kMcTris[256][3 * kMcMaxTris] = {")[1].split("};")[0]
    rows = [[int(x) for x in line.split("{")[1].split("}")[0].split(",")] for line in body.strip().splitlines()]
    flat = [[e for t in tris[c] for e in t] + [255] * (3 * mc_tables.MAX_TRIS - 3 * len(tris[c])) for c in range(256)]
    assert rows == flat


def _random_fields(seed, count, side):
    """`count` random binary fields of side^3 voxels, each in its own block with an empty margin, in one grid."""
    rng = np.random.default_rng(seed)
    per = int(np.ceil(count ** (1 / 3)))
    b = side + 2
    occ = np.zeros((per * b,) * 3, bool)
    for t in range(count):
        i, j, k = np.unravel_index(t, (per,) * 3)
        occ[i * b + 1:i * b + 1 + side, j * b + 1:j * b + 1 + side, k * b + 1:k * b + 1 + side] = \
            rng.random((side,) * 3) < rng.uniform(0.15, 0.85)
    return np.pad(occ, 1)


@pytest.mark.parametrize("seed", [0, 1])
def test_restated_surface_is_closed_manifold_on_random_fields(seed):
    """Thousands of random binary fields: the manifold table gives closed, outward-oriented 2-manifolds."""
    occ = _random_fields(seed, 2000, 5)
    x, F = surface(exterior(occ))
    assert manifold_problems(F, len(x)) == []
    assert signed_volume(x, F) > 0


def test_old_table_is_not_manifold_on_the_same_fields():
    """The fan from the lowest edge leaves edges with four faces on these fields (why the second table exists)."""
    occ = _random_fields(0, 2000, 5)
    x, F = surface(exterior(occ), tab=TAB_OLD)
    assert manifold_problems(F, len(x)) != []


def test_enclosed_cavities_count_as_solid():
    occ = np.zeros((8, 8, 8), bool)
    occ[2:6, 2:6, 2:6] = True
    occ[3:5, 3:5, 3:5] = False                                          # a cavity
    x, F = surface(exterior(occ))
    occ[3:5, 3:5, 3:5] = True
    x2, F2 = surface(exterior(occ))
    assert np.array_equal(x, x2) and np.array_equal(F, F2)
    assert manifold_problems(F, len(x)) == []


def test_argument_errors(pcu):
    v = np.random.rand(4, 3)
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.make_mesh_watertight(v.astype(np.int64), f)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.make_mesh_watertight(v, f.astype(np.float32))
    with pytest.raises(ValueError, match="zero elements"):
        pcu.make_mesh_watertight(v[:0], f)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.make_mesh_watertight(v[:, :2], f)
    with pytest.raises(ValueError, match="Invalid type"):
        pcu.make_mesh_watertight(v.tolist(), f)


def test_signature():
    import inspect
    import pcu_b200 as pcu
    sig = inspect.signature(pcu.make_mesh_watertight)
    assert list(sig.parameters) == ["v", "f", "resolution", "seed", "device"]
    assert sig.parameters["resolution"].default == 20_000 and sig.parameters["seed"].default == -1
    assert sig.parameters["device"].kind == inspect.Parameter.KEYWORD_ONLY
    assert "make_mesh_watertight" in pcu.__all__


# ---- meshes --------------------------------------------------------------------------------------------------------
def cube(offset=(0.0, 0.0, 0.0)):
    v = CORNERS[[0, 1, 2, 3, 4, 5, 6, 7]].astype(np.float64) + np.asarray(offset)
    f = np.array([[0, 3, 2], [0, 2, 1], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [3, 7, 6], [3, 6, 2], [0, 4, 7],
                  [0, 7, 3], [1, 2, 6], [1, 6, 5]], np.int64)
    return v, f


def soups():
    """Open and non-manifold inputs: name -> (v, f, connected)."""
    rng = np.random.default_rng(7)
    out = {}
    v, f = icosphere(4)
    cen = v[f].mean(1)
    out["sphere_small_hole"] = (v, f[cen[:, 2] < 0.97], True)
    out["sphere_large_hole"] = (v, f[cen[:, 2] < 0.5], True)
    va, fa = cube()
    vb, fb = cube((1.0, 1.0, 0.0))
    out["cubes_sharing_an_edge"] = (np.concatenate([va, vb]), np.concatenate([fa, fb + 8]), True)
    v, f = icosphere(3)
    out["duplicated_and_flipped"] = (v, np.concatenate([f, f[::3], f[1::3, ::-1]]), True)
    p = rng.random((100_000, 1, 3)) + rng.normal(scale=0.004, size=(100_000, 3, 3))
    out["disjoint_triangles"] = (p.reshape(-1, 3), np.arange(300_000).reshape(-1, 3), False)
    out["single_triangle"] = (np.array([[0.0, 0, 0], [1, 0.2, 0.3], [0.1, 1, 0.5]]), np.array([[0, 1, 2]]), True)
    return out


# ---- GPU: exact ------------------------------------------------------------------------------------------------------
def small_meshes():
    v, f = icosphere(2)
    vt, ft = torus(nu=16, nv=8)
    vc, fc = cube()
    out = {"icosphere": (v, f), "torus": (vt, ft), "cube": (vc * np.array([1.0, 0.5, 0.25]), fc)}
    s = soups()
    out["single_triangle"] = s["single_triangle"][:2]
    out["cubes_sharing_an_edge"] = s["cubes_sharing_an_edge"][:2]
    vh, fh = icosphere(2)
    out["sphere_hole"] = (vh, fh[vh[fh].mean(1)[:, 2] < 0.6])
    # flat and axis-aligned: the square lies on the grid's middle voxel boundary, where the occupancy is the voxelizer's
    # rounding of the boxes on either side (possibly none, giving an empty result)
    out["flat_square"] = (np.array([[0.0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]]), np.array([[0, 1, 2], [0, 2, 3]]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(small_meshes()))
@pytest.mark.parametrize("resolution", [100, 1000, 5000])
def test_matches_restatement_bit_for_bit(pcu, name, resolution):
    v, f = small_meshes()[name]
    vw, fw = pcu.make_mesh_watertight(v, f, resolution)
    x, F, _ = restate(pcu, v, f, resolution)
    assert fw.dtype == f.dtype and vw.dtype == np.float64
    assert np.array_equal(fw, F)
    assert np.array_equal(vw.view(np.int64), x.view(np.int64))


@pytest.mark.gpu
def test_f32_matches_restatement(pcu):
    v, f = icosphere(2)
    v32 = (v * 3 + 1).astype(np.float32)
    vw, fw = pcu.make_mesh_watertight(v32, f.astype(np.int32), 800)
    x, F, _ = restate(pcu, v32, f.astype(np.int32), 800)
    assert vw.dtype == np.float32 and fw.dtype == np.int32
    assert np.array_equal(fw, F)
    assert np.array_equal(vw, x.astype(np.float32))


# ---- GPU: properties at scale -------------------------------------------------------------------------------------
def _check_properties(pcu, v, f, vw, fw, resolution, closed, chi=None, connected=True):
    vw64 = vw.astype(np.float64)
    assert manifold_problems(fw, len(vw)) == []
    if chi is not None:
        e = len(fw) * 3 // 2
        assert len(vw) - e + len(fw) == chi
    if connected:
        cv, nv_, cf, nf_ = pcu.connected_components(vw64, fw)
        assert np.size(nf_) == 1
    assert signed_volume(vw64, fw) > 0
    vv = v.astype(np.float64)
    lo, hi = vv.min(0), vv.max(0)
    L = 1.4 * np.max(hi - lo)
    d = next(d for d in range(3, 11) if len(occupied(pcu, v, f, L / 2 ** d, ((lo + hi) / 2 - L / 2) + L / 2 ** (d + 1)))
             >= resolution or d == 10)
    s = L / 2 ** d
    dist, _, _ = pcu.closest_points_on_mesh(vw64, vv, f)
    assert dist.max() <= s * np.sqrt(1.5) * (1 + 1e-9)
    if closed:
        w_in = pcu.triangle_soup_fast_winding_number(vw64, fw, closed[0])
        w_out = pcu.triangle_soup_fast_winding_number(vw64, fw, closed[1])
        assert np.all(np.abs(w_in - 1) < 0.1) and np.all(np.abs(w_out) < 0.1)


@pytest.mark.gpu
@pytest.mark.parametrize("resolution", [20_000, 100_000, 1_000_000])
def test_icosphere_at_scale(pcu, resolution):
    v, f = icosphere(8)
    assert len(f) > 1.3e6
    vw, fw = pcu.make_mesh_watertight(v, f, resolution)
    rng = np.random.default_rng(0)
    d = rng.normal(size=(2000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    inside, outside = d * rng.uniform(0, 0.9, (2000, 1)), d * rng.uniform(1.1, 2.0, (2000, 1))
    _check_properties(pcu, v, f, vw, fw, resolution, (inside, outside), chi=2)


@pytest.mark.gpu
@pytest.mark.parametrize("resolution", [20_000, 100_000, 1_000_000])
def test_torus_at_scale(pcu, resolution):
    v, f = torus(nu=512, nv=256)
    vw, fw = pcu.make_mesh_watertight(v, f, resolution)
    rng = np.random.default_rng(1)
    u = rng.uniform(0, 2 * np.pi, 2000)
    rr = rng.uniform(0, 0.25, 2000)
    w = rng.uniform(0, 2 * np.pi, 2000)
    inside = np.stack([(1 + rr * np.cos(w)) * np.cos(u), (1 + rr * np.cos(w)) * np.sin(u), rr * np.sin(w)], 1)
    outside = np.concatenate([rng.uniform(-0.5, 0.5, (1000, 3)) * [1, 1, 0.5], rng.normal(size=(1000, 3)) * 3 + [0, 0, 4]])
    outside = outside[np.abs(np.hypot(np.hypot(outside[:, 0], outside[:, 1]) - 1, outside[:, 2]) - 0.35) > 0.1]
    _check_properties(pcu, v, f, vw, fw, resolution, (inside, outside), chi=0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(soups()))
def test_open_and_non_manifold_inputs(pcu, name):
    v, f, connected = soups()[name]
    for resolution in (5_000, 50_000):
        vw, fw = pcu.make_mesh_watertight(v, f, resolution)
        _check_properties(pcu, v, f, vw, fw, resolution, None, connected=connected)


# ---- GPU: forms -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("fdt", [np.int32, np.int64, np.uint32, np.uint64])
def test_dtypes_and_forms(pcu, vdt, fdt):
    import torch
    v, f = icosphere(2)
    v, f = v.astype(vdt), f.astype(fdt)
    vw, fw = pcu.make_mesh_watertight(v, f, 2000)
    assert vw.dtype == vdt and fw.dtype == fdt and isinstance(vw, np.ndarray)
    ref_v, ref_f = pcu.make_mesh_watertight(v, f.astype(np.int64), 2000)
    assert np.array_equal(vw, ref_v) and np.array_equal(fw.astype(np.int64), ref_f)
    vc, fc = pcu.make_mesh_watertight(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), 2000)
    assert vc.is_cuda and fc.is_cuda and str(fc.dtype) == "torch." + np.dtype(fdt).name
    assert np.array_equal(vc.cpu().numpy(), vw) and np.array_equal(fc.cpu().numpy(), fw)
    vt, ft = pcu.make_mesh_watertight(torch.from_numpy(v), torch.from_numpy(f), 2000)
    assert not vt.is_cuda and np.array_equal(vt.numpy(), vw) and np.array_equal(ft.numpy(), fw)
    vd, fd = pcu.make_mesh_watertight(v, f, 2000, device=0)
    assert np.array_equal(vd, vw) and np.array_equal(fd, fw)
    vd, fd = pcu.make_mesh_watertight(v, f, 2000, device="cuda:0")
    assert np.array_equal(vd, vw) and np.array_equal(fd, fw)


@pytest.mark.gpu
def test_seed_is_ignored_and_calls_agree(pcu):
    v, f = torus(nu=64, nv=32)
    a = pcu.make_mesh_watertight(v, f, 30_000)
    b = pcu.make_mesh_watertight(v, f, 30_000, seed=123)
    c = pcu.make_mesh_watertight(v, f, 30_000, 7)
    for x in (b, c):
        assert np.array_equal(a[0].view(np.int64), x[0].view(np.int64)) and np.array_equal(a[1], x[1])


@pytest.mark.gpu
def test_face_count_grows_with_resolution_and_depth_stops_at_ten(pcu):
    v, f = cube()
    counts = [len(pcu.make_mesh_watertight(v, f, r)[1]) for r in (10, 1_000, 10_000, 100_000)]
    assert counts == sorted(counts) and counts[0] < counts[-1]
    big = pcu.make_mesh_watertight(v, f, 1e9)
    huge = pcu.make_mesh_watertight(v, f, 1e15)
    assert np.array_equal(big[1], huge[1]) and np.array_equal(big[0], huge[0])
    # depth 10: the surface of the unit cube at voxel size 1.4 / 1024 (about 1024 / 1.4 voxels per side)
    side = (big[0].max(0) - big[0].min(0))
    assert np.allclose(side, 1.0, atol=1.4 / 1024 * 1.5)
    assert len(big[1]) > 6 * 2 * (1024 / 1.4 - 2) ** 2


@pytest.mark.gpu
def test_errors(pcu):
    import torch
    v, f = cube()
    bad = v.copy()
    bad[7, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        pcu.make_mesh_watertight(bad, f)
    with pytest.raises(ValueError, match="Invalid face indices"):
        pcu.make_mesh_watertight(v, np.concatenate([f, [[0, 1, 8]]]))
    with pytest.raises(ValueError, match="zero extent"):
        pcu.make_mesh_watertight(np.ones((3, 3)), np.array([[0, 1, 2]]))
    with pytest.raises(ValueError, match="device"):
        pcu.make_mesh_watertight(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), device=torch.cuda.device_count())
