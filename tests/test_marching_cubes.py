"""marching_cubes_sparse_voxel_grid: the generated case tables, the result of DESIGN.md §3 restated with numpy (and, at
full size, with torch) and checked for closed, consistently oriented surfaces; on the GPU, the function bit for bit
against the restatement over every dtype, input form and cube arrangement, and the SDF -> mesh pipeline."""
import math
import os
import sys

import numpy as np
import pytest

from meshes import icosphere, to_form, to_numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mc_tables  # noqa: E402

EDGES = np.array(mc_tables.EDGES)
INDEX_DTYPES = [np.int32, np.int64, np.uint32, np.uint64]


def _table_arrays():
    masks, tris = mc_tables.tables()
    tab = np.full((256, mc_tables.MAX_TRIS, 3), -1, np.int64)
    for c, t in enumerate(tris):
        if t:
            tab[c, :len(t)] = t
    return tab, np.array([len(t) for t in tris])


TRI_TAB, TRI_CNT = _table_arrays()


# ---- the restatement -----------------------------------------------------------------------------------------------
def restate(gs, gc, ci, iso):
    """(v, f) of DESIGN.md §3 with numpy: v in gc's dtype T, every operation rounded in T; f as int64.  #v may be 0."""
    T, S = gc.dtype.type, gs.dtype.type
    iso_t = T(S(iso))
    s = gs.reshape(-1).astype(gc.dtype)
    ci = ci.astype(np.int64)
    n, m = len(s), len(ci)
    above = s[ci] > iso_t
    case = (above.astype(np.int64) << np.arange(8)).sum(1)
    cross = above[:, EDGES[:, 0]] != above[:, EDGES[:, 1]]
    cidx, eidx = np.nonzero(cross)                        # slots: cube ascending, then edge ascending
    ia, ib = ci[cidx, EDGES[eidx, 0]], ci[cidx, EDGES[eidx, 1]]
    key = np.minimum(ia, ib) * n + np.maximum(ia, ib)
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    order = np.argsort(first)                             # vertices in order of their first slot
    vid = np.empty_like(order)
    vid[order] = np.arange(len(order))
    slot_vid = vid[inv.reshape(-1)]
    fs = first[order]
    i, j = ia[fs], ib[fs]
    with np.errstate(all="ignore"):
        t = (iso_t - s[i]) / (s[j] - s[i])
        v = gc[i] + t[:, None] * (gc[j] - gc[i])
    slot_of = np.full((m, 12), -1, np.int64)
    slot_of[cidx, eidx] = np.arange(len(cidx))
    cnt = TRI_CNT[case]
    cc = np.repeat(np.arange(m), cnt)
    tt = np.arange(len(cc)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    f = slot_vid[slot_of[cc[:, None], TRI_TAB[case[cc], tt]]] if len(cc) else np.zeros((0, 3), np.int64)
    return v.astype(gc.dtype), f.reshape(-1, 3)


def lattice(k, dtype=np.float64, lo=-1.0, hi=1.0):
    """(coordinates (k^3, 3), cubes ((k-1)^3, 8) int64) of a k^3 lattice, x fastest."""
    ax = np.linspace(lo, hi, k).astype(dtype)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    gc = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    idx = np.arange(k ** 3).reshape(k, k, k)              # [z, y, x]
    b = idx[:-1, :-1, :-1].ravel()
    off = [0, 1, 1 + k, k, k * k, 1 + k * k, 1 + k + k * k, k + k * k]
    return gc, b[:, None] + np.array(off)[None, :]


def edge_counts(f):
    """{directed edge: count} over the faces."""
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    u, c = np.unique(d, axis=0, return_counts=True)
    return {tuple(e): int(k) for e, k in zip(u, c)}


def assert_closed_oriented(f):
    """Every undirected edge is used by exactly two faces, once in each direction."""
    ec = edge_counts(f)
    for (a, b), k in ec.items():
        assert k == 1 and ec.get((b, a)) == 1, (a, b, k, ec.get((b, a)))


def signed_volume(v, f):
    a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


# ---- the tables (CPU) ------------------------------------------------------------------------------------------------
def test_committed_header_is_the_generated_one():
    with open(mc_tables.HEADER) as fh:
        assert fh.read() == mc_tables.render()


def test_every_case_uses_exactly_its_crossing_edges():
    masks, tris = mc_tables.tables()
    for case in range(256):
        crossing = {e for e, (a, b) in enumerate(mc_tables.EDGES) if (case >> a & 1) != (case >> b & 1)}
        assert {e for e in range(12) if masks[case] >> e & 1} == crossing
        used = {e for t in tris[case] for e in t}
        assert used == crossing, case
        cycles = mc_tables.case_cycles(case)
        assert len(tris[case]) == sum(len(c) - 2 for c in cycles), case
        assert all(t[0] == c[0] for c in cycles for t in tris[case] if t[0] in c)   # fans start at the lowest edge
    assert max(len(t) for t in tris) == mc_tables.MAX_TRIS


def test_complementary_cases_reverse_orientation():
    """One corner above and the same corner alone below give the same triangle, reversed."""
    masks, tris = mc_tables.tables()
    single = [1 << k for k in range(8)]
    for case in single:
        (a,), (b,) = tris[case], tris[255 - case]
        assert sorted(a) == sorted(b) and a != b


@pytest.mark.parametrize("seed", range(6))
def test_random_sign_fields_give_closed_oriented_surfaces(seed):
    rng = np.random.default_rng(seed)
    gc, ci = lattice(6)
    k = 6
    s = rng.standard_normal(k ** 3)
    border = (np.abs(gc) == 1.0).any(1)
    s[border] = -1.0                                       # nothing crosses the lattice's outer faces
    v, f = restate(s, gc, ci, 0.0)
    assert len(f) > 0
    assert_closed_oriented(f)
    assert len(np.unique(f)) == len(v)


def test_sphere_sdf_on_64_lattice():
    k, r = 64, 0.7
    gc, ci = lattice(k)
    s = np.linalg.norm(gc, axis=1) - r
    v, f = restate(s, gc, ci, 0.0)
    assert_closed_oriented(f)
    ne = len(edge_counts(f)) // 2
    assert len(v) - ne + len(f) == 2                      # Euler characteristic of a sphere
    h = 2.0 / (k - 1)
    vol = signed_volume(v, f)
    exact = 4.0 / 3.0 * math.pi * r ** 3
    assert vol > 0 and abs(vol - exact) <= 4.0 * math.pi * r * r * h     # within a shell one spacing thick
    on_lattice = np.isclose((v + 1.0) / h, np.round((v + 1.0) / h), atol=0, rtol=0)
    assert (on_lattice.sum(1) >= 2).all()                 # every vertex lies on a lattice edge
    assert np.abs(np.linalg.norm(v, axis=1) - r).max() < h


# ---- argument errors (CPU: raised before any device call) -----------------------------------------------------------
def test_argument_errors():
    import pcu_b200 as pcu
    gc, ci = lattice(3)
    s = np.linalg.norm(gc, axis=1) - 0.5
    mc = pcu.marching_cubes_sparse_voxel_grid
    cases = [
        ((s.astype(np.int32), gc, ci), "Invalid scalar type (int32) for argument 'grid_scalars'"),
        ((s, gc.astype(np.int64), ci), "Invalid scalar type (int64) for argument 'grid_coordinates'"),
        ((s, gc, ci.astype(np.float64)), "Invalid scalar type (float64) for argument 'cube_indices'"),
        ((s[:0], gc[:0], ci), "Invalid grid_coordinates has zero rows!"),
        ((s, gc[:, :2], ci), "Invalid shape for grid_coordinates must have shape (N, 3) but got (27, 2)"),
        ((np.stack([s, s], 1), gc, ci), "Invalid shape for grid_scalars must have shape (N,) or (N, 1) but got (27, 2)"),
        ((s[:5], gc, ci), "grid_coordinates and grid_scalars must have the same number of rows but got grid_coordinates.shape "
                          "= (27, 3), and grid_scalars.shape = (27, 3)"),
        ((s, gc, ci[:0]), "Invalid cube_indices has zero rows!"),
        ((s, gc, ci[:, :6]), "Invalid shape for cube_indices must have shape (N, 8) but got (8, 6)"),
        ((list(s), gc, ci), "Invalid type for grid_scalars"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            mc(*args, 0.0)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        mc(s, gc, ci, 0.0, None)                          # device= is keyword only


# ---- the GPU ----------------------------------------------------------------------------------------------------------
def _gpu():
    import pcu_b200 as pcu
    import torch
    return pcu, torch


def assert_same(got, want):
    gv, gf = got
    wv, wf = want
    assert gv.dtype == wv.dtype and gv.shape == wv.shape
    nan = np.isnan(wv)                                    # a NaN's payload is not part of the definition
    assert np.array_equal(np.isnan(gv), nan)
    bits = np.uint32 if gv.dtype == np.float32 else np.uint64
    assert np.array_equal(np.where(nan, 0, gv).view(bits), np.where(nan, 0, wv).view(bits))
    assert np.array_equal(gf.astype(np.int64), wf)


@pytest.mark.gpu
@pytest.mark.parametrize("cdt", [np.float32, np.float64])
@pytest.mark.parametrize("sdt", [np.float32, np.float64])
@pytest.mark.parametrize("idt", INDEX_DTYPES)
def test_equals_restatement_every_dtype(cdt, sdt, idt):
    pcu, _ = _gpu()
    rng = np.random.default_rng(7)
    gc, ci = lattice(17, cdt)
    s = (np.linalg.norm(gc.astype(np.float64) - 0.1, axis=1) - 0.6 + 0.05 * rng.standard_normal(len(gc))).astype(sdt)
    got = pcu.marching_cubes_sparse_voxel_grid(s, gc, ci.astype(idt), 0.013)
    assert got[1].dtype == idt
    assert_same(got, restate(s, gc, ci, 0.013))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms(form):
    pcu, torch = _gpu()
    gc, ci = lattice(20, np.float32)
    s = (np.linalg.norm(gc, axis=1) - 0.55).astype(np.float32)[:, None]    # (n, 1) scalars
    for idt in (np.int32, np.uint64):
        v, f = pcu.marching_cubes_sparse_voxel_grid(to_form(form, s), to_form(form, gc), to_form(form, ci.astype(idt)), 0.0)
        if form != "numpy":
            assert isinstance(v, torch.Tensor) and v.is_cuda == (form == "cuda") and f.is_cuda == (form == "cuda")
        assert_same((to_numpy(v), to_numpy(f)), restate(s, gc, ci, 0.0))


@pytest.mark.gpu
def test_sparse_shuffled_and_permuted_cubes():
    pcu, _ = _gpu()
    rng = np.random.default_rng(3)
    gc, ci = lattice(24)
    s = np.sin(3 * gc[:, 0]) * np.cos(2 * gc[:, 1]) + gc[:, 2] * 0.5
    sub = ci[rng.random(len(ci)) < 0.4]                   # a random sparse subset
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s, gc, sub, 0.1), restate(s, gc, sub, 0.1))
    shuf = sub[rng.permutation(len(sub))]
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s, gc, shuf, 0.1), restate(s, gc, shuf, 0.1))
    perm = rng.permutation(len(gc))                       # renumber the grid vertices
    inv = np.argsort(perm)
    gc2, s2, ci2 = gc[perm], s[perm], inv[ci]
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s2, gc2, ci2, 0.1), restate(s2, gc2, ci2, 0.1))
    # the same surface, vertex for vertex, up to the numbering
    v1, f1 = pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.1)
    v2, f2 = pcu.marching_cubes_sparse_voxel_grid(s2, gc2, ci2, 0.1)
    assert len(v1) == len(v2) and len(f1) == len(f2)


@pytest.mark.gpu
def test_repeated_corners_and_repeated_cubes():
    pcu, _ = _gpu()
    rng = np.random.default_rng(5)
    gc, ci = lattice(8)
    s = rng.standard_normal(len(gc))
    deg = ci.copy()
    deg[::3, 4:] = deg[::3, :4]                           # flat cubes: top face = bottom face
    deg[1::5, 1] = deg[1::5, 0]
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s, gc, deg, 0.0), restate(s, gc, deg, 0.0))
    one = np.array([[0, 1, 2, 3, 4, 5, 6, 7]], np.int64)
    g1 = lattice(2)[0]
    s1 = np.array([1.0, -1, -1, -1, -1, -1, -1, 0.5])
    many = np.repeat(one, 100000, axis=0)                 # 10^5 copies of one crossing cube: one long run per key
    v, f = pcu.marching_cubes_sparse_voxel_grid(s1, g1, many, 0.0)
    assert_same((v, f), restate(s1, g1, many, 0.0))
    assert len(v) == 6 and len(f) == 100000 * 2


@pytest.mark.gpu
def test_scalars_at_iso_and_nan():
    pcu, _ = _gpu()
    gc, ci = lattice(9)
    s = np.round(np.linalg.norm(gc, axis=1) * 4) / 4 - 0.5    # many scalars exactly 0
    assert (s == 0).sum() > 10
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.0), restate(s, gc, ci, 0.0))
    s2 = s.copy()
    s2[::7] = np.nan
    got = pcu.marching_cubes_sparse_voxel_grid(s2, gc, ci, 0.0)
    assert_same(got, restate(s2, gc, ci, 0.0))
    s32 = s2.astype(np.float32)
    assert_same(pcu.marching_cubes_sparse_voxel_grid(s32, gc.astype(np.float32), ci, 0.0),
                restate(s32, gc.astype(np.float32), ci, 0.0))


@pytest.mark.gpu
def test_bad_indices_and_no_level_set():
    pcu, torch = _gpu()
    gc, ci = lattice(5)
    s = np.linalg.norm(gc, axis=1) - 0.5
    for bad_value, idt in ((len(gc), np.int64), (-1, np.int32), (2 ** 40, np.uint64), (2 ** 32 - 1, np.uint32)):
        bad = ci.astype(idt)
        bad[3, 5] = np.array(bad_value).astype(idt)
        with pytest.raises(ValueError, match="outside"):
            pcu.marching_cubes_sparse_voxel_grid(s, gc, bad, 0.0)
        with pytest.raises(ValueError, match="outside"):
            pcu.marching_cubes_sparse_voxel_grid(to_form("cuda", s), to_form("cuda", gc), to_form("cuda", bad), 0.0)
    with pytest.raises(ValueError) as e:
        pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 5.25)
    assert str(e.value) == "No level set found for isovalue 5.250000"
    with pytest.raises(ValueError, match="No level set found for isovalue -7.000000"):
        pcu.marching_cubes_sparse_voxel_grid(to_form("cuda", s), to_form("cuda", gc), to_form("cuda", ci), -7)
    v, f = pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.0)    # the calls above left nothing behind
    assert_same((v, f), restate(s, gc, ci, 0.0))


def torch_restate(gs, gc, ci, iso):
    """restate() with torch on the GPU (for sizes numpy would take minutes on)."""
    import torch
    T = gc.dtype
    iso_t = torch.tensor(iso, dtype=gs.dtype).to(T)
    s = gs.reshape(-1).to(T)
    ci = ci.long()
    n, m = s.shape[0], ci.shape[0]
    E = torch.from_numpy(EDGES).to(gc.device)
    above = s[ci] > iso_t
    case = (above.long() << torch.arange(8, device=gc.device)).sum(1)
    cross = above[:, E[:, 0]] != above[:, E[:, 1]]
    cidx, eidx = torch.nonzero(cross, as_tuple=True)
    ia, ib = ci[cidx, E[eidx, 0]], ci[cidx, E[eidx, 1]]
    key = torch.minimum(ia, ib) * n + torch.maximum(ia, ib)
    uk, inv = torch.unique(key, return_inverse=True)
    slot = torch.arange(len(key), device=gc.device)
    first = torch.full((len(uk),), len(key), device=gc.device, dtype=torch.long).scatter_reduce(0, inv, slot, "amin")
    order = torch.argsort(first)
    vid = torch.empty_like(order)
    vid[order] = torch.arange(len(order), device=gc.device)
    slot_vid = vid[inv]
    fs = first[order]
    i, j = ia[fs], ib[fs]
    t = (iso_t - s[i]) / (s[j] - s[i])
    v = gc[i] + t[:, None] * (gc[j] - gc[i])
    slot_of = torch.full((m, 12), -1, dtype=torch.long, device=gc.device)
    slot_of[cidx, eidx] = slot
    tab, cnt_t = torch.from_numpy(TRI_TAB).to(gc.device), torch.from_numpy(TRI_CNT).to(gc.device)
    cnt = cnt_t[case]
    cc = torch.repeat_interleave(torch.arange(m, device=gc.device), cnt)
    tt = torch.arange(len(cc), device=gc.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    f = slot_vid[slot_of[cc[:, None], tab[case[cc], tt]]]
    return v, f


@pytest.mark.gpu
def test_full_size_dense_against_torch_restatement():
    pcu, torch = _gpu()
    k = 256
    ax = torch.linspace(-1, 1, k, device="cuda", dtype=torch.float64)
    z, y, x = torch.meshgrid(ax, ax, ax, indexing="ij")
    gc = torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], 1).float()
    idx = torch.arange(k ** 3, device="cuda", dtype=torch.int32).reshape(k, k, k)
    b = idx[:-1, :-1, :-1].reshape(-1)
    off = torch.tensor([0, 1, 1 + k, k, k * k, 1 + k * k, 1 + k + k * k, k + k * k], device="cuda", dtype=torch.int32)
    ci = b[:, None] + off[None, :]
    s = (gc.double().norm(dim=1) - 0.8 + 0.1 * torch.sin(9 * gc[:, 0].double())).float()
    v, f = pcu.marching_cubes_sparse_voxel_grid(s, gc, ci, 0.0)
    wv, wf = torch_restate(s, gc, ci, 0.0)
    assert torch.equal(v.view(torch.int32), wv.view(torch.int32))
    assert torch.equal(f.long(), wf)
    assert f.dtype == torch.int32 and len(v) > 10 ** 5


@pytest.mark.gpu
def test_signed_distance_pipeline():
    pcu, _ = _gpu()
    mv, mf = icosphere(4)
    k = 48
    gc, ci = lattice(k, np.float64, -1.3, 1.3)
    sdf = pcu.signed_distance_to_mesh(gc, mv, mf)[0]
    v, f = pcu.marching_cubes_sparse_voxel_grid(sdf, gc, ci, 0.0)
    assert_closed_oriented(f)
    inside = np.array([[0.0, 0.0, 0.0], [0.3, -0.2, 0.1], [-0.5, 0.4, 0.2]])
    outside = np.array([[1.3, 0.0, 0.0], [0.9, 0.9, 0.9], [-2.0, 1.0, 0.0]])
    w = pcu.triangle_soup_fast_winding_number(v, f, np.concatenate([inside, outside]))
    assert np.abs(w[:3] - 1.0).max() < 1e-2 and np.abs(w[3:]).max() < 1e-2
    h = 2.6 / (k - 1)
    d = pcu.closest_points_on_mesh(v, mv, mf)[0]
    assert np.abs(d).max() <= h * math.sqrt(3)
