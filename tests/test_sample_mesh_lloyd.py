"""sample_mesh_lloyd and the Voronoi cells restricted to a triangle mesh against a brute-force numpy oracle
(DESIGN.md §3, restricted cell / Lloyd sampling of a mesh).

The oracle clips every (face, seed) pair by the bisector of every other seed, vectorised over the pairs, and integrates
each polygon by a fan.  It is pinned by its own checks on the CPU; the initial sample, the Lloyd step and the L-BFGS
Newton phase are restated on top of it and compared with the GPU."""
import inspect

import numpy as np
import pytest

from meshes import icosphere
from test_mesh_sampling import degenerate_mesh, dense_samples, flat_grid, spanning_mesh
from test_voronoi_lloyd import cell_moments


# ---- the oracle --------------------------------------------------------------------------------------------------
def _clip(P, cnt, nrm, d):
    """Sutherland-Hodgman of every polygon (P (N, K, 3), cnt (N,)) by {w : nrm . w <= d} (nrm (N, 3), d (N,))."""
    N, K, _ = P.shape
    if K == 0:
        return P, cnt
    k = np.arange(K)[None, :]
    valid = k < cnt[:, None]
    nxt = (k + 1) % np.maximum(cnt, 1)[:, None]
    Q = np.take_along_axis(P, nxt[..., None].repeat(3, axis=2), axis=1)
    h = np.einsum("nkd,nd->nk", P, nrm) - d[:, None]
    hq = np.take_along_axis(h, nxt, axis=1)
    ins, insq = h <= 0, hq <= 0
    keep = valid & ins
    cross = valid & (ins != insq)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(cross, h / (h - hq), 0.0)
    X = P + (Q - P) * t[..., None]
    n_out = keep.astype(np.int64) + cross
    pos = np.cumsum(n_out, axis=1) - n_out
    new_cnt = n_out.sum(axis=1)
    out = np.zeros((N, max(int(new_cnt.max(initial=0)), 1), 3))
    r, c = np.nonzero(keep)
    out[r, pos[r, c]] = P[r, c]
    r, c = np.nonzero(cross)
    out[r, pos[r, c] + keep[r, c]] = X[r, c]
    return out, new_cnt


def _fan(P, cnt):
    """(N, 5) area, first and second moments of every polygon about the origin, fanned from vertex 0."""
    out = np.zeros((len(P), 5))
    for j in range(1, P.shape[1] - 1):
        on = j + 1 < cnt
        A, B, C = P[:, 0], P[:, j], P[:, j + 1]
        a = 0.5 * np.linalg.norm(np.cross(B - A, C - A), axis=1) * on
        s = A + B + C
        out[:, 0] += a
        out[:, 1:4] += a[:, None] * s / 3.0
        out[:, 4] += a / 12.0 * ((A * A).sum(1) + (B * B).sum(1) + (C * C).sum(1) + (s * s).sum(1))
    return out


def restricted_moments(x, v, f):
    """(n, 5): area, first moment about the seed (x, y, z), second moment about the seed of every restricted cell."""
    x = np.asarray(x, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    f = np.asarray(f, dtype=np.int64)
    n = len(x)
    seed, face = np.repeat(np.arange(n), len(f)), np.tile(np.arange(len(f)), n)
    P = v[f[face]] - x[seed][:, None, :]
    cnt = np.full(len(seed), 3)
    # a duplicate of a lower index owns nothing
    first = np.array([np.argmax(np.all(x == x[i], axis=1)) for i in range(n)])
    cnt[first[seed] < seed] = 0
    for j in range(n):
        nrm = x[j] - x[seed]
        same = np.all(nrm == 0.0, axis=1)
        d = 0.5 * (nrm * nrm).sum(1)
        nrm[same], d[same] = 0.0, 1.0            # no cut
        P, cnt = _clip(P, cnt, nrm, d)
    m = _fan(P, cnt)
    out = np.zeros((n, 5))
    np.add.at(out, seed, m)
    return out


def centroids(x, v, f):
    m = restricted_moments(x, v, f)
    g = x.copy()
    ok = m[:, 0] > 1e-30
    g[ok] = x[ok] + m[ok, 1:4] / m[ok, :1]
    return g


def face_areas(v, f):
    a, b, c = (v[f[:, k]] for k in range(3))
    return 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)


def initial_sample(v, f, n, seed):
    return dense_samples(np.asarray(v, dtype=np.float64), f, n, seed, positions=True)[2]


def lloyd_restated(v, f, n, seed, num_lloyd, num_newton):
    """The initial sample, num_lloyd Lloyd steps and the L-BFGS Newton phase of DESIGN.md §3 on the oracle's cells."""
    x = initial_sample(v, f, n, seed)
    for _ in range(num_lloyd):
        x = centroids(x, v, f)
    energies = []
    if num_newton <= 0:
        return x, energies

    def evaluate(x):
        m = restricted_moments(x, v, f)
        return m[:, 4].sum(), (-2.0 * m[:, 1:4]).ravel()

    F, g = evaluate(x)
    energies.append(F)
    S, Y, rho, gamma = [], [], [], 1.0
    xf = x.ravel()
    for _ in range(num_newton):
        if g @ g == 0.0:
            break
        q = g.copy()
        alpha = []
        for s, y, r in zip(reversed(S), reversed(Y), reversed(rho)):
            a = r * (s @ q)
            alpha.append(a)
            q -= a * y
        q *= gamma
        for (s, y, r), a in zip(zip(S, Y, rho), reversed(alpha)):
            q += (a - r * (y @ q)) * s
        p = -q
        gtp = g @ p
        if not gtp < 0.0:
            break
        t, accepted = 1.0, False
        for _h in range(21):
            xt = xf + t * p                      # no domain test: every trial is evaluated
            Ft, gt = evaluate(xt.reshape(n, 3))
            if Ft <= F + 1e-4 * t * gtp:
                accepted = True
                break
            t *= 0.5
        if not accepted:
            break
        s, y = xt - xf, gt - g
        if s @ y > 0:
            S.append(s)
            Y.append(y)
            rho.append(1.0 / (s @ y))
            gamma = (s @ y) / (y @ y)
            S, Y, rho = S[-7:], Y[-7:], rho[-7:]
        xf, F, g = xt, Ft, gt
        energies.append(F)
    return xf.reshape(n, 3), energies


def _scale(v):
    return float(np.abs(np.asarray(v, dtype=np.float64)).max())


# ---- CPU: the oracle pinned --------------------------------------------------------------------------------------
def test_oracle_partitions_the_surface():
    v, f = icosphere(2, 0.02, 3)
    x = v[np.random.default_rng(0).choice(len(v), 40, replace=False)] * 1.01
    m = restricted_moments(x, v, f)
    A = face_areas(v, f)
    assert abs(m[:, 0].sum() - A.sum()) < 1e-12 * A.sum()
    c = v[f].mean(axis=1)
    np.testing.assert_allclose((m[:, :1] * x + m[:, 1:4]).sum(0), (A[:, None] * c).sum(0), atol=1e-12)
    assert np.all(m[:, 0] > 0) and np.all(m[:, 4] > 0)


def test_oracle_flat_square_is_the_2d_cell():
    v, f = flat_grid(3)
    x2 = np.random.default_rng(1).random((30, 2))
    m = restricted_moments(np.c_[x2, np.zeros(30)], v, f)
    ref = cell_moments(x2)
    np.testing.assert_allclose(m[:, [0, 1, 2, 4]], ref[:, [0, 1, 2, 4]], atol=1e-13)
    assert np.all(m[:, 3] == 0.0)


def test_oracle_lifted_seeds():
    v, f = flat_grid(2)
    x = np.c_[np.random.default_rng(2).random((20, 2)), np.zeros(20)]
    h = 0.3
    m0 = restricted_moments(x, v, f)
    m1 = restricted_moments(x + [0.0, 0.0, h], v, f)
    np.testing.assert_allclose(m1[:, 0], m0[:, 0], atol=1e-14)
    np.testing.assert_allclose(m1[:, 4], m0[:, 4] + m0[:, 0] * h * h, atol=1e-13)
    np.testing.assert_allclose(m1[:, 3], -h * m0[:, 0], atol=1e-14)


def test_oracle_duplicates():
    v, f = icosphere(1)
    x = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0], [1.0, 0.0, 0.0]])
    m = restricted_moments(x, v, f)
    assert np.all(m[[2, 4]] == 0.0) and np.all(m[[0, 1, 3], 0] > 0)
    np.testing.assert_allclose(m[:, 0].sum(), face_areas(v, f).sum(), rtol=1e-12)
    np.testing.assert_allclose(m[[0, 1, 3]], restricted_moments(x[[0, 1, 3]], v, f), atol=1e-15)


def test_restatement_decreases_energy():
    v, f = icosphere(1, 0.02, 4)
    x, e = lloyd_restated(v, f, 12, 99, 1, 4)
    assert len(e) >= 2 and all(b <= a for a, b in zip(e, e[1:]))


def test_signature(pcu):
    ps = list(inspect.signature(pcu.sample_mesh_lloyd).parameters.values())
    assert [p.name for p in ps] == ["v", "f", "num_samples", "num_lloyd", "num_newton", "return_mesh", "device"]
    assert [p.default for p in ps[3:6]] == [10, 10, False]
    assert ps[6].kind == inspect.Parameter.KEYWORD_ONLY and ps[6].default is None
    assert "sample_mesh_lloyd" in pcu.__all__


def test_argument_errors(pcu):
    v, f = icosphere(1)
    with pytest.raises(ValueError, match="num_samples must be > 0"):
        pcu.sample_mesh_lloyd(v, f, 0)
    with pytest.raises(ValueError, match="num_samples must be > 0"):
        pcu.sample_mesh_lloyd(v, f, -5)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.sample_mesh_lloyd(v.astype(np.int32), f, 10)
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.sample_mesh_lloyd(v, f.astype(np.int16), 10)
    with pytest.raises(ValueError, match="zero elements"):
        pcu.sample_mesh_lloyd(v[:0], f, 10)
    with pytest.raises(ValueError, match="Only 3D inputs"):
        pcu.sample_mesh_lloyd(v[:, :2], f, 10)
    with pytest.raises(ValueError, match="Invalid type"):
        pcu.sample_mesh_lloyd(v.tolist(), f, 10)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _check_moments(pcu, x, v, f, tol=1e-9):
    got = pcu._lloyd._restricted_cell_moments(x, v, f)
    ref = restricted_moments(x, v, f)
    L = max(_scale(v), _scale(x))
    scale = np.array([L ** 2, L ** 3, L ** 3, L ** 3, L ** 4])
    err = np.abs(got - ref) / scale
    assert err.max() <= tol, (err.max(axis=0), np.unravel_index(err.argmax(), err.shape))
    return got


@pytest.mark.gpu
def test_moments_closed_sphere(pcu):
    v, f = icosphere(2, 0.01, 5)
    rng = np.random.default_rng(5)
    x = initial_sample(v, f, 60, 17)
    got = _check_moments(pcu, x, v, f)
    assert abs(got[:, 0].sum() - face_areas(v, f).sum()) < 1e-12 * face_areas(v, f).sum()
    # seeds off the surface, inside and outside the sphere
    _check_moments(pcu, x * rng.uniform(0.7, 1.3, (60, 1)), v, f)
    _check_moments(pcu, rng.normal(size=(40, 3)), v, f)


@pytest.mark.gpu
def test_moments_degenerate_soup_and_duplicates(pcu):
    v, f = degenerate_mesh()
    rng = np.random.default_rng(6)
    x = np.c_[rng.random((25, 2)), rng.normal(0, 0.05, 25)]
    x = np.concatenate([x, x[[3, 0, 7]], x[:2]])
    got = _check_moments(pcu, x, v, f)
    assert np.all(got[25:] == 0.0)
    for fdt in (np.int32, np.uint32, np.uint64):
        assert np.array_equal(pcu._lloyd._restricted_cell_moments(x, v.astype(np.float32), f.astype(fdt)),
                              pcu._lloyd._restricted_cell_moments(x, v.astype(np.float32).astype(np.float64), f))
    vs, fs = spanning_mesh()
    _check_moments(pcu, vs[fs].mean(axis=1)[::2] + rng.normal(0, 0.1, (20, 3)), vs, fs)
    _check_moments(pcu, np.array([[0.3, 0.2, 0.1]]), v, f)            # one seed owns every face


@pytest.mark.gpu
def test_flat_square_matches_the_2d_cells(pcu):
    v, f = flat_grid(1)
    x2 = np.random.default_rng(7).random((100_000, 2))
    got = pcu._lloyd._restricted_cell_moments(np.c_[x2, np.zeros(len(x2))], v, f)
    _, ref = pcu._lloyd._cell_moments(x2)
    np.testing.assert_allclose(got[:, [0, 1, 2, 4]], ref[:, [0, 1, 2, 4]], rtol=0, atol=1e-9)
    assert np.all(got[:, 3] == 0.0)
    assert pcu._lloyd.last_pass_counts[0] >= len(x2)


@pytest.mark.gpu
def test_cluster_runs_through_every_pass(pcu):
    rng = np.random.default_rng(8)
    d = rng.normal(size=(20_000, 2))
    d *= (0.01 * rng.random(20_000) ** 0.5 / np.linalg.norm(d, axis=1))[:, None]
    x2 = np.concatenate([0.5 + d, rng.random((300, 2))])
    v, f = flat_grid(1)
    got = pcu._lloyd._restricted_cell_moments(np.c_[x2, np.zeros(len(x2))], v, f)
    passes = pcu._lloyd.last_pass_counts
    assert passes[1] > 0 and passes[2] > 0, passes
    _, ref = pcu._lloyd._cell_moments(x2)
    np.testing.assert_allclose(got[:, [0, 1, 2, 4]], ref[:, [0, 1, 2, 4]], rtol=0, atol=1e-9)


@pytest.mark.gpu
def test_no_iterations_is_the_initial_sample(pcu):
    v, f = icosphere(3, 0.01, 2, np.float32)
    np.random.seed(11)
    seed = int(np.random.randint(2 ** 31 - 1))
    np.random.seed(11)
    got = pcu.sample_mesh_lloyd(v, f, 5000, 0, 0)
    assert got.dtype == np.float64 and got.shape == (5000, 3)
    assert np.array_equal(got, initial_sample(v, f, 5000, seed))
    assert pcu._lloyd.last_newton_energies == []


@pytest.mark.gpu
def test_lloyd_and_newton_match_the_restatement(pcu):
    v, f = icosphere(1, 0.02, 9)
    for num_lloyd, num_newton in ((3, 0), (1, 4)):
        np.random.seed(23)
        seed = int(np.random.randint(2 ** 31 - 1))
        np.random.seed(23)
        got = pcu.sample_mesh_lloyd(v, f, 24, num_lloyd, num_newton)
        ref, energies = lloyd_restated(v, f, 24, seed, num_lloyd, num_newton)
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-8)
        if num_newton:
            np.testing.assert_allclose(pcu._lloyd.last_newton_energies, energies, rtol=1e-9)


@pytest.mark.gpu
def test_newton_energies_decrease_and_calls_repeat(pcu):
    v, f = icosphere(4, 0.005, 3)
    np.random.seed(4)
    a = pcu.sample_mesh_lloyd(v, f, 3000, 3, 8)
    e = pcu._lloyd.last_newton_energies
    assert len(e) >= 2 and all(y <= x for x, y in zip(e, e[1:]))
    np.random.seed(4)
    b = pcu.sample_mesh_lloyd(v, f, 3000, 3, 8)
    assert np.array_equal(a, b)
    # evenly spread: the nearest-neighbour distances of the result vary less than the initial sample's
    from scipy.spatial import cKDTree
    np.random.seed(4)
    x0 = pcu.sample_mesh_lloyd(v, f, 3000, 0, 0)
    spread = [np.std(cKDTree(p).query(p, 2)[0][:, 1]) / np.mean(cKDTree(p).query(p, 2)[0][:, 1]) for p in (x0, a)]
    assert spread[1] < 0.5 * spread[0], spread


@pytest.mark.gpu
def test_planar_mesh_stays_in_its_plane(pcu):
    v, f = flat_grid(8)
    v[:, 2] = 0.25
    np.random.seed(5)
    x = pcu.sample_mesh_lloyd(v, f, 400, 5, 5)
    assert np.all(x[:, 2] == 0.25)
    assert x[:, :2].min() >= 0.0 and x[:, :2].max() <= 1.0


@pytest.mark.gpu
def test_input_forms_and_dtypes(pcu):
    import torch
    v, f = icosphere(2, 0.01, 1)
    np.random.seed(3)
    ref = pcu.sample_mesh_lloyd(v, f, 200, 2, 2)
    for vdt in (np.float32, np.float64):
        vv = v.astype(vdt)
        np.random.seed(3)
        base = pcu.sample_mesh_lloyd(vv, f, 200, 2, 2)
        if vdt == np.float64:
            assert np.array_equal(base, ref)
        for fdt in (np.int32, np.int64, np.uint32, np.uint64):
            ff = f.astype(fdt)
            np.random.seed(3)
            assert np.array_equal(pcu.sample_mesh_lloyd(vv, ff, 200, 2, 2), base)
            if fdt in (np.int32, np.int64):
                np.random.seed(3)
                out = pcu.sample_mesh_lloyd(torch.from_numpy(vv).cuda(), torch.from_numpy(ff).cuda(), 200, 2, 2)
                assert out.is_cuda and out.dtype == torch.float64 and np.array_equal(out.cpu().numpy(), base)
                np.random.seed(3)
                out = pcu.sample_mesh_lloyd(torch.from_numpy(vv), torch.from_numpy(ff), 200, 2, 2)
                assert not out.is_cuda and out.dtype == torch.float64 and np.array_equal(out.numpy(), base)
    np.random.seed(3)
    assert np.array_equal(pcu.sample_mesh_lloyd(v, f, 200, 2, 2, True, device=0), ref)
    with pytest.raises(ValueError):
        pcu.sample_mesh_lloyd(torch.from_numpy(v).cuda(), torch.from_numpy(f), 10)


@pytest.mark.gpu
def test_bad_meshes_raise(pcu):
    v, f = flat_grid(4)
    bad = f.copy()
    bad[3, 1] = len(v) + 5
    with pytest.raises(ValueError, match=r"Invalid face indices: 1 faces have a corner outside \[0, #v\)"):
        pcu.sample_mesh_lloyd(v, bad, 10)
    flat = v.copy()
    flat[:, 1] = 0.0
    with pytest.raises(ValueError, match="Mesh has zero area"):
        pcu.sample_mesh_lloyd(flat, f, 10)
    with pytest.raises(ValueError, match="Invalid face indices"):
        pcu._lloyd._restricted_cell_moments(np.zeros((3, 3)), v, bad)
    # a mesh of zero area has empty cells
    assert np.all(pcu._lloyd._restricted_cell_moments(np.zeros((3, 3)), flat, f) == 0.0)
