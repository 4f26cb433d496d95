"""voronoi_centroids_unit_cube, lloyd_3d and lloyd_2d against a scipy oracle (DESIGN.md §3, Voronoi cell / Lloyd).

The oracle computes every cell as the intersection of the cube's (square's) half-spaces and the bisectors of every other
seed (scipy's HalfspaceIntersection, from a Chebyshev centre) and integrates it by a fan of the convex hull's facets.
It is pinned by its own checks; the initial sample, the Lloyd step and the L-BFGS Newton phase are restated on top of
it and compared with the GPU."""
import numpy as np
import pytest
from scipy.optimize import linprog
from scipy.spatial import ConvexHull, HalfspaceIntersection

import pcu_b200 as pcu


# ---- the oracle --------------------------------------------------------------------------------------------------
def cell_moments(x, rows=None):
    """(n, 5): volume, first moment about the seed (3, zero-padded in 2-D), second moment about the seed (only `rows`
    filled when given)."""
    x = np.asarray(x, dtype=np.float64)
    n, d = x.shape
    out = np.zeros((n, 5))
    box = []
    for a in range(d):
        e = np.zeros(d)
        e[a] = -1.0
        box.append(np.r_[e, 0.0])
        e = np.zeros(d)
        e[a] = 1.0
        box.append(np.r_[e, -1.0])
    for i in range(n) if rows is None else rows:
        same = np.all(x == x[i], axis=1)
        if np.argmax(same) < i:          # a duplicate of a lower index: empty cell
            continue
        others = x[~same]
        hs = np.array(box + [np.r_[o - x[i], -(o @ o - x[i] @ x[i]) / 2] for o in others])
        A, b = hs[:, :d], -hs[:, d]
        norm = np.linalg.norm(A, axis=1)
        res = linprog(np.r_[np.zeros(d), -1.0], A_ub=np.c_[A, norm], b_ub=b, bounds=[(None, None)] * d + [(0, None)])
        if res.x[d] <= 0:
            continue
        h = HalfspaceIntersection(hs, res.x[:d])
        pts = h.intersections
        hull = ConvexHull(pts)
        c = pts.mean(axis=0)
        vol, m1, m2 = 0.0, np.zeros(d), 0.0
        for s in hull.simplices:
            P = np.vstack([c, pts[s]])
            v = abs(np.linalg.det(P[1:] - c)) / (6.0 if d == 3 else 2.0)
            w = P - x[i]
            vol += v
            m1 += v * w.mean(axis=0)
            m2 += v / ((d + 1) * (d + 2)) * ((w * w).sum() + (w.sum(axis=0) ** 2).sum())
        out[i, 0], out[i, 1:1 + d], out[i, 4] = vol, m1, m2
    return out


def cell_moments_row(x, i):
    """cell_moments of one row, from the bisectors of every other seed."""
    return cell_moments(x, [i])[i]


def centroids(x):
    x = np.asarray(x, dtype=np.float64)
    m = cell_moments(x)
    d = x.shape[1]
    g = x.copy()
    ok = m[:, 0] > 1e-30
    g[ok] = x[ok] + m[ok, 1:1 + d] / m[ok, :1]
    return g


def lattice(k, d):
    return (np.stack(np.meshgrid(*[np.arange(k)] * d, indexing="ij"), -1).reshape(-1, d) + 0.5) / k


# ---- restatements of the initial sample and the drivers ----------------------------------------------------------
def mix32(h):
    h = np.asarray(h, dtype=np.uint32)
    with np.errstate(over="ignore"):
        h = h ^ (h >> np.uint32(16))
        h = h * np.uint32(0x7feb352d)
        h = h ^ (h >> np.uint32(15))
        h = h * np.uint32(0x846ca68b)
        h = h ^ (h >> np.uint32(16))
    return h


def initial_sample(n, seed, d):
    c = 2 * np.arange(n * d, dtype=np.uint64)

    def word(c):
        lo, hi = (c & np.uint64(0xFFFFFFFF)).astype(np.uint32), (c >> np.uint64(32)).astype(np.uint32)
        return mix32(np.uint32(seed) ^ mix32(lo ^ mix32(hi)))

    a = (word(c) >> np.uint32(5)).astype(np.float64)
    b = (word(c + np.uint64(1)) >> np.uint32(6)).astype(np.float64)
    return ((a * 67108864.0 + b) / 9007199254740992.0).reshape(n, d)


def lloyd(n, d, seed, num_lloyd, num_newton):
    x = initial_sample(n, seed, d)
    for _ in range(num_lloyd):
        x = centroids(x)
    energies = []
    if num_newton <= 0:
        return x, energies

    def evaluate(x):
        m = cell_moments(x)
        return m[:, 4].sum(), (-2.0 * m[:, 1:1 + d]).ravel()

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
            xt = xf + t * p
            if np.all((xt >= 0.0) & (xt <= 1.0)):
                Ft, gt = evaluate(xt.reshape(n, d))
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
    return xf.reshape(n, d), energies


# ---- CPU: the oracle pinned --------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [2, 3])
def test_oracle_partition_and_moments(d):
    x = np.random.default_rng(d).random((120, d))
    m = cell_moments(x)
    assert abs(m[:, 0].sum() - 1.0) < 1e-12
    np.testing.assert_allclose((m[:, :1] * x + m[:, 1:1 + d]).sum(axis=0), 0.5, atol=1e-12)
    # second moments add up to the cube's about each seed: sum_i int_{V_i} |y - c_i|^2 >= 0, and the CVT energy of a
    # lattice is the box's
    lat = lattice(4, d)
    ml = cell_moments(lat)
    np.testing.assert_allclose(ml[:, 0], 0.25 ** d, rtol=1e-12)
    np.testing.assert_allclose(ml[:, 1:1 + d], 0.0, atol=1e-15)
    np.testing.assert_allclose(ml[:, 4], 0.25 ** d * d * 0.25 ** 2 / 12, rtol=1e-10)


def test_oracle_boxes_on_uneven_lattice():
    xs = np.array([0.1, 0.3, 0.8])
    x = np.stack(np.meshgrid(xs, xs, xs, indexing="ij"), -1).reshape(-1, 3)
    walls = np.r_[0.0, (xs[:-1] + xs[1:]) / 2, 1.0]
    lo, hi = walls[:-1], walls[1:]
    g = centroids(x).reshape(3, 3, 3, 3)
    for a in range(3):
        for i in range(3):
            idx = [slice(None)] * 3
            idx[a] = i
            np.testing.assert_allclose(g[tuple(idx)][..., a], (lo[i] + hi[i]) / 2, atol=1e-14)


def test_oracle_duplicates():
    x = np.array([[0.2, 0.2, 0.2], [0.7, 0.7, 0.7], [0.2, 0.2, 0.2]])
    m = cell_moments(x)
    assert m[2, 0] == 0.0 and abs(m[:, 0].sum() - 1) < 1e-14
    assert np.array_equal(centroids(x)[2], x[2])


def test_initial_sample_restatement():
    a = initial_sample(1000, 12345, 3)
    assert a.shape == (1000, 3) and a.min() >= 0 and a.max() < 1
    assert abs(a.mean() - 0.5) < 0.02
    assert np.array_equal(a, initial_sample(1000, 12345, 3))
    assert not np.array_equal(a, initial_sample(1000, 12346, 3))
    # the 53 bits are all used: every value is a multiple of 2^-53 and not of 2^-32
    assert np.all((a * 2.0 ** 53) % 1 == 0) and np.any((a * 2.0 ** 32) % 1 != 0)


def test_lloyd_restatement_decreases_energy():
    x, e = lloyd(40, 2, 7, 2, 5)
    assert len(e) >= 2 and all(b <= a for a, b in zip(e, e[1:]))
    assert x.min() >= 0 and x.max() <= 1


def test_argument_errors():
    with pytest.raises(ValueError, match="Invalid scalar type"):
        pcu.voronoi_centroids_unit_cube(np.zeros((3, 3), dtype=np.int32))
    with pytest.raises(ValueError, match="Invalid shape"):
        pcu.voronoi_centroids_unit_cube(np.zeros((3, 2)))
    with pytest.raises(ValueError, match=r"Centers of voronoi diagram must lie in the unit cube \[0, 1\]\^3"):
        pcu.voronoi_centroids_unit_cube(np.array([[0.5, 0.5, 1.5]]))
    with pytest.raises(ValueError, match=r"Centers of voronoi diagram must lie in the unit cube \[0, 1\]\^3"):
        pcu.voronoi_centroids_unit_cube(np.array([[0.5, -1e-300, 0.5]]))
    with pytest.raises(ValueError, match=r"Centers of voronoi diagram must lie in the unit cube \[0, 1\]\^3"):
        pcu.voronoi_centroids_unit_cube(np.array([[0.5, np.nan, 0.5]]))
    with pytest.raises(ValueError, match="Invalid type"):
        pcu.voronoi_centroids_unit_cube([[0.5, 0.5, 0.5]])
    for f in (pcu.lloyd_2d, pcu.lloyd_3d):
        with pytest.raises(ValueError, match=r"n must be a positive integer. Got n = 0"):
            f(0)
        with pytest.raises(ValueError, match=r"n must be a positive integer. Got n = -3"):
            f(-3)


def test_empty_input():
    out = pcu.voronoi_centroids_unit_cube(np.zeros((0, 3), dtype=np.float32))
    assert out.shape == (0, 3) and out.dtype == np.float64


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _cases():
    rng = np.random.default_rng(5)
    lat = lattice(6, 3)
    cluster = np.concatenate([0.5 + 1e-3 * (rng.random((270, 3)) - 0.5), rng.random((30, 3))])
    corners = np.array([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], dtype=float)
    faces = np.concatenate([corners, [[0, 0.3, 0.6], [1, 0.5, 0.5], [0.2, 0, 1], [0.5, 0.5, 0], [0.7, 1, 0.1]],
                            rng.random((20, 3))])
    dup = np.concatenate([rng.random((30, 3)), rng.random((30, 3))[:10]])
    dup = np.concatenate([dup, dup[[3, 7, 3, 12]]])
    t = np.linspace(0.05, 0.95, 12)
    collinear = np.stack([t, t, t], 1)
    coplanar = np.c_[rng.random((25, 2)), np.full(25, 0.5)]
    return {
        "uniform": rng.random((300, 3)),
        "cluster": cluster,
        "lattice": lat,
        "lattice_jitter": np.clip(lat + 1e-12 * (rng.random(lat.shape) - 0.5), 0, 1),
        "faces_edges_corners": faces,
        "duplicates": dup,
        "n1": np.array([[0.1, 0.9, 0.3]]),
        "n2": np.array([[0.2, 0.2, 0.2], [0.9, 0.5, 0.1]]),
        "collinear": collinear,
        "coplanar": coplanar,
    }


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_cases()))
def test_centroids_match_oracle(name):
    x = _cases()[name]
    got = pcu.voronoi_centroids_unit_cube(x)
    assert got.dtype == np.float64 and got.shape == x.shape
    np.testing.assert_allclose(got, centroids(x), rtol=0, atol=1e-9)
    if name == "cluster":
        passes = pcu._lloyd.last_pass_counts
        assert passes[0] == len(x) and passes[1] > 0 and passes[2] > 0, passes
    if name == "n1":
        np.testing.assert_allclose(got, [[0.5, 0.5, 0.5]], atol=1e-15)
    if name == "duplicates":
        m = cell_moments(x)
        empty = m[:, 0] == 0
        assert empty.sum() >= 4 and np.array_equal(got[empty], x[empty])


@pytest.mark.gpu
def test_centroids_input_forms():
    import torch
    x = np.random.default_rng(9).random((200, 3))
    for dt in (np.float32, np.float64):
        xd = x.astype(dt)
        ref = centroids(xd.astype(np.float64))
        a = pcu.voronoi_centroids_unit_cube(xd)
        np.testing.assert_allclose(a, ref, atol=1e-9, rtol=0)
        b = pcu.voronoi_centroids_unit_cube(torch.from_numpy(xd).cuda())
        assert b.is_cuda and b.dtype == torch.float64
        assert np.array_equal(b.cpu().numpy(), a)
        c = pcu.voronoi_centroids_unit_cube(torch.from_numpy(xd))
        assert not c.is_cuda and c.dtype == torch.float64
        assert np.array_equal(c.numpy(), a)


def ball(rng, n, r, d=3):
    v = rng.normal(size=(n, d))
    v *= (r * rng.random(n) ** (1 / d) / np.linalg.norm(v, axis=1))[:, None]
    return 0.5 + v


@pytest.mark.gpu
def test_cluster_through_last_resort():
    """9e4 seeds in a ball of radius 0.01 among 1e4 uniform ones: the sparse seeds next to the ball have cells of
    hundreds of faces, bounded in turn by more bisectors than the last resort's first capacity has plane numbers
    (which are recycled), and the last resort certifies them."""
    rng = np.random.default_rng(21)
    x = np.concatenate([ball(rng, 90_000, 0.01), rng.random((10_000, 3))])
    g, m = pcu._lloyd._cell_moments(x)
    passes = pcu._lloyd.last_pass_counts
    assert passes[1] > 0 and passes[2] > 0, passes
    assert abs(m[:, 0].sum() - 1.0) < 1e-9
    np.testing.assert_allclose((m[:, :1] * x + m[:, 1:4]).sum(axis=0), 0.5, atol=1e-9)
    assert np.array_equal(pcu.voronoi_centroids_unit_cube(x), g)
    # the sparse seeds nearest the ball, and a few of the ball's own, against the oracle
    dist = np.linalg.norm(x[90_000:] - 0.5, axis=1)
    rows = np.r_[90_000 + np.argsort(dist)[:3], 0]
    ref = np.array([cell_moments_row(x, i) for i in rows])
    np.testing.assert_allclose(m[rows, 0], ref[:, 0], rtol=1e-9, atol=1e-15)
    gr = x[rows] + ref[:, 1:4] / ref[:, :1]
    np.testing.assert_allclose(g[rows], gr, atol=1e-9, rtol=0)


@pytest.mark.gpu
def test_cluster_2d_runs_every_pass():
    rng = np.random.default_rng(22)
    x = np.concatenate([ball(rng, 270, 0.02, 2), rng.random((30, 2))])
    g, m = pcu._lloyd._cell_moments(x)
    passes = pcu._lloyd.last_pass_counts
    assert passes[0] == len(x) and passes[1] > 0 and passes[2] > 0, passes
    np.testing.assert_allclose(m, cell_moments(x), atol=1e-12, rtol=0)
    np.testing.assert_allclose(g, centroids(x), atol=1e-9, rtol=0)


@pytest.mark.gpu
def test_centroids_million():
    x = np.random.default_rng(11).random((1_000_000, 3))
    a = pcu.voronoi_centroids_unit_cube(x)
    b = pcu.voronoi_centroids_unit_cube(x)
    assert np.array_equal(a, b)
    g, m = pcu._lloyd._cell_moments(x)
    assert np.array_equal(g, a)
    assert abs(m[:, 0].sum() - 1.0) < 1e-9
    np.testing.assert_allclose((m[:, :1] * x + m[:, 1:4]).sum(axis=0), 0.5, atol=1e-9)
    assert a.min() >= 0 and a.max() <= 1
    d, i = pcu.k_nearest_neighbors(a, x, 1)
    own = i == np.arange(len(x))
    if not own.all():   # a tie: the own seed is as near as the one returned
        rows = np.nonzero(~own)[0]
        dd = np.sqrt(((a[rows] - x[rows]) ** 2).sum(1))
        np.testing.assert_allclose(dd, d[rows], rtol=1e-12)
    assert own.mean() > 0.9999


@pytest.mark.gpu
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("num_newton", [0, 5])
def test_lloyd_matches_restatement(d, num_newton):
    f = pcu.lloyd_3d if d == 3 else pcu.lloyd_2d
    np.random.seed(123)
    got = f(200, 3, num_newton)
    np.random.seed(123)
    seed = int(np.random.randint(2 ** 31 - 1))
    ref, energies = lloyd(200, d, seed, 3, num_newton)
    assert got.shape == (200, d) and got.dtype == np.float64
    assert got.min() >= 0 and got.max() <= 1
    np.testing.assert_allclose(got, ref, atol=1e-8, rtol=0)
    e = pcu._lloyd.last_newton_energies
    if num_newton:
        assert len(e) == len(energies)
        np.testing.assert_allclose(e, energies, rtol=1e-10)
        assert all(b <= a for a, b in zip(e, e[1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("d", [2, 3])
def test_lloyd_no_iterations_is_initial_sample(d):
    f = pcu.lloyd_3d if d == 3 else pcu.lloyd_2d
    np.random.seed(4)
    got = f(500, 0, 0)
    np.random.seed(4)
    assert np.array_equal(got, initial_sample(500, int(np.random.randint(2 ** 31 - 1)), d))
    np.random.seed(4)
    assert np.array_equal(f(500, -1, -2), got)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [2, 3])
def test_lloyd_defaults_energy_and_bounds(d):
    f = pcu.lloyd_3d if d == 3 else pcu.lloyd_2d
    np.random.seed(8)
    a = f(3000)
    e = pcu._lloyd.last_newton_energies
    np.random.seed(8)
    b = f(3000)
    assert np.array_equal(a, b)
    assert a.shape == (3000, d) and a.min() >= 0 and a.max() <= 1
    assert len(e) >= 2 and all(y <= x for x, y in zip(e, e[1:]))
