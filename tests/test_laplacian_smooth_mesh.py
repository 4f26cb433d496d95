"""laplacian_smooth_mesh: the result of DESIGN.md §3 restated with scipy (sparse L and M, spsolve in fp64); the
restatement pinned to a literal dense transcription of the reference's loop (src/smooth.cpp:37-75, with libigl's
cotmatrix, massmatrix, doublearea and barycenter written out) on meshes of at most 50 vertices, to the properties of L
itself, and to unit total area after every cotan-mode step; the argument errors in the reference's order; on the GPU,
both modes at num_iters 1, 3 and 10 within 1e-9 of the bounding-box diagonal (float64) and 1 ulp (float32; the
float64 tolerance for coordinates within it of 0) of the restatement on a noisy icosphere, a subdivided twisted cube and a cleaned marching-cubes mesh, a 1.3 * 10^6-face noisy
icosphere, repeatability, the input forms and the RuntimeWarning of a capped solve."""
import numpy as np
import pytest

from meshes import noisy_icosphere, to_form, to_numpy
from test_mesh_geometry import corner_dot, face_area

DBL_EPS = np.finfo(np.float64).eps


# ---- the restatement ------------------------------------------------------------------------------------------------
def cot_laplacian(u, f):
    """(off-diagonal L as CSR, its diagonal): L_ij = sum of cot / 2 of the corners opposite edge ij, 0 for a face with
    dblA = 0; L_ii = -sum_j L_ij."""
    import scipy.sparse as sp
    n = len(u)
    q = [u[f[:, 0]], u[f[:, 1]], u[f[:, 2]]]
    A = face_area(*q)
    rows, cols, vals = [], [], []
    for k in range(3):
        with np.errstate(divide="ignore", invalid="ignore"):
            hc = np.where(A == 0, 0.0, 0.5 * (corner_dot(q[k], q[(k + 1) % 3], q[(k + 2) % 3]) / A))
        a, b = f[:, (k + 1) % 3], f[:, (k + 2) % 3]
        rows += [a, b]
        cols += [b, a]
        vals += [hc, hc]
    off = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n)).tocsr()
    off.setdiag(0.0)   # a repeated-corner face's self entries (always 0)
    off.eliminate_zeros()
    return off, -np.asarray(off.sum(axis=1)).ravel()


def mass(u, f, lone):
    A = face_area(u[f[:, 0]], u[f[:, 1]], u[f[:, 2]])
    m = np.zeros(len(u))
    np.add.at(m, f.ravel(), np.repeat(A / 6.0, 3))
    return np.where((m == 0) & lone, 1.0, m)


def rescale(u, f):
    q = [u[f[:, 0]], u[f[:, 1]], u[f[:, 2]]]
    A = face_area(*q)
    c = (A[:, None] * ((q[0] + q[1]) + q[2]) / 3.0).sum(0) / A.sum()
    return (u - c) / np.sqrt(0.5 * A.sum()) + c


def solve_cg(S, b, x0):
    """scipy's conjugate gradients, Jacobi-preconditioned, per column to |r| <= 1e-14 |b|: for meshes too large for
    spsolve's factorisation (minutes at 6.5 * 10^5 vertices)."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spl
    P = sp.diags(1.0 / S.diagonal())
    out = np.empty_like(b)
    for c in range(b.shape[1]):
        out[:, c], info = spl.cg(S, b[:, c], x0=x0[:, c], rtol=1e-14, atol=0.0, maxiter=100000, M=P)
        assert info == 0
    return out


def restate_smooth(v, f, num_iters, step_size=0.1, use_cotan_weights=False, trace=None, iterative=False):
    """(M - h L) u' = M u per step with scipy's spsolve (or, iterative, its CG), fp64, rounded once to v's dtype."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spl
    f = np.asarray(f, np.int64)
    u = v.astype(np.float64)
    if num_iters == 0:
        return v.copy()
    h = step_size * 1e-3 if use_cotan_weights else step_size
    off, diag = cot_laplacian(u, f)
    L = (off + sp.diags(diag)).tocsc()
    lone = np.diff(off.indptr) == 0
    for _ in range(num_iters):
        m = mass(u, f, lone) if use_cotan_weights else np.ones(len(u))
        M = sp.diags(m)
        S = (M - h * L).tocsc()
        u = solve_cg(S.tocsr(), M @ u, u) if iterative else spl.spsolve(S, M @ u)
        if use_cotan_weights:
            u = rescale(u, f)
        if trace is not None:
            trace.append(u.copy())
    return u.astype(v.dtype)


def literal_smooth(v, f, num_iters, step_size=0.1, use_cotan_weights=False):
    """src/smooth.cpp:37-75 with dense matrices and np.linalg.solve, in fp64; igl::cotmatrix (cot / 2 from the edge
    lengths, (l1^2 + l2^2 - l0^2) / dblA / 4), igl::massmatrix(BARYCENTRIC), igl::doublearea and igl::barycenter
    written out."""
    f = np.asarray(f, np.int64)
    n = len(v)
    if use_cotan_weights:
        step_size *= 1e-3

    def dbl_area(u):
        out = np.zeros(len(f))
        for i, (a, b, c) in enumerate(f):
            out[i] = np.linalg.norm(np.cross(u[b] - u[a], u[c] - u[a]))
        return out

    u = v.astype(np.float64)
    L = np.zeros((n, n))
    dblA = dbl_area(u)
    for i, face in enumerate(f):
        for k in range(3):
            a, b, c = face[k], face[(k + 1) % 3], face[(k + 2) % 3]
            l0, l1, l2 = (np.sum((u[b] - u[c]) ** 2), np.sum((u[a] - u[b]) ** 2), np.sum((u[a] - u[c]) ** 2))
            C = (l1 + l2 - l0) / dblA[i] / 4.0
            L[b, c] += C
            L[c, b] += C
            L[b, b] -= C
            L[c, c] -= C
    M = np.eye(n)
    for _ in range(num_iters):
        if use_cotan_weights:
            M = np.zeros((n, n))
            dA = dbl_area(u)
            for i, face in enumerate(f):
                for k in range(3):
                    M[face[k], face[k]] += dA[i] / 6.0
        u = np.linalg.solve(M - step_size * L, M @ u)
        if use_cotan_weights:
            dA = dbl_area(u)
            area = 0.5 * dA.sum()
            bc = np.array([u[face].mean(0) for face in f])
            centroid = np.zeros(3)
            for i in range(len(f)):
                centroid += 0.5 * dA[i] / area * bc[i]
            u = (u - centroid) / np.sqrt(area) + centroid
    return u


# ---- meshes ---------------------------------------------------------------------------------------------------------
def twisted_cube(sub):
    """A unit cube's 12 triangles, loop-free midpoint subdivision `sub` times, twisted about z."""
    v = np.array([[x, y, z] for z in (0, 1) for y in (0, 1) for x in (0, 1)], np.float64) - 0.5
    f = np.array([[0, 2, 1], [1, 2, 3], [4, 5, 6], [5, 7, 6], [0, 1, 4], [1, 5, 4], [2, 6, 3], [3, 6, 7], [0, 4, 2],
                  [2, 4, 6], [1, 3, 5], [3, 7, 5]], np.int64)
    for _ in range(sub):
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        uk, inv = np.unique(np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1]), return_inverse=True)
        mid = len(v) + inv.reshape(3, -1).T
        v = np.concatenate([v, 0.5 * (v[uk >> 32] + v[uk & 0xFFFFFFFF])])
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        f = np.concatenate([np.stack([a, mid[:, 0], mid[:, 2]], 1), np.stack([b, mid[:, 1], mid[:, 0]], 1),
                            np.stack([c, mid[:, 2], mid[:, 1]], 1), mid])
    t = 1.2 * v[:, 2]
    x, y = v[:, 0] * np.cos(t) - v[:, 1] * np.sin(t), v[:, 0] * np.sin(t) + v[:, 1] * np.cos(t)
    return np.stack([x, y, v[:, 2]], 1), f


def planar(n, seed):
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.random((n, 2)), [[0, 0], [1, 0], [0, 1], [1, 1]]])
    tri = Delaunay(p)
    boundary = np.zeros(len(p), bool)
    boundary[tri.convex_hull.ravel()] = True
    return np.concatenate([p, np.zeros((len(p), 1))], 1), tri.simplices.astype(np.int64), boundary


# ---- the CPU --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cotan", [False, True])
def test_restatement_is_the_reference_loop(cotan):
    for v, f in (noisy_icosphere(1, 1), twisted_cube(1), noisy_icosphere(0, 2, 0.2)):
        assert len(v) <= 50
        diag = np.linalg.norm(v.max(0) - v.min(0))
        for k in (1, 3):
            got, want = restate_smooth(v, f, k, 0.1, cotan), literal_smooth(v, f, k, 0.1, cotan)
            assert np.abs(got - want).max() <= 1e-11 * diag, (cotan, k, np.abs(got - want).max())
        got, want = restate_smooth(v, f, 2, 0.7, cotan), literal_smooth(v, f, 2, 0.7, cotan)
        assert np.abs(got - want).max() <= 1e-11 * diag


def test_laplacian_properties():
    for v, f in (noisy_icosphere(3, 3), twisted_cube(2)):
        off, diag = cot_laplacian(v, f)
        L = (off + __import__("scipy.sparse", fromlist=["diags"]).diags(diag)).toarray()
        assert np.array_equal(L, L.T)
        assert np.abs(L @ np.ones(len(v))).max() <= 64 * DBL_EPS * np.abs(L).max()
    v, f, boundary = planar(300, 4)
    off, diag = cot_laplacian(v, f)
    L = off.toarray() + np.diag(diag)
    for x in (v[:, 0], v[:, 1], 2.0 * v[:, 0] - 3.0 * v[:, 1] + 0.5):
        r = L @ x
        assert np.abs(r[~boundary]).max() <= 1e-9 * np.abs(L).max(), np.abs(r[~boundary]).max()
        assert np.abs(r[boundary]).max() > 1e-6                           # the boundary rows are not harmonic


def test_cotan_mode_unit_area():
    for v, f in (noisy_icosphere(3, 5), twisted_cube(2)):
        trace = []
        restate_smooth(v, f, 4, 0.1, True, trace)
        for u in trace:
            A = face_area(u[f[:, 0]], u[f[:, 1]], u[f[:, 2]])
            assert abs(0.5 * A.sum() - 1.0) <= 1e-12


def test_zero_and_identity_rows():
    v, f = noisy_icosphere(1, 6)
    v = np.concatenate([v, [[5.0, 5.0, 5.0]]])                             # an isolated vertex stays put
    for cotan in (False, True):
        u = restate_smooth(v, f, 3, 0.1, cotan)
        assert np.array_equal(u[-1], v[-1]) or cotan                      # cotan mode moves it with the rescale
    assert np.array_equal(restate_smooth(v, f, 0), v)


def test_argument_errors(pcu):
    v = np.zeros((4, 3))
    f = np.array([[0, 1, 2]], np.int64)
    sm = pcu.laplacian_smooth_mesh
    cases = [
        ((v.astype(np.int32), f, 1), "Invalid scalar type (int32) for argument 'v'"),
        ((v, f.astype(np.uint32), 1), "for argument 'f'. Expected one of ['int32', 'int64']"),
        ((v[:0], f, 1), "Invalid input mesh with zero elements"),
        ((v, f[:0], 1), "Invalid input mesh with zero elements"),
        ((v[:, :2], f, 1), "Only 3D inputs are supported"),
        ((v, f[:, :2], 1), "Only 3D inputs are supported"),
        ((list(v), f, 1), "Invalid type for v"),
        ((v, f, -1), "Invalid value for argument num_iters in smooth_mesh_laplacian. Must be a positive integer or 0."),
        ((v[:0], f, -1), "Invalid input mesh with zero elements"),                # the mesh checks come first
        ((v.astype(np.int32), f.astype(np.float32), -1), "for argument 'v'"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError) as e:
            sm(*args)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        sm(v, f, 1, 0.1, False, None)                                           # device= is keyword only
    out = sm(v, f, 0)
    assert out is not v and np.array_equal(out, v)                            # num_iters = 0: a copy


# ---- the GPU --------------------------------------------------------------------------------------------------------
def check_close(got, want, v):
    got = to_numpy(got)
    assert got.dtype == want.dtype and got.shape == want.shape
    tol = 1e-9 * np.linalg.norm(v.astype(np.float64).max(0) - v.astype(np.float64).min(0))
    diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    if want.dtype == np.float64:
        assert diff.max() <= tol, (diff.max(), tol)
    else:   # 1 ulp, or the float64 tolerance where a coordinate is so close to 0 that its ulp is finer
        assert np.all(diff <= np.maximum(np.spacing(np.abs(want)).astype(np.float64), tol)), diff.max()


def cleaned_mc_mesh(pcu):
    from test_connected_components import noisy_mc_mesh
    v, f = noisy_mc_mesh(pcu, 48, 7)
    cv, nv, cf, nf = pcu.connected_components(v, f)
    big = np.argsort(nf)[-20:]
    mask = np.isin(cv, big)
    vk, fk = pcu.remove_mesh_vertices(v, f, mask[: len(v)])
    return pcu.remove_unreferenced_mesh_vertices(vk, fk)[:2]


@pytest.mark.gpu
@pytest.mark.parametrize("cotan", [False, True])
@pytest.mark.parametrize("vdt", [np.float64, np.float32])
def test_smooth_meshes(pcu, cotan, vdt):
    meshes = [noisy_icosphere(4, 7), twisted_cube(3), cleaned_mc_mesh(pcu)]
    for v, f in meshes:
        v = v.astype(vdt)
        for k in (1, 3, 10):
            for fdt in (np.int64, np.int32):
                check_close(pcu.laplacian_smooth_mesh(v, f.astype(fdt), k, 0.1, cotan), restate_smooth(v, f, k, 0.1, cotan), v)


@pytest.mark.gpu
@pytest.mark.parametrize("cotan", [False, True])
def test_large_icosphere(pcu, cotan):
    v, f = noisy_icosphere(8, 8, 0.01)
    got = pcu.laplacian_smooth_mesh(v, f, 2, 0.1, cotan)
    check_close(got, restate_smooth(v, f, 2, 0.1, cotan, iterative=True), v)
    again = pcu.laplacian_smooth_mesh(v, f, 2, 0.1, cotan)
    assert np.array_equal(got.view(np.uint8), again.view(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_forms_and_repeatability(pcu, form):
    import torch
    v, f = noisy_icosphere(3, 9)
    v = v.astype(np.float32)
    kind = np.ndarray if form == "numpy" else torch.Tensor
    for cotan in (False, True):
        a = pcu.laplacian_smooth_mesh(to_form(form, v), to_form(form, f), 3, 0.1, cotan)
        b = pcu.laplacian_smooth_mesh(to_form(form, v), to_form(form, f), 3, 0.1, cotan)
        assert isinstance(a, kind) and (form == "numpy" or a.is_cuda == (form == "cuda"))
        assert np.array_equal(to_numpy(a).view(np.uint8), to_numpy(b).view(np.uint8))
        check_close(a, restate_smooth(v, f, 3, 0.1, cotan), v)
    z = pcu.laplacian_smooth_mesh(to_form(form, v), to_form(form, f), 0, use_cotan_weights=True)
    assert isinstance(z, kind) and np.array_equal(to_numpy(z), v)


@pytest.mark.gpu
def test_isolated_vertex_and_shapes(pcu):
    v, f = noisy_icosphere(2, 10)
    v = np.concatenate([v, [[5.0, 5.0, 5.0]]])
    for cotan in (False, True):
        check_close(pcu.laplacian_smooth_mesh(v, f, 3, 0.1, cotan), restate_smooth(v, f, 3, 0.1, cotan), v)
    one = pcu.laplacian_smooth_mesh(np.array([[1.0, 2.0, 3.0]]), np.array([[0, 0, 0]]), 2)
    assert one.shape == (3,) and np.array_equal(one, [1.0, 2.0, 3.0])


@pytest.mark.gpu
def test_errors_on_the_device(pcu):
    v, f = noisy_icosphere(1, 11)
    with pytest.raises(ValueError, match="Invalid face indices: 1 faces have a corner outside"):
        pcu.laplacian_smooth_mesh(v, np.concatenate([f, [[0, 1, len(v)]]]), 1)
    bad = v.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError, match="not finite"):
        pcu.laplacian_smooth_mesh(bad, f, 1)
    with pytest.raises(ValueError, match="zero total area"):
        pcu.laplacian_smooth_mesh(np.zeros_like(v), f, 1, use_cotan_weights=True)


@pytest.mark.gpu
def test_capped_solve_warns(pcu, monkeypatch):
    from pcu_b200 import _mesh_geometry
    v, f = noisy_icosphere(4, 12)
    monkeypatch.setattr(_mesh_geometry, "_CG_MAX_ITERS", 2)
    with pytest.warns(RuntimeWarning, match="stopped after 2 conjugate-gradient iterations at a relative residual of"):
        out = pcu.laplacian_smooth_mesh(v, f, 2)
    assert out.shape == v.shape and np.isfinite(out).all()
    with pytest.warns(RuntimeWarning):
        _, iters = _mesh_geometry._smooth(v, f, 2, 0.1, False, None)
    assert len(iters) == 2 and all(k <= 2 for k in iters)
