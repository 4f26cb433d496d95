"""closest_points_on_mesh: the definition of DESIGN.md §3 (point-to-mesh distance) restated with array operations, the
GPU results against it bit for bit, ties, the reference's own consistency check, full size, input forms and errors."""
import inspect

import numpy as np
import pytest

from meshes import icosphere
from test_mesh_sampling import MESHES, degenerate_mesh, flat_grid, spanning_mesh  # noqa: F401

FDTYPES = [np.int32, np.int64, np.uint32, np.uint64]


# ---- the restatement: one elementwise op per step (numpy arrays, or torch CUDA tensors for the full-size checks) -----
REGIONS = ["A", "B", "AB", "C", "AC", "BC", "interior", "edges"]


def _where(x):
    if type(x).__module__.startswith("torch"):
        import torch
        return torch.where
    return np.where


def _dot(u, w):
    return (u[0] * w[0] + u[1] * w[1]) + u[2] * w[2]      # ((ux wx + uy wy) + uz wz), each op rounded


def _sub3(u, w):
    return [u[k] - w[k] for k in range(3)]


def _d2(p, c):
    dx, dy, dz = p[0] - c[0], p[1] - c[1], p[2] - c[2]
    return (dx * dx + dy * dy) + dz * dz


def _segment(p, x, y, where, zero):
    """d^2 and t of the closest point of segment [x, y] (x at t = 0, y at t = 1, else x + t e)."""
    e = _sub3(y, x)
    ll = _dot(e, e)
    t = _dot(_sub3(p, x), e) / ll
    t = where(t < 0, zero, where(t > 1, zero + 1, t))
    t = where(ll > 0, t, zero)
    mid = [x[k] + t * e[k] for k in range(3)]
    c = [where(t == 0, x[k] + zero, where(t == 1, y[k] + zero, mid[k])) for k in range(3)]
    return _d2(p, c), t


def face_hits(p, a, b, c, degenerate):
    """Per (query, face): d^2, (b0, b1, b2) and the region index (REGIONS).  p: 3 arrays (Q, 1); a, b, c: 3 arrays
    (1, F) each; degenerate: (1, F) bool.  Every operation is a separate elementwise op in the input precision."""
    where = _where(p[0])
    zero = 0.0 * abs(p[0] + a[0])       # (Q, F) zeros (+0) of the working type
    one = zero + 1
    ab, ac = _sub3(b, a), _sub3(c, a)
    ap, bp, cp = _sub3(p, a), _sub3(p, b), _sub3(p, c)
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    s = (va + vb) + vc
    vi, wi = vb / s, vc / s

    def ratio(n, d):
        return where(d > 0, n / d, zero)

    cands = []
    cands.append(((d1 <= 0) & (d2 <= 0), _d2(p, a) + zero, (one, zero, zero)))
    cands.append(((d3 >= 0) & (d4 <= d3), _d2(p, b) + zero, (zero, one, zero)))
    v = ratio(d1, d1 - d3)
    cands.append(((vc <= 0) & (d1 >= 0) & (d3 <= 0), _d2(p, [a[k] + v * ab[k] for k in range(3)]), (one - v, v, zero)))
    cands.append(((d6 >= 0) & (d5 <= d6), _d2(p, c) + zero, (zero, zero, one)))
    w = ratio(d2, d2 - d6)
    cands.append(((vb <= 0) & (d2 >= 0) & (d6 <= 0), _d2(p, [a[k] + w * ac[k] for k in range(3)]), (one - w, zero, w)))
    w = ratio(e43, e43 + e56)
    bc_ = _sub3(c, b)
    cands.append(((va <= 0) & (e43 >= 0) & (e56 >= 0), _d2(p, [b[k] + w * bc_[k] for k in range(3)]), (zero, one - w, w)))
    inside = (s > 0) & (vi >= 0) & (wi >= 0) & ((vi + wi) <= 1)
    cands.append((inside, _d2(p, [(a[k] + ab[k] * vi) + ac[k] * wi for k in range(3)]), ((one - vi) - wi, vi, wi)))
    # the union of the edges AB, BC, CA, the first on ties
    e_d2, t = _segment(p, a, b, where, zero)
    e_bc = [one - t, t, zero]
    for (x, y, slot) in ((b, c, (None, 0, 1)), (c, a, (1, None, 0))):
        d2s, t = _segment(p, x, y, where, zero)
        better = d2s < e_d2
        e_d2 = where(better, d2s, e_d2)
        new = [zero if slot[k] is None else (one - t if slot[k] == 0 else t) for k in range(3)]
        e_bc = [where(better, new[k], e_bc[k]) for k in range(3)]
    out_d2, out_bc, region = e_d2, list(e_bc), (zero != zero) * 0 + 7
    taken = (zero != zero) | degenerate       # degenerate faces keep the edges; the others take the first region that holds
    for r, (cond, cd2, cbc) in enumerate(cands):
        use = cond & ~taken
        out_d2 = where(use, cd2, out_d2)
        out_bc = [where(use, cbc[k], out_bc[k]) for k in range(3)]
        region = where(use, r + 0 * region, region)
        taken = taken | cond
    return out_d2, out_bc, region


def face_degenerate(a, b, c):
    """D = (e1.e1)(e2.e2) - (e1.e2)^2 not positive, e1 = b - a, e2 = c - a (per face, in the input precision)."""
    e1, e2 = _sub3(b, a), _sub3(c, a)
    D = _dot(e1, e1) * _dot(e2, e2) - _dot(e1, e2) * _dot(e1, e2)
    return ~(D > 0)


def restate(p, v, f, chunk=64):
    """(d, fi, bc) of the definition: the lexicographic minimum of (d^2, face index) over all faces.  numpy arrays, or
    torch CUDA tensors (p, v; f as int64)."""
    where = _where(p)
    is_torch = type(p).__module__.startswith("torch")
    xp = __import__("torch") if is_torch else np
    fi64 = f.long() if is_torch else f.astype(np.int64)
    A, B, C = (v[fi64[:, k]] for k in range(3))
    a = [A[None, :, k] for k in range(3)]
    b = [B[None, :, k] for k in range(3)]
    c = [C[None, :, k] for k in range(3)]
    degenerate = face_degenerate(a, b, c)
    ds, fis, bcs = [], [], []
    for s in range(0, p.shape[0], chunk):
        q = p[s:s + chunk]
        pp = [q[:, None, k] for k in range(3)]
        if is_torch:
            d2, bc, _ = face_hits(pp, a, b, c, degenerate)
        else:
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                d2, bc, _ = face_hits(pp, a, b, c, degenerate)
        key = where(d2 != d2, d2 * 0 + float("inf"), d2)           # a NaN d^2 is never chosen
        best = key.min(1, keepdims=True) if not is_torch else key.min(1, keepdim=True).values
        j = (key == best).int().argmax(1) if is_torch else np.argmax(key == best, axis=1)
        rows = xp.arange(q.shape[0], device=q.device) if is_torch else np.arange(q.shape[0])
        ds.append(xp.sqrt(best[:, 0]))
        fis.append(j)
        bcs.append(xp.stack([x[rows, j] for x in bc], 1))
    cat = xp.cat if is_torch else np.concatenate
    return cat(ds), cat(fis), cat(bcs)


def one_face(p, a, b, c, dtype=np.float64):
    """(d, bc, region name) of the definition for one query and one triangle."""
    P = [np.array([[x]], dtype=dtype) for x in p]
    Aa, Bb, Cc = ([np.array([[x]], dtype=dtype) for x in q] for q in (a, b, c))
    with np.errstate(divide="ignore", invalid="ignore"):
        d2, bc, region = face_hits(P, Aa, Bb, Cc, face_degenerate(Aa, Bb, Cc))
    return float(np.sqrt(d2[0, 0])), [float(x[0, 0]) for x in bc], REGIONS[int(region[0, 0])]


# ---- an independent formulation (fp64): plane projection when it falls inside, else the nearest edge ---------------
def independent(p, a, b, c):
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(-1)
    h = ((p - a) * n).sum(-1) / nn
    q = p - h[:, None] * n

    def side(x, y):
        return (np.cross(y - x, q - x) * n).sum(-1)

    inside = (side(a, b) >= 0) & (side(b, c) >= 0) & (side(c, a) >= 0)

    def seg(x, y):
        e = y - x
        t = np.clip(((p - x) * e).sum(-1) / (e * e).sum(-1), 0.0, 1.0)
        return np.linalg.norm(p - (x + t[:, None] * e), axis=-1)

    return np.where(inside, np.abs(h) * np.sqrt(nn), np.minimum(np.minimum(seg(a, b), seg(b, c)), seg(c, a)))


# ---- queries -------------------------------------------------------------------------------------------------------
def queries(v, f, n, seed):
    """n near-surface queries (points on random faces plus noise), n uniform in the box twice the mesh's, n far away."""
    rng = np.random.default_rng(seed)
    v64 = v.astype(np.float64)
    f64 = f.astype(np.int64)
    lo, hi = v64.min(0), v64.max(0)
    scale = float((hi - lo).max()) or 1.0
    fi = rng.integers(0, len(f64), n)
    r = rng.random((n, 2))
    s = np.sqrt(r[:, :1])
    bc = np.concatenate([1 - s, s * (1 - r[:, 1:]), s * r[:, 1:]], 1)
    near = (v64[f64[fi]] * bc[:, :, None]).sum(1) + 0.01 * scale * rng.standard_normal((n, 3))
    centre, half = (lo + hi) / 2, np.maximum(hi - lo, 1e-3 * scale)
    box = centre + (rng.random((n, 3)) - 0.5) * 2 * half
    far = centre + 1e3 * scale * rng.standard_normal((n, 3))
    return np.concatenate([near, box, far]).astype(v.dtype)


def assert_bits(got, ref, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.dtype == ref.dtype and got.shape == ref.shape, what
    g, r = got.view(np.uint8).reshape(len(got), -1), ref.view(np.uint8).reshape(len(ref), -1)
    assert np.array_equal(g, r), "%s: %d rows differ" % (what, int((g != r).any(1).sum()))


# ---- CPU: interface, arguments, the definition -----------------------------------------------------------------------
def test_signature(pcu):
    ps = list(inspect.signature(pcu.closest_points_on_mesh).parameters.values())
    assert [p.name for p in ps] == ["p", "v", "f", "device"]
    assert ps[3].kind == inspect.Parameter.KEYWORD_ONLY and ps[3].default is None
    assert "closest_points_on_mesh" in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    cp = pcu.closest_points_on_mesh
    v, f = icosphere(1)
    p = np.zeros((4, 3))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'p'"):
        cp(p.astype(np.int32), v, f)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'v'. Expected it to match argument "
                                         r"'p' which is of type float64."):
        cp(p, v.astype(np.float32), f)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'f'"):
        cp(p, v, f.astype(np.float64))
    with pytest.raises(ValueError, match="Only 3D inputs are supported: v must have shape"):
        cp(p[:, :2], v, f)
    with pytest.raises(ValueError, match="Only 3D inputs are supported: v must have shape"):
        cp(p[0], v, f)
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        cp(p, v[:0], f)
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        cp(p, v, f[:0])
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        cp(p, v[:, :2], f)
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        cp(p, v, f[:, :2])
    with pytest.raises(ValueError, match="NumPy array"):
        cp(p.tolist(), v, f)


def test_no_queries_return_empty_outputs_without_a_launch(pcu):
    import torch
    v, f = icosphere(1, dtype=np.float32)
    before = pcu.launch_count()
    for fdt in FDTYPES:
        d, fi, bc = pcu.closest_points_on_mesh(np.zeros((0, 3), np.float32), v, f.astype(fdt))
        assert d.shape == (0,) and d.dtype == np.float32 and fi.shape == (0,) and fi.dtype == fdt
        assert bc.shape == (0, 3) and bc.dtype == np.float32
    d, fi, bc = pcu.closest_points_on_mesh(torch.zeros((0, 3), dtype=torch.float64), torch.from_numpy(v.astype(np.float64)),
                                           torch.from_numpy(f))
    assert isinstance(d, torch.Tensor) and d.dtype == torch.float64 and fi.dtype == torch.int64 and bc.shape == (0, 3)
    assert pcu.launch_count() == before


# Every region of the unit right triangle a = 0, b = x, c = y, hand-computed.
TRI = ([0, 0, 0], [1, 0, 0], [0, 1, 0])
HAND = [
    ((-1, -1, 0), np.sqrt(2), [1, 0, 0], "A"),
    ((2, -1, 0), np.sqrt(2), [0, 1, 0], "B"),
    ((0.25, -2, 0), 2.0, [0.75, 0.25, 0], "AB"),
    ((-1, 2, 0), np.sqrt(2), [0, 0, 1], "C"),
    ((-3, 0.5, 0), 3.0, [0.5, 0, 0.5], "AC"),
    ((1, 1, 0), np.sqrt(0.5), [0, 0.5, 0.5], "BC"),
    ((0.25, 0.5, 2), 2.0, [0.25, 0.25, 0.5], "interior"),
]


@pytest.mark.parametrize("case", range(len(HAND)))
def test_hand_computed_regions(case):
    p, d, bc, region = HAND[case]
    got_d, got_bc, got_region = one_face(p, *TRI)
    assert got_region == region
    assert got_d == pytest.approx(d, rel=1e-15)
    assert got_bc == pytest.approx(bc, abs=1e-15)


def test_degenerate_faces_are_their_edges():
    # a segment [0, 2] on the x axis written as a triangle with a repeated corner, and as three collinear corners
    d, bc, region = one_face((1.5, 1, 0), (0, 0, 0), (2, 0, 0), (2, 0, 0))
    assert region == "edges" and d == 1.0 and bc == [0.25, 0.75, 0.0]
    d, bc, region = one_face((3, 0, 4), (0, 0, 0), (1, 0, 0), (2, 0, 0))     # beyond c: the corner c (edge BC, t = 1)
    assert region == "edges" and d == pytest.approx(np.sqrt(17.0)) and bc == [0.0, 0.0, 1.0]
    # a point: every edge has zero length, so the closest point is the corner itself
    d, bc, region = one_face((1, 2, 2), (1, 1, 1), (1, 1, 1), (1, 1, 1))
    assert region == "edges" and d == pytest.approx(np.sqrt(2.0)) and bc == [1.0, 0.0, 0.0]


def test_vertex_regions_return_the_corner_bit_for_bit():
    a, b, c = [0.1, 0.7, -0.3], [1.3, 0.2, 0.4], [-0.2, 1.9, 0.6]
    for corner, name, bc in ((a, "A", [1, 0, 0]), (b, "B", [0, 1, 0]), (c, "C", [0, 0, 1])):
        centre = (np.array(a) + b + c) / 3
        p = np.array(corner) + 5 * (np.array(corner) - centre)
        d, got_bc, region = one_face(p, a, b, c)
        assert region == name and got_bc == bc
        assert d == np.sqrt(_d2([np.float64(x) for x in p], [np.float64(x) for x in corner]))


def test_restatement_agrees_with_an_independent_formulation():
    rng = np.random.default_rng(17)
    n = 20000
    a, b, c = (rng.standard_normal((n, 3)) for _ in range(3))
    p = 2 * rng.standard_normal((n, 3))
    cols = [[x[:, k] for k in range(3)] for x in (p, a, b, c)]        # query i against triangle i
    with np.errstate(divide="ignore", invalid="ignore"):
        d2, _, region = face_hits(*cols, face_degenerate(*cols[1:]))
    got = np.sqrt(d2)
    ref = independent(p, a, b, c)
    scale = np.abs(np.concatenate([a, b, c, p])).max()
    assert np.abs(got - ref).max() <= 1e-12 * scale
    assert set(np.unique(region)) >= set(range(7))          # every region was exercised


# ---- GPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_matches_the_definition_bit_for_bit(pcu, vdtype):
    for name, make in MESHES.items():
        v, f = make(vdtype)
        p = queries(v, f, 1000, 3)
        ref = restate(p, v, f)
        for fdt in FDTYPES:
            d, fi, bc = pcu.closest_points_on_mesh(p, v, f.astype(fdt))
            assert fi.dtype == fdt, name
            assert_bits(d, ref[0], "%s d %s" % (name, fdt.__name__))
            assert np.array_equal(fi.astype(np.int64), ref[1]), "%s fi %s" % (name, fdt.__name__)
            assert_bits(bc, ref[2], "%s bc %s" % (name, fdt.__name__))


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_ties_take_the_lowest_face(pcu, vdtype):
    v, f = flat_grid(8, vdtype)
    g = np.arange(0, 8.5, 0.5) / 8                 # every vertex and every edge midpoint of the grid
    xy = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    diag = (xy[:-1] + xy[1:]) / 2
    pts = np.concatenate([xy, diag])
    p = np.concatenate([np.concatenate([pts, np.zeros((len(pts), 1))], 1),
                        np.concatenate([pts, np.full((len(pts), 1), 0.5)], 1)]).astype(vdtype)
    d, fi, bc = pcu.closest_points_on_mesh(p, v, f)
    ref = restate(p, v, f)
    assert_bits(d, ref[0], "grid d")
    assert np.array_equal(fi, ref[1]) and np.array_equal(bc, ref[2])
    # the centre of an icosphere: every face is nearly equidistant, nothing can be pruned
    v, f = icosphere(4, 0.0, 0, vdtype)
    p = np.zeros((1, 3), vdtype)
    d, fi, bc = pcu.closest_points_on_mesh(p, v, f)
    ref = restate(p, v, f)
    assert_bits(d, ref[0], "centre d")
    assert np.array_equal(fi, ref[1]) and np.array_equal(bc, ref[2])
    # a face list concatenated with itself: the first copy always wins
    v, f = icosphere(3, 0.01, 1, vdtype)
    p = queries(v, f, 1000, 9)
    one = pcu.closest_points_on_mesh(p, v, f)
    two = pcu.closest_points_on_mesh(p, v, np.concatenate([f, f]))
    assert (two[1] < len(f)).all()
    for x, y in zip(one, two):
        assert np.array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_the_reference_consistency_check(pcu, vdtype):
    # the reference's test_examples.py::test_closest_points_on_mesh: the point the coordinates name is d away from p
    tol = 1e-6 if vdtype == np.float32 else 1e-12
    for name, make in MESHES.items():
        v, f = make(vdtype)
        p = queries(v, f, 2000, 5)[:4000]                 # near-surface and box queries
        d, fi, bc = pcu.closest_points_on_mesh(p, v, f)
        x = (v[f[fi]].astype(np.float64) * bc[:, :, None].astype(np.float64)).sum(1)
        scale = np.abs(np.concatenate([v, p])).max()
        assert np.abs(np.linalg.norm(p.astype(np.float64) - x, axis=-1) - d).max() <= tol * scale, name


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_full_size(pcu, vdtype):
    import torch
    v, f = icosphere(8, 1e-4, 5, vdtype)                 # 1 310 720 faces
    f = f.astype(np.int32)
    rng = np.random.default_rng(8)
    n = 10 ** 6
    fi = rng.integers(0, len(f), n)
    r = rng.random((n, 2))
    s = np.sqrt(r[:, :1])
    bc = np.concatenate([1 - s, s * (1 - r[:, 1:]), s * r[:, 1:]], 1)
    p = ((v.astype(np.float64)[f[fi]] * bc[:, :, None]).sum(1) + 1e-3 * rng.standard_normal((n, 3))).astype(vdtype)
    pt, vt, ft = (torch.from_numpy(x).cuda() for x in (p, v, f))
    d, fi, bc = pcu.closest_points_on_mesh(pt, vt, ft)
    again = pcu.closest_points_on_mesh(pt, vt, ft)
    assert d.is_cuda and fi.dtype == torch.int32 and bc.dtype == pt.dtype
    for x, y in zip((d, fi, bc), again):
        assert torch.equal(x, y)
    rows = torch.from_numpy(rng.choice(n, 1000, replace=False)).cuda()
    ref = restate(pt[rows], vt, ft, chunk=4)
    assert torch.equal(d[rows], ref[0])
    assert torch.equal(fi[rows].long(), ref[1].long())
    assert torch.equal(bc[rows], ref[2])


@pytest.mark.gpu
def test_input_forms_and_device(pcu):
    import torch
    v, f = icosphere(3, 0.02, 7, np.float32)
    p = queries(v, f, 500, 1)
    a = pcu.closest_points_on_mesh(p, v, f)
    assert all(isinstance(x, np.ndarray) for x in a) and a[1].dtype == np.int64
    tc = pcu.closest_points_on_mesh(*(torch.from_numpy(x).cuda() for x in (p, v, f)))
    assert all(t.is_cuda for t in tc) and tc[1].dtype == torch.int64 and tc[0].dtype == torch.float32
    cpu = pcu.closest_points_on_mesh(*(torch.from_numpy(x) for x in (p, v, f)))
    assert all(isinstance(t, torch.Tensor) and not t.is_cuda for t in cpu)
    dev = pcu.closest_points_on_mesh(p, v, f, device="cuda:0")
    for i in range(3):
        assert np.array_equal(tc[i].cpu().numpy(), a[i]) and np.array_equal(cpu[i].numpy(), a[i])
        assert np.array_equal(dev[i], a[i])


@pytest.mark.gpu
def test_bad_indices_raise_without_a_fault(pcu):
    v, f = icosphere(2)
    p = queries(v, f, 100, 2)
    cases = []
    g = f.astype(np.uint64)
    g[[3, 7], 1] = len(v)
    g[9, 2] = 2 ** 63 + 5
    cases.append((g, 3))
    g = f.astype(np.int32)
    g[[0, 1], 0] = -1
    cases.append((g, 2))
    g = f.astype(np.int64)
    g[5, 2] = len(v) + 100
    cases.append((g, 1))
    for g, count in cases:
        with pytest.raises(ValueError, match=r"Invalid face indices: %d faces have a corner outside \[0, #v\)" % count):
            pcu.closest_points_on_mesh(p, v, g)
    d, fi, bc = pcu.closest_points_on_mesh(p, v, f)      # the device is fine afterwards
    assert np.array_equal(fi, restate(p, v, f)[1])
