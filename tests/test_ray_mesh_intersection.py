"""ray_mesh_intersection and RayMeshIntersector: the definition of DESIGN.md §3 (ray casting) restated with array
operations and checked against closed forms and for watertightness; on the GPU, both forms bit for bit against the
restatement, the reference's own check, watertightness, scale, precision, the handle, edge cases and full size."""
import inspect

import numpy as np
import pytest

from meshes import icosphere
from test_closest_points import FDTYPES, assert_bits
from test_winding_numbers import ALL_MESHES

F32 = np.float32


# ---- the restatement: fp32, one elementwise op per step (numpy arrays, or torch CUDA tensors at full size) -----------
def _xp(x):
    if type(x).__module__.startswith("torch"):
        import torch
        return torch
    return np


def _pick(xp, a, k):
    """a[..., k[i]] for every ray i (a: (rays, faces, 3), k: (rays,))."""
    idx = k.reshape(-1, 1, 1).expand(-1, a.shape[1], 1) if xp is not np else np.broadcast_to(k.reshape(-1, 1, 1), a.shape[:2] + (1,))
    return (xp.take_along_dim if xp is not np else np.take_along_axis)(a, idx, 2)[..., 0]


def restate(o, d, v, f, near=0.0, far=np.inf, chunk=128):
    """(fid as int64 with -1 on a miss, b1, b2, t) as float32, and the fp64 (1 - b1) - b2, for rays (o_i, d_i) against
    (v, f): numpy arrays, or torch CUDA tensors (f as int64)."""
    xp = _xp(d)
    if xp is np:
        o, d, v = (np.asarray(x, np.float64).astype(F32) for x in (o, d, v))
        fi = np.asarray(f).astype(np.int64)
        f64 = np.float64
    else:
        o, d, v, fi = o.float(), d.float(), v.float(), f.long()
        f64 = xp.float64
    o = o.reshape(-1, 3)
    if o.shape[0] == 1:
        o = o.expand(d.shape[0], 3) if xp is not np else np.broadcast_to(o, d.shape)
    near, far = float(F32(near)), float(F32(far))
    finite = lambda x: xp.isfinite(x).all(1)
    valid = finite(o) & finite(d) & (d != 0).any(1)
    ds = xp.where(valid[:, None], d, xp.ones_like(d))
    kz = xp.argmax(abs(ds), 1)
    kx = (kz + 1) % 3
    ky = (kx + 1) % 3
    dz = (xp.take_along_axis if xp is np else xp.take_along_dim)(ds, kz[:, None], 1)[:, 0]
    swap = dz < 0
    kx, ky = xp.where(swap, ky, kx), xp.where(swap, kx, ky)
    g = lambda k: (xp.take_along_axis if xp is np else xp.take_along_dim)(ds, k[:, None], 1)[:, 0]
    sx, sy, sz = g(kx) / dz, g(ky) / dz, (xp.ones_like(dz) / dz)
    corners = [v[fi[:, k]] for k in range(3)]
    with np.errstate(all="ignore"):
        outs = _restate_chunks(xp, o, ds, valid, corners, kx, ky, kz, sx, sy, sz, near, far, chunk, f64)
    cat = np.concatenate if xp is np else xp.cat
    fid, b1, b2, t = (cat([x[k] for x in outs]) for k in range(4))
    return fid, b1, b2, t


def _restate_chunks(xp, o, d, valid, corners, kx, ky, kz, sx, sy, sz, near, far, chunk, f64):
    outs = []
    for s in range(0, d.shape[0], chunk):
        e = slice(s, s + chunk)
        oc = o[e][:, None, :]
        rel = [X[None, :, :] - oc for X in corners]
        zs = [_pick(xp, R, kz[e]) for R in rel]
        xs = [_pick(xp, R, kx[e]) - sx[e][:, None] * z for R, z in zip(rel, zs)]
        ys = [_pick(xp, R, ky[e]) - sy[e][:, None] * z for R, z in zip(rel, zs)]
        (Ax, Bx, Cx), (Ay, By, Cy) = xs, ys
        U, V, W = Cx * By - Cy * Bx, Ax * Cy - Ay * Cx, Bx * Ay - By * Ax
        zero = (U == 0) | (V == 0) | (W == 0)
        w = lambda p: p.astype(f64) if xp is np else p.to(f64)
        n = lambda p: p.astype(F32) if xp is np else p.float()
        U = xp.where(zero, n(w(Cx) * w(By) - w(Cy) * w(Bx)), U)
        V = xp.where(zero, n(w(Ax) * w(Cy) - w(Ay) * w(Cx)), V)
        W = xp.where(zero, n(w(Bx) * w(Ay) - w(By) * w(Ax)), W)
        mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
        det = (U + V) + W
        Az, Bz, Cz = (sz[e][:, None] * z for z in zs)
        T = (U * Az + V * Bz) + W * Cz
        t = T / det
        b1, b2 = V / det, W / det
        hit = ~mixed & (det != 0) & (t > near) & (t <= far) & valid[e][:, None]
        inf = xp.full_like(t, float("inf"))
        tm = xp.where(hit, t, inf)
        tmin = tm.min(1)
        tmin = tmin[0] if xp is not np else tmin
        first = hit & (t == tmin[:, None])
        anyhit = first.any(1)
        face = xp.argmax(first.astype(np.int8) if xp is np else first.to(xp.int8), 1)
        col = lambda a: (xp.take_along_axis if xp is np else xp.take_along_dim)(a, face[:, None], 1)[:, 0]
        zf = xp.zeros_like(tmin)
        outs.append((xp.where(anyhit, face, -xp.ones_like(face)), xp.where(anyhit, col(b1), zf), xp.where(anyhit, col(b2), zf),
                     xp.where(anyhit, tmin, inf[:, 0])))
    return outs


def expected(ref, dtype):
    """The outputs of the definition in the output dtype: bc = (fl((1 - b1) - b2 in fp64), b1, b2), t widened."""
    fid, b1, b2, t = ref
    xp = _xp(t)
    if xp is np:
        b0 = ((1.0 - b1.astype(np.float64)) - b2.astype(np.float64))
        b0 = np.where(fid >= 0, b0, 0.0)
        return fid, np.stack([b0.astype(dtype), b1.astype(dtype), b2.astype(dtype)], 1), t.astype(dtype)
    b0 = xp.where(fid >= 0, (1.0 - b1.double()) - b2.double(), xp.zeros_like(b1.double()))
    return fid, xp.stack([b0.to(dtype), b1.to(dtype), b2.to(dtype)], 1), t.to(dtype)


# ---- rays ----------------------------------------------------------------------------------------------------------
def ray_sets(v, f, seed):
    """(name, o, d) families: random, a pinhole camera, aimed at vertices and edge midpoints, axis-aligned, from the
    surface, scaled directions and invalid rays."""
    rng = np.random.default_rng(seed)
    v64, fi = v.astype(np.float64), f.astype(np.int64)
    lo, hi = v64.min(0), v64.max(0)
    c, ext = (lo + hi) / 2, float((hi - lo).max()) or 1.0
    out = []
    o = c + ext * rng.standard_normal((400, 3))
    out.append(("random", o, c + 0.3 * ext * rng.standard_normal((400, 3)) - o))
    u = np.linspace(-0.6, 0.6, 24)
    px = np.stack(np.meshgrid(u, u, indexing="ij"), -1).reshape(-1, 2)
    d = np.concatenate([px, np.ones((len(px), 1))], 1)
    out.append(("camera", np.broadcast_to(c - [0, 0, 2 * ext], d.shape), d))
    corner = v64[fi[rng.integers(0, len(fi), 200)]]
    targets = np.concatenate([corner[:, 0], 0.5 * (corner[:, 0] + corner[:, 1])])
    o = c + 2 * ext * rng.standard_normal((len(targets), 3))
    out.append(("vertices and edges", o, targets - o))
    axes = np.eye(3)[rng.integers(0, 3, 300)] * rng.choice([-1.0, 1.0], (300, 1))
    o = c + 0.6 * ext * (rng.random((300, 3)) - 0.5) - 2 * ext * axes
    out.append(("axis-aligned", o, axes))
    bc = rng.dirichlet([1, 1, 1], 200)
    on = (v64[fi[rng.integers(0, len(fi), 200)]] * bc[:, :, None]).sum(1)
    out.append(("from the surface", on, rng.standard_normal((200, 3))))
    o = c + ext * rng.standard_normal((200, 3))
    dd = c - o
    out.append(("scaled 1e-3", o, 1e-3 * dd))
    out.append(("scaled 1e3", o, 1e3 * dd))
    bad_o = np.tile(c - [0, 0, 2 * ext], (6, 1))
    bad_d = np.array([[0, 0, 0], [np.nan, 0, 1], [0, np.inf, 1], [0, 0, 1], [0, 0, 1], [0, 0, 1]], dtype=np.float64)
    bad_o[3, 0], bad_o[4, 1], bad_o[5, 2] = np.nan, np.inf, -np.inf
    out.append(("invalid", bad_o, bad_d))
    return out


def _as(dtype, *xs):
    return [np.ascontiguousarray(np.asarray(x, dtype=dtype)) for x in xs]


# ---- CPU: interface, arguments, the definition -----------------------------------------------------------------------
def test_signatures(pcu):
    ps = list(inspect.signature(pcu.ray_mesh_intersection).parameters.values())
    assert [p.name for p in ps] == ["v", "f", "ray_o", "ray_d", "ray_near", "ray_far", "device"]
    assert ps[4].default == 0.0 and ps[5].default == np.inf
    assert ps[6].kind == inspect.Parameter.KEYWORD_ONLY and ps[6].default is None
    ps = list(inspect.signature(pcu.RayMeshIntersector).parameters.values())
    assert [p.name for p in ps] == ["mesh_v", "mesh_f", "device"] and ps[2].kind == inspect.Parameter.KEYWORD_ONLY
    ps = list(inspect.signature(pcu.RayMeshIntersector.intersect_rays).parameters.values())
    assert [p.name for p in ps] == ["self", "ray_o", "ray_d", "ray_near", "ray_far"]
    assert ps[3].default == 0.0 and ps[4].default == np.inf
    assert "ray_mesh_intersection" in pcu.__all__ and "RayMeshIntersector" in pcu.__all__


def test_argument_errors_come_before_the_device(pcu):
    rm = pcu.ray_mesh_intersection
    v, f = icosphere(1)
    o, d = np.zeros((4, 3)), np.ones((4, 3))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(int32\) for argument 'v'"):
        rm(v.astype(np.int32), f, o, d)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'f'"):
        rm(v, f.astype(np.float64), o, d)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'ray_o'. Expected it to match "
                                         r"argument 'v' which is of type float64."):
        rm(v, f, o.astype(np.float32), d)
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'ray_d'. Expected it to match argument 'v'"):
        rm(v, f, o, d.astype(np.float32))
    with pytest.raises(ValueError, match="ray_o and ray_d must have the same number of rows"):
        rm(v, f, o[:2], d)
    with pytest.raises(ValueError, match=r"Invalid shape for ray_o must have shape \(N, 3\) but got \(4, 2\)."):
        rm(v, f, o[:, :2], d)
    with pytest.raises(ValueError, match=r"Invalid shape for ray_d must have shape \(N, 3\) but got \(4, 2\)."):
        rm(v, f, o, d[:, :2])
    with pytest.raises(ValueError, match=r"Invalid shape for ray_d must have shape \(N, 3\) but got \(3, 1\)."):
        rm(v, f, o[0], d[0])
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        rm(v[:0], f, o, d)
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        rm(v, f[:0], o, d)
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        rm(v[:, :2], f, o, d)
    with pytest.raises(ValueError, match="NumPy array"):
        rm(v, f, o.tolist(), d)
    # the class: its mesh checks in the constructor, its ray checks (ray_d must match ray_o) in intersect_rays
    with pytest.raises(ValueError, match="Invalid input mesh with zero elements"):
        pcu.RayMeshIntersector(v, f[:0])
    with pytest.raises(ValueError, match="Only 3D inputs are supported"):
        pcu.RayMeshIntersector(v, f[:, :2])
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float32\) for argument 'f'"):
        pcu.RayMeshIntersector(v, f.astype(np.float32))


def test_closed_forms():
    # an axis-aligned ray onto the triangle (0,0,0), (2,0,0), (0,4,0) from (0.5, 1, 3) downwards: t = 3, bc = (0.5, 0.25, 0.25)
    v = np.array([[0, 0, 0], [2, 0, 0], [0, 4, 0]], np.float64)
    f = np.array([[0, 1, 2]])
    fid, b1, b2, t = restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v, f)
    assert fid[0] == 0 and t[0] == 3.0 and b1[0] == 0.25 and b2[0] == 0.25
    # the same from below (the back side counts), and with the direction scaled: t in units of |d|
    fid, b1, b2, t = restate([0.5, 1, -3], np.array([[0, 0, 2.0]]), v, f)
    assert fid[0] == 0 and t[0] == 1.5 and (b1[0], b2[0]) == (0.25, 0.25)
    # near and far: t = 3 is outside (3, inf) and inside (2, 3]
    assert restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v, f, near=3.0)[0][0] == -1
    assert restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v, f, near=2.0, far=3.0)[0][0] == 0
    assert restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v, f, far=2.99)[0][0] == -1
    # a miss beside the triangle, zero and non-finite rays
    d = np.array([[0, 0, -1.0], [0, 0, 0], [np.nan, 0, -1], [0, 0, -np.inf]])
    fid = restate(np.array([[3, 3, 3], [0.5, 1, 3], [0.5, 1, 3], [0.5, 1, 3]]), d, v, f)[0]
    assert (fid == -1).all()
    # two stacked copies: the nearer wins; the same face twice: the lower index wins
    v2 = np.concatenate([v, v + [0, 0, 1]])
    fid, _, _, t = restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v2, np.array([[0, 1, 2], [3, 4, 5], [0, 1, 2]]))
    assert fid[0] == 1 and t[0] == 2.0
    fid = restate([0.5, 1, 3], np.array([[0, 0, -1.0]]), v, np.array([[0, 1, 2], [0, 1, 2]]))[0]
    assert fid[0] == 0


def test_restatement_is_watertight():
    # from the centre of a closed icosphere, rays towards every vertex and every edge midpoint: none passes between faces
    v, f = icosphere(3)
    v32 = v.astype(F32).astype(np.float64)
    edges = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    d = np.concatenate([v32, 0.5 * (v32[edges[:, 0]] + v32[edges[:, 1]])])
    fid, b1, b2, t = restate(np.zeros(3), d, v, f)
    assert (fid >= 0).all()
    a, b, c = (v32[f[fid, k]] for k in range(3))
    n = np.cross(b - a, c - a)
    assert ((n * d).sum(1) > 0).all()           # the face hit is left through its outer side


# ---- GPU -----------------------------------------------------------------------------------------------------------
def check(got, ref, dtype, fdt, what):
    fid, bc, t = got
    efid, ebc, et = expected(ref, dtype)
    assert fid.dtype == fdt, what
    assert np.array_equal(fid.astype(np.int64), efid.astype(fdt).astype(np.int64)), what + " fid"
    assert_bits(bc, ebc, what + " bc")
    assert_bits(t, et, what + " t")


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_matches_the_definition_bit_for_bit(pcu, vdtype):
    for name, make in ALL_MESHES.items():
        v, f = make(vdtype)
        isect = pcu.RayMeshIntersector(v, f)
        for setname, o, d in ray_sets(v, f, 11):
            o, d = _as(vdtype, o, d)
            for near, far in ((0.0, np.inf), (0.25, np.inf), (0.0, 2.0)):
                ref = restate(o, d, v, f, near, far)
                for fdt in FDTYPES:
                    got = pcu.ray_mesh_intersection(v, f.astype(fdt), o, d, near, far)
                    check(got, ref, vdtype, fdt, "%s %s %s %s" % (name, setname, fdt.__name__, (near, far)))
                check(isect.intersect_rays(o, d, near, far), ref, vdtype, np.int32, "%s %s class" % (name, setname))
        isect.close()


@pytest.mark.gpu
def test_rays_from_the_surface_and_far_cut_off(pcu):
    v, f = icosphere(3, 0.01, 1, np.float32)
    rng = np.random.default_rng(4)
    bc = rng.dirichlet([1, 1, 1], 500)
    o = (v.astype(np.float64)[f[rng.integers(0, len(f), 500)]] * bc[:, :, None]).sum(1).astype(F32)
    d = rng.standard_normal((500, 3)).astype(F32)
    for near, far in ((0.0, np.inf), (1e-4, np.inf), (0.0, 0.5), (0.1, 1.0)):
        ref = restate(o, d, v, f, near, far)
        check(pcu.ray_mesh_intersection(v, f, o, d, near, far), ref, F32, np.int64, "surface %s" % ((near, far),))


@pytest.mark.gpu
def test_the_reference_check(pcu):
    # the reference's test_examples.py::test_ray_mesh_intersection on a mesh normalised to [-1, 1]^3
    v, f = ALL_MESHES["torus"](np.float64)
    v = v - v.min(0)
    v = v / v.max(0)
    v = (v - 0.5) * 2.0
    d = np.concatenate([np.stack([a.ravel() for a in np.mgrid[-0.1:0.1:64j, -0.1:0.1:64j]], axis=-1),
                        0.1 * np.ones([64 ** 2, 1])], axis=-1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    o1 = np.array([0.3, 0.2, -2.0])
    fid1, bc1, t1 = pcu.ray_mesh_intersection(v, f, o1, d)
    mask1 = np.isfinite(t1)
    assert mask1.sum() > 0
    p11 = pcu.interpolate_barycentric_coords(f, fid1[mask1], bc1[mask1], v)
    assert np.allclose(p11, o1 + t1[mask1, None] * d[mask1], atol=1e-5)
    o2 = np.stack([o1] * d.shape[0])
    out2 = pcu.ray_mesh_intersection(v, f, o2, d)
    for a, b in zip((fid1, bc1, t1), out2):
        assert np.array_equal(a, b)
    out3 = pcu.ray_mesh_intersection(v, f, o1[None], d)       # a (1, 3) origin: its three elements in order
    for a, b in zip((fid1, bc1, t1), out3):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_watertight(pcu):
    for vdtype in (np.float32, np.float64):
        v, f = icosphere(4, 0.0, 0, vdtype)
        v32 = v.astype(F32).astype(np.float64)
        edges = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        d = np.concatenate([v32, 0.5 * (v32[edges[:, 0]] + v32[edges[:, 1]])]).astype(vdtype)
        fid, bc, t = pcu.ray_mesh_intersection(v, f, np.zeros(3, vdtype), d)
        assert (fid >= 0).all()
        a, b, c = (v32[f[fid, k]] for k in range(3))
        assert ((np.cross(b - a, c - a) * d).sum(1) > 0).all()
        ref = restate(np.zeros(3), d, v, f)
        check((fid, bc, t), ref, vdtype, np.int64, "watertight")


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [2.0 ** 20, 2.0 ** -14])
def test_scale(pcu, scale):
    for name in ("icosphere", "torus", "grid"):
        v, f = ALL_MESHES[name](F32)
        unit = []
        for setname, o, d in ray_sets(v, f, 5)[:-1]:
            o, d = _as(F32, o, d)
            unit.append(pcu.ray_mesh_intersection(v, f, o, d))
            s = F32(scale)
            got = pcu.ray_mesh_intersection(v * s, f, o * s, d)
            assert np.array_equal(got[0], unit[-1][0]), (name, setname)
            assert_bits(got[1], unit[-1][1], "%s %s bc" % (name, setname))
            assert_bits(got[2], unit[-1][2] * s, "%s %s t" % (name, setname))


@pytest.mark.gpu
def test_precision_handle_and_devices(pcu):
    import torch
    v, f = icosphere(3, 0.01, 1, F32)
    sets = ray_sets(v, f, 8)
    o = np.concatenate([s[1] for s in sets[:-1]]).astype(F32)
    d = np.concatenate([s[2] for s in sets[:-1]]).astype(F32)
    a32 = pcu.ray_mesh_intersection(v, f, o, d)
    a64 = pcu.ray_mesh_intersection(v.astype(np.float64), f, o.astype(np.float64), d.astype(np.float64))
    assert np.array_equal(a32[0], a64[0])
    assert_bits(np.ascontiguousarray(a64[1][:, 1:]), a32[1][:, 1:].astype(np.float64), "fp64 b1, b2")
    assert_bits(a64[1][:, 0].astype(F32), np.ascontiguousarray(a32[1][:, 0]), "fp64 b0")     # (1 - b1) - b2 is kept in fp64 there
    assert_bits(a64[2], a32[2].astype(np.float64), "fp64 t")
    for mesh_dtype in (F32, np.float64):
        isect = pcu.RayMeshIntersector(v.astype(mesh_dtype), f)
        assert isect.v.dtype == mesh_dtype and isect.f is f
        for ray_dtype, ref in ((F32, a32), (np.float64, a64)):
            parts = [isect.intersect_rays(o[s:s + 700].astype(ray_dtype), d[s:s + 700].astype(ray_dtype)) for s in range(0, len(o), 700)]
            got = [np.concatenate([p[k] for p in parts]) for k in range(3)]
            assert got[0].dtype == np.int32 and np.array_equal(got[0], ref[0].astype(np.int32))
            assert_bits(got[1], ref[1], "class bc")
            assert_bits(got[2], ref[2], "class t")
        tc = isect.intersect_rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda())
        assert all(x.is_cuda for x in tc) and tc[0].dtype == torch.int32
        assert np.array_equal(tc[0].cpu().numpy(), a32[0].astype(np.int32))
        cpu = isect.intersect_rays(torch.from_numpy(o), torch.from_numpy(d))
        assert all(not x.is_cuda for x in cpu) and np.array_equal(cpu[2].numpy(), a32[2])
        if torch.cuda.device_count() > 1:
            with pytest.raises(ValueError, match="the rays live on"):
                isect.intersect_rays(torch.from_numpy(o).cuda(1), torch.from_numpy(d).cuda(1))
        isect.close()
        with pytest.raises(ValueError, match="has been closed"):
            isect.intersect_rays(o, d)
    # the function's input forms
    tc = pcu.ray_mesh_intersection(*(torch.from_numpy(x).cuda() for x in (v, f, o, d)))
    assert all(x.is_cuda for x in tc) and tc[0].dtype == torch.int64
    cpu = pcu.ray_mesh_intersection(*(torch.from_numpy(x) for x in (v, f, o, d)))
    for i in range(3):
        assert np.array_equal(tc[i].cpu().numpy(), a32[i]) and np.array_equal(cpu[i].numpy(), a32[i])
    isect = pcu.RayMeshIntersector(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert np.array_equal(isect.intersect_rays(o, d)[0], a32[0].astype(np.int32))
    with pytest.raises(ValueError, match=r"argument 'ray_d'. Expected it to match argument 'ray_o'"):
        isect.intersect_rays(o, d.astype(np.float64))
    with pytest.raises(ValueError, match="ray_o and ray_d must have the same number of rows"):
        isect.intersect_rays(o[:5], d)


@pytest.mark.gpu
def test_edge_cases(pcu):
    v, f = icosphere(2, 0.0, 0, F32)
    o = np.array([[0, 0, 5], [0, 0, 0]], F32)
    d = np.array([[1, 0, 0], [0, 0, 1]], F32)           # the first misses, the second hits
    for fdt, miss in ((np.uint32, 2 ** 32 - 1), (np.uint64, 2 ** 64 - 1), (np.int32, -1), (np.int64, -1)):
        fid, bc, t = pcu.ray_mesh_intersection(v, f.astype(fdt), o, d)
        assert fid.dtype == fdt and int(fid[0]) == miss and int(fid[1]) != miss
        assert t[0] == np.inf and (bc[0] == 0).all() and np.isfinite(t[1])
    before = pcu.launch_count()
    for fdt in FDTYPES:
        fid, bc, t = pcu.ray_mesh_intersection(v, f.astype(fdt), np.zeros((0, 3), F32), np.zeros((0, 3), F32))
        assert fid.shape == (0,) and fid.dtype == fdt and bc.shape == (0, 3) and t.dtype == F32
    assert pcu.launch_count() == before
    fid, bc, t = pcu.ray_mesh_intersection(v, f, np.zeros(3, F32), np.zeros((0, 3), F32))
    assert fid.shape == (0,)
    isect = pcu.RayMeshIntersector(v, f)
    before = pcu.launch_count()
    fid, bc, t = isect.intersect_rays(np.zeros((0, 3)), np.zeros((0, 3)))
    assert fid.dtype == np.int32 and bc.dtype == np.float64 and pcu.launch_count() == before
    # bad face indices raise without a fault, in the function and in the constructor
    for g, count in ((f.astype(np.int64), 2), (f.astype(np.uint32), 1)):
        g[[3, 7][:count], 1] = len(v) + 3
        with pytest.raises(ValueError, match=r"Invalid face indices: %d faces have a corner outside \[0, #v\)" % count):
            pcu.ray_mesh_intersection(v, g, o, d)
        with pytest.raises(ValueError, match=r"Invalid face indices: %d faces" % count):
            pcu.RayMeshIntersector(v, g)
    assert np.array_equal(isect.intersect_rays(o, d)[0], pcu.ray_mesh_intersection(v, f, o, d)[0].astype(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
def test_full_size(pcu, vdtype):
    import torch
    v, f = icosphere(8, 1e-4, 5, vdtype)                 # 1 310 720 faces
    f = f.astype(np.int32)
    rng = np.random.default_rng(12)
    n = 10 ** 6
    o = (rng.standard_normal((n, 3)) * 2).astype(vdtype)
    d = (rng.standard_normal((n, 3)) * 0.3 - o).astype(vdtype)
    ot, dt, vt, ft = (torch.from_numpy(x).cuda() for x in (o, d, v, f))
    fid, bc, t = pcu.ray_mesh_intersection(vt, ft, ot, dt)
    assert fid.dtype == torch.int32 and (fid >= 0).float().mean() > 0.5
    isect = pcu.RayMeshIntersector(vt, ft)
    again = isect.intersect_rays(ot, dt)
    assert torch.equal(again[0], fid) and torch.equal(again[1], bc) and torch.equal(again[2], t)
    rows = torch.from_numpy(rng.choice(n, 3000, replace=False)).cuda()
    ref = restate(ot[rows], dt[rows], vt, ft, chunk=4)
    efid, ebc, et = expected(ref, vt.dtype)
    assert torch.equal(fid[rows].long(), efid)
    assert torch.equal(bc[rows], ebc) and torch.equal(t[rows], et)
