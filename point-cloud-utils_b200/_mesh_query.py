"""closest_points_on_mesh, triangle_soup_fast_winding_number, point_cloud_fast_winding_number,
estimate_point_cloud_areas, signed_distance_to_mesh, pointcloud_apss_curvature and project_points_onto_apss -- the
reference's names, arguments and outputs (the reference's src/closest_point_on_mesh.cpp, src/fast_winding_numbers.cpp,
src/point_areas.cpp, src/signed_distance.cpp and src/curvature.cpp), computed by csrc/meshquery.cuh, csrc/winding.cuh,
csrc/point_areas.cuh and csrc/apss.cuh.

Input forms and validation follow _call.py: numpy arrays in -> numpy out; CUDA torch tensors in -> CUDA tensors
out; CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
from . import _pcu_internal
from ._call import (_INDEX_KINDS, _check_float, _check_index, _check_match, _dtype_name, _form, _matrix_shape, _raise_bad, _run,
                    _same_device, _torch, _validate_mesh)


def _validate_points(p, v, f):
    """The binding's dtype checks (npe_arg(v, npe_matches(p)) among them), then validate_point_cloud(p), which allows
    zero rows (src/common/common.h).  validate_mesh follows."""
    _check_float(p, "p")
    _check_match(v, "v", p, "p")
    _check_index(f, "f", _INDEX_KINDS)
    if len(p.shape) != 2 or p.shape[1] != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =%s."
                         % (tuple(p.shape),))


def closest_points_on_mesh(p, v, f, *, device=None):
    """
    Compute distances from a set of points p to a triangle mesh (v, f)

    Args:
        p : (#p, 3)-shaped array of query point positions (float32 / float64)
        v : (#v, 3)-shaped array of mesh vertex positions (p's dtype)
        f : (#f, 3)-shaped array of triangle face indices (int32 / int64 / uint32 / uint64)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        d : a (#p,)-shaped array of shortest distances for each query point p (p's dtype)
        f_idx : a (#p,)-shaped array of indices into f of the face containing the closest point to each query point
                (f's dtype)
        bc : a (#p, 3)-shaped array of barycentric coordinates for each query point (p's dtype)

    Mirrors the reference's src/closest_point_on_mesh.cpp (igl::point_mesh_squared_distance).  The result is a pure
    function of (p, v, f), defined in DESIGN.md §3: for every face, Ericson's Voronoi-region closest point in p's
    precision with every operation rounded on its own (a face whose corners are collinear or coincident is the union of
    its edges, as in libigl); the chosen face is the lexicographic minimum of (squared distance, face index), so among
    faces at exactly the same distance the lowest index wins.  d = sqrt(d^2), and bc are the chosen face's coordinates
    of the closest point.
    Divergences: libigl's choice among tied faces depends on its tree and is not reproduced; a face corner outside
    [0, #v) raises ValueError (the reference reads out of bounds).
    """
    form = _form([p, v, f], ["p", "v", "f"])
    _validate_points(p, v, f)
    _validate_mesh(v, f, ("int32", "int64", "uint32", "uint64"))
    torch = _torch()
    n = int(p.shape[0])
    if n == 0:
        if form == "numpy":
            import numpy as np
            return np.zeros(0, dtype=p.dtype), np.zeros(0, dtype=f.dtype), np.zeros((0, 3), dtype=p.dtype)
        if form == "cuda":
            _same_device(p, device)
        return (torch.zeros(0, dtype=p.dtype, device=p.device), torch.zeros(0, dtype=f.dtype, device=p.device),
                torch.zeros((0, 3), dtype=p.dtype, device=p.device))

    def body(pt, vt, ft, dev, stream):
        d = torch.empty(n, dtype=pt.dtype, device=pt.device)
        fidx = torch.empty(n, dtype=ft.dtype, device=pt.device)
        bc = torch.empty((n, 3), dtype=pt.dtype, device=pt.device)
        bad = torch.empty(1, dtype=torch.int64, device=pt.device)
        _pcu_internal._closest_points_on_mesh_device(pt.dtype == torch.float64, pt.data_ptr(), n, vt.data_ptr(), int(vt.shape[0]),
                                                     ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)], d.data_ptr(),
                                                     fidx.data_ptr(), bc.data_ptr(), bad.data_ptr(), dev, stream)
        _raise_bad(bad)
        return d, fidx, bc

    return _run(form, [p, v, f], device, body, index=(f, [1]))


def _validate_nonempty_points(p):
    """validate_point_cloud(p, false) (src/common/common.h:58-74): zero rows are an error."""
    if len(p.shape) == 2 and p.shape[0] == 0:
        raise ValueError("Invalid input point cloud with zero points: points must have shape (n, 3) (n > 0). Got points.shape "
                         "=%s." % (tuple(p.shape),))
    if len(p.shape) != 2 or p.shape[1] != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =%s."
                         % (tuple(p.shape),))


def triangle_soup_fast_winding_number(v, f, p, *, device=None):
    """
    Compute a consistent inside/outside field given a triangle soup and evaluate that field
    at a set of query points

    Args:
        v: (#v, 3)-shaped array of mesh vertex positions (float32 / float64)
        f: (#f, 3)-shaped array of mesh face indexes into v (int32 / int64 / uint32 / uint64)
        p: (#p, 3)-shaped array of query positions at which to evaluate the winding number field (v's dtype, #p > 0)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        w : a (#p,)-shaped array of winding numbers (v's dtype): about 1 inside and 0 outside a closed mesh whose faces
            are oriented outwards, -1 inside when they are oriented inwards, k inside k nested shells

    Mirrors the reference's src/fast_winding_numbers.cpp (libigl's fast winding numbers, Barill et al. 2018) and, like
    libigl, evaluates the field in fp32 whatever v's dtype: corners and queries are rounded to fp32, every face near the
    query contributes its exact solid angle, and a group of faces whose area-weighted centre is more than twice their
    radius away contributes Barill's order-2 far-field expansion instead.  The terms are summed in fp64 in a fixed order,
    so the result depends only on (v, f, p_i) (DESIGN.md §3).
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    form = _form([v, f, p], ["v", "f", "p"])
    _check_float(v, "v")
    _check_index(f, "f", _INDEX_KINDS)
    _check_match(p, "p", v, "v")
    _validate_mesh(v, f, tuple(_INDEX_KINDS))
    _validate_nonempty_points(p)
    torch = _torch()

    def body(vt, ft, pt, dev, stream):
        n = int(pt.shape[0])
        w = torch.empty(n, dtype=pt.dtype, device=pt.device)
        bad = torch.empty(1, dtype=torch.int64, device=pt.device)
        _pcu_internal._fast_winding_number_device(pt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(),
                                                  int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)], pt.data_ptr(), n, 2.0, w.data_ptr(),
                                                  bad.data_ptr(), dev, stream)
        _raise_bad(bad)
        return w

    return _run(form, [v, f, p], device, body)


def _validate_point_cloud_normals(p, n):
    """validate_point_cloud_normals(p, n) (src/common/common.h:78-109): zero points are allowed."""
    ps, ns = tuple(p.shape), tuple(n.shape)
    if len(ps) != 2 or ps[1] != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =%s." % (ps,))
    if len(ns) != 2 or ns[1] != 3:
        raise ValueError("Invalid shape for normals: must have shape (n, 3) (n > 0). Got normals.shape =%s." % (ns,))
    if ns[0] != ps[0]:
        raise ValueError("Invalid input point cloud. Number of normals must match number of points. Got points.shape =%s and "
                         "normals.shape = %d, %d" % (ps, ns[0], ns[1]))


def point_cloud_fast_winding_number(p, n, a, q, *, device=None):
    """
    Compute a consistent inside/outside field given a point cloud and evaluate that field
    at a set of query points

    Args:
        p : (#p, 3)-shaped array of points (float32 / float64)
        n : (#p, 3)-shaped array of point normals at p (p's dtype), used as given (not normalised)
        a : array of #p point areas (p's dtype), of any shape with #p elements, e.g. (#p,) or (#p, 1)
        q : (#q, 3)-shaped array of query positions at which to evaluate the winding number field (p's dtype, #q > 0)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        w : a (#q,)-shaped array of winding numbers (p's dtype): about 1 inside and 0 outside a closed surface sampled with
            outward normals and areas that sum to its area, -1 inside with inward normals

    Mirrors the reference's src/fast_winding_numbers.cpp (libigl's fast winding numbers for point clouds, Barill et al.
    2018).  Point i contributes the dipole a_i n_i . (p_i - q) / |p_i - q|^3 / 4 pi, evaluated in fp32 whatever p's dtype:
    points and queries are rounded to fp32, a_i n_i is formed in p's dtype and rounded to fp32, every point near the query
    contributes its exact term (none when the query is on the point), and a group of points whose |a|-weighted centre is
    more than twice their radius away contributes Barill's order-2 far-field expansion instead.  The terms are summed in
    fp64 in a fixed order, so the result depends only on (p, n, a, q_i) (DESIGN.md §3).
    Divergences: a of any shape with exactly #p elements is accepted and any other size raises ValueError (the reference
    reads a short vector out of bounds); #p = 0 gives w = 0 for every query.
    For a scanned cloud, `estimate_point_cloud_areas(p, k_nearest_neighbors(p, p, k)[1], n)` gives the areas a.
    """
    form = _form([p, n, a, q], ["p", "n", "a", "q"])
    _check_float(p, "p")
    for x, name in ((n, "n"), (a, "a"), (q, "q")):
        _check_match(x, name, p, "p")
    _validate_point_cloud_normals(p, n)
    _validate_nonempty_points(q)
    na = 1
    for s in a.shape:
        na *= int(s)
    if na != int(p.shape[0]):
        raise ValueError("Invalid shape for areas: a must have #p = %d elements, e.g. shape (#p,) or (#p, 1). Got a.shape =%s."
                         % (int(p.shape[0]), tuple(a.shape)))
    torch = _torch()

    def body(pt, nt, at, qt, dev, stream):
        m, nq = int(pt.shape[0]), int(qt.shape[0])
        w = torch.empty(nq, dtype=qt.dtype, device=qt.device)
        _pcu_internal._point_cloud_fast_winding_number_device(qt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), at.data_ptr(), m,
                                                              qt.data_ptr(), nq, 2.0, w.data_ptr(), dev, stream)
        return w

    return _run(form, [p, n, a, q], device, body)


_AREAS_MAX_K = 256   # kAreaMaxK of csrc/point_areas.cuh


def estimate_point_cloud_areas(p, i, n, *, device=None):
    """
    Estimate the area of the surface around each point of an oriented point cloud

    Args:
        p : (#p, 3)-shaped array of 3D points (float32 / float64)
        i : (#p, k)-shaped array of indices where i[a, b] is the index of the b^th nearest neighbor to point p[a]
            (int32 / int64 / uint32 / uint64), with the point itself in column 0 -- what k_nearest_neighbors(p, p, k)[1]
            returns; a (#p,)-shaped array counts as k = 1.  k <= 256.
        n : (#p, 3)-shaped array of point normals (p's dtype)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        a : a (#p,)-shaped array of areas (p's dtype): a[r] is the area of point i[r, 0] from the neighbours in row r, for
            the areas `point_cloud_fast_winding_number` takes

    Mirrors the reference's src/point_areas.cpp (libigl's igl::copyleft::cgal::point_areas, which is not in the
    reference's tree).  The result is a pure function of (p, n, i[r]), defined in DESIGN.md §3: the neighbours whose
    normals have a positive dot product with the centre's are projected onto their PCA plane; the centre's star in the
    2-D Delaunay triangulation of the projected points is walked from its nearest neighbour, with fixed rules for ties;
    the area is Meyer et al.'s mixed Voronoi area of the centre over that star, or 0 when fewer than three neighbours
    are kept or the star is empty.  Everything is computed in fp64 and rounded once to p's dtype.
    Divergence: an entry of i outside [0, #p), such as the -1 that k_nearest_neighbors writes when k > #p, raises
    ValueError (the reference reads out of bounds).
    """
    form = _form([p, i, n], ["p", "i", "n"])
    _check_float(p, "p")
    _check_index(i, "i", _INDEX_KINDS)
    _check_match(n, "n", p, "p")
    _validate_point_cloud_normals(p, n)
    m = int(p.shape[0])
    rows, k = (int(i.shape[0]), 1 if len(i.shape) == 1 else int(i.shape[1])) if len(i.shape) in (1, 2) else (-1, 0)
    if rows != m:
        shape = _matrix_shape(i)
        raise ValueError("Invalid shape for i (knn indices), must be (#p, k) where #p is the number of input points (%d). "
                         "Got (%d, %d)" % (m, shape[0], shape[1]))
    if k > _AREAS_MAX_K:
        raise ValueError("Invalid shape for i (knn indices): at most %d neighbours per point are supported, got k = %d"
                         % (_AREAS_MAX_K, k))
    torch = _torch()
    if m == 0:
        if form == "numpy":
            import numpy as np
            return np.zeros(0, dtype=p.dtype)
        if form == "cuda":
            _same_device(p, device)
        return torch.zeros(0, dtype=p.dtype, device=p.device)

    def body(pt, it, nt, dev, stream):
        a = torch.empty(m, dtype=pt.dtype, device=pt.device)
        bad = torch.empty(1, dtype=torch.int64, device=pt.device)
        _pcu_internal._estimate_point_cloud_areas_device(pt.dtype == torch.float64, pt.data_ptr(), m, nt.data_ptr(), it.data_ptr(), k,
                                                         _INDEX_KINDS[_dtype_name(i)], a.data_ptr(), bad.data_ptr(), dev, stream)
        _raise_bad(bad, "Invalid knn indices: %d entries of i are outside [0, #p)")
        return a

    return _run(form, [p, i, n], device, body, squeeze=True)


def signed_distance_to_mesh(p, v, f, lower_bound=-float("inf"), upper_bound=float("inf"), *, device=None):
    """
    Computes signed distances of a point cloud with respect to a Mesh using Fast Winding Numbers

    Args:
        p : (#p, 3)-shaped array point cloud (float32 / float64, #p > 0)
        v : (#v, 3)-shaped array of mesh vertex positions (p's dtype)
        f : (#f, 3)-shaped array of mesh face indexes into v (int32 / int64 / uint32 / uint64)
        lower_bound : the lower end of the band of distances to compute (rounded to float32), -inf by default
        upper_bound : the upper end of the band of distances to compute (rounded to float32), +inf by default
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        s : a (#p,)-shaped array of signed distances (p's dtype): negative inside, positive outside
        fi : a (#p,)-shaped int32 array of indices of the closest face
        bc : a (#p, 3)-shaped array of barycentric coordinates of the closest point on that face (p's dtype)

    Mirrors the reference's src/signed_distance.cpp (libigl's signed_distance with the fast-winding-number sign).
    fi and bc are exactly those of `closest_points_on_mesh(p, v, f)`, and s = sigma * d with d that function's
    distance and sigma = 1 - 2|w|, w exactly `triangle_soup_fast_winding_number(v, f, p)`.  sigma is libigl's continuous
    factor, not a sign: it is about -1 inside and +1 outside a closed, consistently oriented mesh, and -3 inside two
    nested shells (|w| = 2), as in libigl.  With max_abs = max(-lower_bound, upper_bound), a query whose squared distance
    is at least max_abs^2, or below max(max_abs - (upper_bound - lower_bound), 0)^2, is out of the band: s = NaN,
    fi = #f + 1 and bc = NaN (DESIGN.md §3).  The default bounds give no band.
    Divergences: out of the band, bc is NaN (libigl reads face #f + 1 out of bounds); a face corner outside [0, #v)
    raises ValueError (the reference reads out of bounds).
    """
    import numpy as np
    form = _form([p, v, f], ["p", "v", "f"])
    _check_float(p, "p")
    _check_match(v, "v", p, "p")
    _validate_mesh(v, f, tuple(_INDEX_KINDS))
    _validate_nonempty_points(p)
    lower, upper = float(np.float32(lower_bound)), float(np.float32(upper_bound))
    torch = _torch()

    def body(pt, vt, ft, dev, stream):
        n = int(pt.shape[0])
        s = torch.empty(n, dtype=pt.dtype, device=pt.device)
        fidx = torch.empty(n, dtype=torch.int32, device=pt.device)
        bc = torch.empty((n, 3), dtype=pt.dtype, device=pt.device)
        bad = torch.empty(1, dtype=torch.int64, device=pt.device)
        _pcu_internal._signed_distance_to_mesh_device(pt.dtype == torch.float64, pt.data_ptr(), n, vt.data_ptr(), int(vt.shape[0]),
                                                      ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)], lower, upper,
                                                      s.data_ptr(), fidx.data_ptr(), bc.data_ptr(), bad.data_ptr(), dev, stream)
        _raise_bad(bad)
        return s, fidx, bc

    return _run(form, [p, v, f], device, body)


def _apss_radius(r):
    """The ball radius of the APSS functions: a finite number > 0."""
    import math
    try:
        r = float(r)
    except (TypeError, ValueError):
        raise ValueError("Invalid radius r (%r): must be a finite number greater than 0." % (r,)) from None
    if not (math.isfinite(r) and r > 0.0):
        raise ValueError("Invalid radius r (%r): must be a finite number greater than 0." % (r,))
    return r


def _apss_device(pt, nt, qt, nq, r, out_x, out_n, kh, dev, stream):
    """One native call: qt None runs the queries at the points themselves; out_x / out_n None are not written."""
    torch = _torch()
    _pcu_internal._apss_device(pt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), int(pt.shape[0]),
                               0 if qt is None else qt.data_ptr(), nq, r, 0 if out_x is None else out_x.data_ptr(),
                               0 if out_n is None else out_n.data_ptr(), kh.data_ptr(), dev, stream)


def pointcloud_apss_curvature(p, n, r, *, device=None):
    """
    Estimate the mean curvature of the surface an oriented point cloud samples, with an algebraic point set surface

    Args:
        p : (#p, 3)-shaped array of points (float32 / float64)
        n : (#p, 3)-shaped array of point normals (p's dtype), normalised in fp64 before use; a zero normal leaves its
            point out of every fit
        r : the radius of the ball each fit uses, a true distance (not squared), finite and > 0
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        kh : a (#p,)-shaped array (p's dtype): the mean curvature of the surface at the projection of each point, +1/R
             on a sphere of radius R with outward normals; NaN where it is undetermined

    The reference declares pointcloud_apss_curvature(v, f) in src/curvature.cpp with its body commented out; APSS needs
    oriented points and no faces, so this takes (p, n, r).  kh[i] is exactly project_points_onto_apss(p, n, p, r)[2][i]:
    see that function for the surface and DESIGN.md §3 for the rules.
    """
    form = _form([p, n], ["p", "n"])
    _check_float(p, "p")
    _check_match(n, "n", p, "p")
    _validate_point_cloud_normals(p, n)
    r = _apss_radius(r)
    m = int(p.shape[0])
    torch = _torch()
    if m == 0:
        if form == "numpy":
            import numpy as np
            return np.zeros(0, dtype=p.dtype)
        if form == "cuda":
            _same_device(p, device)
        return torch.zeros(0, dtype=p.dtype, device=p.device)

    def body(pt, nt, dev, stream):
        kh = torch.empty(m, dtype=pt.dtype, device=pt.device)
        _apss_device(pt, nt, None, m, r, None, None, kh, dev, stream)
        return kh

    return _run(form, [p, n], device, body)


def project_points_onto_apss(p, n, q, r, *, device=None):
    """
    Project query points onto the algebraic point set surface of an oriented point cloud

    Args:
        p : (#p, 3)-shaped array of points (float32 / float64)
        n : (#p, 3)-shaped array of point normals (p's dtype), normalised in fp64 before use; a zero normal leaves its
            point out of every fit
        q : (#q, 3)-shaped array of query points (p's dtype, #q > 0)
        r : the radius of the ball each fit uses, a true distance (not squared), finite and > 0
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        x : a (#q, 3)-shaped array of the projected points (p's dtype)
        nx : a (#q, 3)-shaped array of unit surface normals at x (p's dtype), oriented like n
        kh : a (#q,)-shaped array of mean curvatures at x (p's dtype), +1/R on a sphere of radius R with outward normals

    The surface is Guennebaud and Gross's APSS (SIGGRAPH 2007) with the spherical parameter 1: around an iterate x,
    every point within distance r whose normal is not zero is weighted by (1 - |p_j - x|^2 / r^2)^4, an algebraic
    sphere is fitted to those points and normals in closed form, and x moves to the closest point of that sphere.
    The iteration starts at q and stops after a step of at most 1e-10 r, or after 20 steps.  nx and kh come from the
    last fitted sphere.  A query whose ball holds fewer than 4 points with a normal, or whose sphere gives no step, is
    undetermined: x = NaN, nx = 0, kh = NaN; so is every query when #p = 0.  Everything is computed in fp64 and rounded
    once to p's dtype (DESIGN.md §3).
    """
    form = _form([p, n, q], ["p", "n", "q"])
    _check_float(p, "p")
    _check_match(n, "n", p, "p")
    _check_match(q, "q", p, "p")
    _validate_point_cloud_normals(p, n)
    _validate_nonempty_points(q)
    r = _apss_radius(r)
    torch = _torch()

    def body(pt, nt, qt, dev, stream):
        nq = int(qt.shape[0])
        x = torch.empty((nq, 3), dtype=pt.dtype, device=pt.device)
        nx = torch.empty((nq, 3), dtype=pt.dtype, device=pt.device)
        kh = torch.empty(nq, dtype=pt.dtype, device=pt.device)
        _apss_device(pt, nt, qt, nq, r, x, nx, kh, dev, stream)
        return x, nx, kh

    return _run(form, [p, n, q], device, body)
