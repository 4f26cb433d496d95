"""mesh_face_areas, estimate_mesh_face_normals, estimate_mesh_vertex_normals, mesh_principal_curvatures,
mesh_mean_and_gaussian_curvatures and laplacian_smooth_mesh -- the reference's names, arguments and outputs (the
reference's src/face_areas.cpp, src/mesh_normals.cpp, src/curvature.cpp and src/smooth.cpp), computed by
csrc/mesh_geometry.cuh, csrc/curvature.cuh and csrc/laplacian.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages and in its order, before any
device call.  Shapes are the reference's through npe::move, which squeezes them as numpy does: a single face gives a
0-d area and a (3,) normal, a single vertex a (3,) result."""
import math
import warnings

from . import _pcu_internal
from ._call import _INDEX_KINDS, _dtype_name, _form, _run, _torch, _validate_mesh

_SIGNED_KINDS = {"int32": 0, "int64": 1}
_MAX_VERTICES = 2 ** 31 - 2
_MAX_FACES = (2 ** 31 - 1) // 6
_WEIGHTINGS = {"uniform": 0, "area": 1, "angle": 2}
_CG_MAX_ITERS = 10000   # conjugate-gradient iterations per smoothing step before it stops with a RuntimeWarning
_CG_TOL = 1e-12         # a step's solve converges when |r| <= _CG_TOL |b| in every column (csrc/laplacian.cuh)


def _check_size(name, v, f):
    nvert, nface = int(v.shape[0]), int(f.shape[0])
    if nvert > _MAX_VERTICES or nface > _MAX_FACES:
        raise ValueError("%s: at most %d vertices and %d faces are supported, got %d and %d" % (name, _MAX_VERTICES, _MAX_FACES, nvert, nface))
    return nvert, nface


def _face_pass(v, f, normal, device):
    form = _form([v, f], ["v", "f"])
    nvert, nface = _check_size("estimate_mesh_face_normals" if normal else "mesh_face_areas", v, f)
    torch = _torch()

    def body(vt, ft, dev, stream):
        out = torch.empty((nface, 3) if normal else (nface,), dtype=vt.dtype, device=vt.device)
        _pcu_internal._mesh_face_device(vt.dtype == torch.float64, normal, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                        _INDEX_KINDS[_dtype_name(f)], out.data_ptr(), dev, stream)
        return out

    return _run(form, [v, f], device, body, squeeze=True)


def mesh_face_areas(v, f, num_threads=-1, *, device=None):
    """
    Compute the areas of each face of a triangle mesh

    Args:
        v : #v by 3 array of vertex positions (each row is a vertex)
        f : #f by 3 Matrix of face (triangle) indices
        num_threads : accepted and ignored (the reference's CPU thread count; the result never depended on it)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        areas : a numpy array of shape (#faces,) where areas[i] is the area of the face f[i]

    Dtypes: v float32 / float64, f int32 / int64; areas has v's dtype.  Defined in DESIGN.md §3 as the reference
    computes it (src/face_areas.cpp), operation for operation in v's precision: Heron's formula on the edge lengths
    sqrt((x x + y y) + z z).  One face gives a 0-d array.
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _SIGNED_KINDS)
    return _face_pass(v, f, False, device)


def estimate_mesh_face_normals(v, f, *, device=None):
    """
    Compute the unit normals of the faces of a triangle mesh

    Args:
        v : (#v, 3)-shaped NumPy array of mesh vertex 3D positions
        f : (#f, 3)-shaped NumPy array of face (triangle) indices
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        n : (#f, 3)-shaped NumPy array of face normals (i.e. n[i] is the normal at face f[i]). Note that any degenerate faces will have a zero normal.

    Dtypes: v float32 / float64, f int32 / int64 / uint32 / uint64; n has v's dtype.  Defined in DESIGN.md §3:
    n = (v1 - v0) x (v2 - v0) divided by its norm sqrt((x x + y y) + z z), the zero vector where that norm is 0, in
    fp64 and rounded once to v's dtype.  The reference computes it with libigl's per_face_normals, whose rounding is
    not pinned here.  One face gives shape (3,).
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    return _face_pass(v, f, True, device)


def estimate_mesh_vertex_normals(v, f, weighting_type="uniform", *, device=None):
    """
    Compute vertex normals of a mesh from its vertices and faces

    Args:
        v : (#v, 3)-shaped NumPy array of mesh vertex 3D positions
        f : (#f, 3)-shaped NumPy array of face (triangle) indices
        weighting_type : Weighting type must be one of 'uniform', 'angle', or 'area' (default is 'uniform')
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        n : (#v, 3)-shaped NumPy array of vertex normals (i.e. n[i] is the normal at vertex v[i])

    Dtypes: v float32 / float64, f int32 / int64 / uint32 / uint64; n has v's dtype.  Defined in DESIGN.md §3: for
    every vertex the sum of w n_f over its corners in ascending (face, corner) order -- n_f the unit face normal of
    `estimate_mesh_face_normals` -- divided by its norm, the zero vector where the sum is zero (a vertex no face uses
    included), in fp64 and rounded once to v's dtype.  w is 1 ('uniform'), |e1 x e2| ('area') or the corner's interior
    angle atan2(|e1 x e2|, e1 . e2) ('angle'), with e1, e2 the corner's two edges.  The reference computes it with
    libigl's per_vertex_normals, whose rounding and value at an isolated vertex are not pinned here.
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    if weighting_type not in _WEIGHTINGS:
        raise ValueError("Invalid weighting_type must be one of 'uniform', 'angle', or 'area', but got '%s'" % (weighting_type,))
    nvert, nface = _check_size("estimate_mesh_vertex_normals", v, f)
    torch = _torch()

    def body(vt, ft, dev, stream):
        out = torch.empty((nvert, 3), dtype=vt.dtype, device=vt.device)
        _pcu_internal._mesh_vertex_normals_device(vt.dtype == torch.float64, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                                  _INDEX_KINDS[_dtype_name(f)], _WEIGHTINGS[weighting_type], out.data_ptr(), dev, stream)
        return out

    return _run(form, [v, f], device, body, squeeze=True)


def mesh_principal_curvatures(v, f, r=-1.0, *, device=None):
    """
    Compute the principal curvatures and principal directions at every vertex of a triangle mesh

    Args:
        v : (#v, 3)-shaped array of mesh vertex 3D positions
        f : (#f, 3)-shaped array of face (triangle) indices
        r : the radius of the ball each vertex's quadric is fitted over; r <= 0 (default) uses the one-ring estimate
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        k1 : (#v,)-shaped array of the larger principal curvature at each vertex
        k2 : (#v,)-shaped array of the smaller principal curvature at each vertex
        d1 : (#v, 3)-shaped array of the unit principal direction of k1 at each vertex
        d2 : (#v, 3)-shaped array of the unit principal direction of k2 at each vertex

    Dtypes: v float32 / float64, f int32 / int64 / uint32 / uint64; every output has v's dtype.  Defined in DESIGN.md
    §3, computed in fp64 and rounded once.  On a sphere of radius R whose faces wind counter-clockwise seen from
    outside, k1 = k2 = 1 / R; reversed faces flip the sign.  k1 >= k2.  d1's component of largest magnitude is positive
    and d2 = n x d1.  A vertex whose curvature is undetermined (no face of nonzero area, fewer than 5 neighbours in the
    ball, ...) gets k1 = k2 = NaN and zero directions.
      r <= 0: Rusinkiewicz's (2004) one-ring tensor estimate, with Max's vertex normals and mixed Voronoi areas.
      r > 0: a quadric z = a x^2 + b x y + c y^2 + d x + e y fitted, in the frame of the vertex normal, to every other
             vertex j with |v_j - v_i|^2 < r^2; more robust on noisy meshes.  A ball that reaches another sheet of the
             surface (thin parts) mixes both sheets.
    The reference declares this function but ships no implementation.
    Divergences: a non-finite r and a face corner outside [0, #v) raise ValueError.
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    r = float(r)
    if not math.isfinite(r):
        raise ValueError("mesh_principal_curvatures: r must be finite, got %r" % (r,))
    nvert, nface = _check_size("mesh_principal_curvatures", v, f)
    torch = _torch()

    def body(vt, ft, dev, stream):
        k1, k2 = (torch.empty((nvert,), dtype=vt.dtype, device=vt.device) for _ in range(2))
        d1, d2 = (torch.empty((nvert, 3), dtype=vt.dtype, device=vt.device) for _ in range(2))
        _pcu_internal._mesh_curvatures_device(vt.dtype == torch.float64, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                              _INDEX_KINDS[_dtype_name(f)], r, k1.data_ptr(), k2.data_ptr(), d1.data_ptr(),
                                              d2.data_ptr(), dev, stream)
        return k1, k2, d1, d2

    return _run(form, [v, f], device, body, squeeze=True)


def mesh_mean_and_gaussian_curvatures(v, f, r=-1.0, *, device=None):
    """
    Compute the mean and Gaussian curvatures at every vertex of a triangle mesh

    Args:
        v : (#v, 3)-shaped array of mesh vertex 3D positions
        f : (#f, 3)-shaped array of face (triangle) indices
        r : see `mesh_principal_curvatures`
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        kh : (#v,)-shaped array of mean curvatures, 0.5 * (k1 + k2)
        kg : (#v,)-shaped array of Gaussian curvatures, k1 * k2

    Computed from `mesh_principal_curvatures`' k1 and k2 in their dtype and form; NaN where they are.
    """
    k1, k2, _, _ = mesh_principal_curvatures(v, f, r, device=device)
    return 0.5 * (k1 + k2), k1 * k2


def _smooth(v, f, num_iters, step_size, use_cotan_weights, device):
    """laplacian_smooth_mesh's result and the conjugate-gradient iterations of every step."""
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _SIGNED_KINDS)
    num_iters = int(num_iters)
    if num_iters < 0:
        raise ValueError("Invalid value for argument num_iters in smooth_mesh_laplacian. Must be a positive integer or 0.")
    nvert, nface = _check_size("laplacian_smooth_mesh", v, f)
    torch = _torch()
    if num_iters == 0:
        return (v.copy() if form == "numpy" else v.detach().clone()).squeeze(), []
    iters = residual = None

    def body(vt, ft, dev, stream):
        nonlocal iters, residual
        out = torch.empty((nvert, 3), dtype=vt.dtype, device=vt.device)
        iters, residual = _pcu_internal._laplacian_smooth_device(vt.dtype == torch.float64, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                                                 _INDEX_KINDS[_dtype_name(f)], num_iters, float(step_size),
                                                                 bool(use_cotan_weights), int(_CG_MAX_ITERS), out.data_ptr(), dev, stream)
        return out

    out = _run(form, [v, f], device, body, squeeze=True)
    for step, (k, res) in enumerate(zip(iters, residual)):
        if not res <= _CG_TOL:
            warnings.warn("laplacian_smooth_mesh: the solve of step %d stopped after %d conjugate-gradient iterations at a relative "
                          "residual of %.3g (tolerance %g); its iterate is returned" % (step, k, res, _CG_TOL), RuntimeWarning,
                          stacklevel=3)
    return out, iters


def laplacian_smooth_mesh(v, f, num_iters, step_size=0.1, use_cotan_weights=False, *, device=None):
    """
    Smooth a mesh using Laplacian smoothing

    Args:
        v : #v by 3 Matrix of mesh vertex 3D positions
        f : #f by 3 Matrix of face (triangle) indices
        num_iters : Number of smoothing iterations to perform
        step_size : Step size per iteration (default is 0.1)
        use_cotan_weights : see below (default is False)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v_smooth : (#v, 3)-shaped array of smoothed vertex positions

    Dtypes: v float32 / float64, f int32 / int64; v_smooth has v's dtype.  Defined in DESIGN.md §3 as the reference
    computes it (src/smooth.cpp), quirks included:
      1. num_iters < 0 raises the reference's ValueError, after the mesh checks.
      2. num_iters = 0 returns a copy of v.
      3. L is the cotangent Laplacian of the INPUT v, built once: L_ij = (cot a_ij + cot b_ij) / 2, L_ii = -sum_j L_ij.
         It is cotangent in both modes: use_cotan_weights=False means M = I, not uniform weights.
      4. With use_cotan_weights=True the step is multiplied by 1e-3; before each solve M is the barycentric lumped
         mass of the CURRENT u (M_ii = sum of dblA / 6 over the faces containing i); after each solve the mesh is
         moved about its area-weighted centroid and scaled by 1 / sqrt(area), so its total area becomes 1.
      5. Each iteration solves (M - h L) u' = M u.
      6. Corner k of a face with twice-area dblA has cot_k = (e_ki . e_kj) / dblA; a face with dblA = 0 contributes
         neither weights nor mass.
      7. A row with no mass and no weight is the identity: that vertex stays where it is.
      8. u is carried in fp64 across iterations and rounded once to v's dtype at the end.
      9. Divergences: a face corner outside [0, #v), coordinates that are not finite and (use_cotan_weights) a total
         area of 0 raise ValueError.  The reference factorises S in v's precision (Eigen's SimplicialLLT); here
         every step is a Jacobi-preconditioned conjugate-gradient solve in fp64 to |r| <= 1e-12 |b| per column, so
         the result carries less rounding than the reference's.  A step that does not converge within
         _CG_MAX_ITERS iterations issues a RuntimeWarning with the residual reached and keeps its iterate.
    """
    return _smooth(v, f, num_iters, step_size, use_cotan_weights, device)[0]
