"""ray_surfel_intersection, RaySurfelIntersector, pointcloud_surfel_geometry and pointcloud_sphere_geometry -- the
reference's names, arguments and outputs (the reference's src/ray_point_cloud_intersection.cpp,
point_cloud_utils/_ray_point_cloud_intersector.py and _point_cloud_geometry.py), computed by csrc/raycast.cuh on the
surfel tree of csrc/meshquery.cuh, and by the geometry kernels of csrc/meshquery.cuh.

Input forms and validation follow _call.py: numpy arrays in -> numpy out; CUDA torch tensors in -> CUDA tensors
out; CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
import numpy as np

from . import _pcu_internal
from ._call import _call_args, _check_float, _check_match, _dtype_name, _form, _is_tensor, _matrix_shape, _run, _same_device, _torch, _upload
from ._ray_mesh import _Prepared, _bounds, _cast, _validate_rays

_MAX_SUBDIVS = 2 ** 24


def _validate_radius(p, r):
    """_validate_point_radius_internal (point_cloud_utils/_point_cloud_geometry.py:24-42): a scalar, a list or tuple,
    or an (N,) or (N, 1) array (a tensor here too)."""
    if not (isinstance(r, np.ndarray) or _is_tensor(r)):
        if np.isscalar(r):
            r = r * np.ones(p.shape[0])
        elif isinstance(r, (list, tuple)):
            r = np.array(r).astype(_dtype_name(p))
        else:
            raise ValueError("Argument r must be a scalar or numpy array with the same number of rows as p")
    if r.shape[0] != p.shape[0]:
        raise ValueError("Argument r have the same number of rows as p")
    if len(r.shape) != 1:
        r = r.squeeze()
    if len(r.shape) != 1:
        raise ValueError("Invalid shape for argument r, must have shape (N,) or (N, 1)")
    return r


def _validate_surfels(p, n, subdivs):
    """validate_point_cloud_normals (src/common/common.h:78-110, zero points allowed), then the subdivision check of
    validate_point_geometry (src/ray_point_cloud_intersection.cpp:57-63).  Returns subdivs as an int."""
    (prows, pcols), (nrows, ncols) = _matrix_shape(p), _matrix_shape(n)
    if pcols != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =(%d, %d)."
                         % (prows, pcols))
    if ncols != 3:
        raise ValueError("Invalid shape for normals: must have shape (n, 3) (n > 0). Got normals.shape =(%d, %d)."
                         % (nrows, ncols))
    if nrows != prows:
        raise ValueError("Invalid input point cloud. Number of normals must match number of points. Got points.shape "
                         "=(%d, %d) and normals.shape = %d, %d" % (prows, pcols, nrows, ncols))
    subdivs = int(subdivs)
    if subdivs < 4:
        raise ValueError("Invalid geometry_subdivisions_1 is less than or equal to 4.")
    if subdivs > _MAX_SUBDIVS:
        raise ValueError("subdivs must be at most 2^24 (got %d)" % subdivs)
    return subdivs


def _radius_like(r, p, form):
    """r in p's dtype and form (a CUDA tensor on p's device for CUDA inputs)."""
    if form == "cuda":
        torch = _torch()
        r = r if _is_tensor(r) else torch.from_numpy(np.ascontiguousarray(r))
        return r.to(device=p.device, dtype=p.dtype).contiguous()
    r = r.detach().cpu().numpy() if _is_tensor(r) else r
    return np.ascontiguousarray(np.asarray(r).astype(_dtype_name(p)))


def ray_surfel_intersection(p, n, ray_o, ray_d, r=0.1, subdivs=4, ray_near=0.0, ray_far=np.inf, *, device=None):
    """
    Compute intersection between a set of rays and a point cloud converted to surfels (i.e. circular patches oriented
    with the point normals)

    Args:
        p : \\#p by 3 array of vertex positions (each row is a vertex) (float32 / float64)
        n : \\#p by 3 Matrix of vertex normals (each row is a vertex) (p's dtype)
        ray_o : array of shape (#rays, 3) of ray origins (one per row) or a single array of shape (3,) to use (p's dtype)
        ray_d : array of shape (#rays, 3) of ray directions (one per row) (p's dtype)
        r : Array or Scalar describing the size of each geometry element (Either one radius per vertex, or a global size
            for the whole point cloud); cast to p's dtype
        subdivs : Number of times to subdivide the patch geometry for each point (i.e. # tris per circle), 4 to 2^24
        ray_near : an optional floating point value indicating the distance along each ray to start searching (default 0.0)
        ray_far : an optional floating point value indicating the maximum distance along each ray to search (default inf)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        pid : a (#rays,) shaped int32 array of the points hit (-1 for a ray miss)
        t : a (#rays,) shaped array (p's dtype) of the distance along each ray to the hit, in units of |ray_d| (inf for
            missed rays)

    The reference returns (pid, t), although its docstring says (t, pid); the order here is the code's.  Each point is
    the reference's fan of `subdivs` triangles (generate_splat_geometry, "circle"), computed in float32 op by op, with
    cos and sin of the reference's float32 angles taken from the C library in float64 (DESIGN.md §3).  The result is
    ray_mesh_intersection on those fans with pid = face // subdivs: the lexicographic minimum of (t, point, triangle)
    over the triangles hit with ray_near < t <= ray_far, so ties go to the lowest point id.  A point whose fan has a
    non-finite coordinate (a zero normal, a non-finite p or r) is never hit; #p = 0 is allowed and every ray misses.
    Divergences: Embree's arithmetic, its pick among tied triangles and the C library's float cos and sin are not
    reproduced; a 3-element ray_o of any shape is taken in element order.
    """
    r = _validate_radius(p, r)
    form = _form([p, n, ray_o, ray_d], ["p", "n", "ray_o", "ray_d"])
    _check_float(p, "v")
    _check_match(n, "n", p, "v")
    _check_match(ray_o, "ray_o", p, "v")
    _check_match(ray_d, "ray_d", p, "v")
    single, nr = _validate_rays(ray_o, ray_d)
    subdivs = _validate_surfels(p, n, subdivs)
    near, far = _bounds(ray_near, ray_far)
    torch = _torch()

    def call(scene, ot, o_stride, dt, out, dev, stream):
        pt, nt, rt = scene
        _pcu_internal._ray_surfel_intersection_device(dt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), rt.data_ptr(),
                                                      int(pt.shape[0]), subdivs, ot.data_ptr(), o_stride, dt.data_ptr(), nr,
                                                      near, far, *(o.data_ptr() for o in out), dev, stream)

    return _cast(form, [p, n, _radius_like(r, p, form)], ray_o, ray_d, single, nr, device, [((), "int32"), ((), None)], call)


class RaySurfelIntersector(_Prepared):
    """
    Class used to find the intersection between rays and a point cloud converted to surfels (i.e. a point cloud
    represented as circles centered at each point and oriented perpendicularly to each normal).

    The surfels' tree is built once, on the GPU, when the object is made; every `intersect_rays` call only casts its
    rays.  The results are those of `ray_surfel_intersection(p, n, ray_o, ray_d, r, subdivs, ...)`.  `close()` (or
    garbage collection) frees the device memory.
    """
    _what = "the surfels"

    def __init__(self, p, n, r=0.1, subdivs=7, *, device=None):
        """
        Construct a RaySurfelIntersector which can be used to compute the intersection between a set of rays and a
        point cloud converted to circular patches oriented with the point normals

        Args:
            p : \\#p by 3 array of vertex positions (each row is a vertex) (float32 / float64)
            n : \\#p by 3 Matrix of vertex normals (each row is a vertex) (p's dtype)
            r : Array or Scalar describing the size of each geometry element (Either one radius per vertex, or a global
                size for the whole point cloud)
            subdivs : Number of times to subdivide the patch geometry for each point (i.e. # tris per circle)
            device : (keyword only, not in the reference) the GPU of a numpy cloud, see `k_nearest_neighbors`; a cloud
                     of CUDA tensors stays on its device.

        Divergence: r is cast to p's dtype (the reference hands a float64 r to its float32 binding, which refuses it).
        """
        r = _validate_radius(p, r)
        form = _form([p, n], ["p", "n"])
        _check_float(p, "v")
        _check_match(n, "n", p, "v")
        subdivs = _validate_surfels(p, n, subdivs)
        self.p = p
        self.n = n
        self.r = r
        self.num_subdivs = subdivs
        torch = _torch()
        pt, nt, rt = _upload(form, [p, n, _radius_like(r, p, form)], device)
        dev, stream = _call_args(pt)
        handle = _pcu_internal._surfel_prepare_device(pt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), rt.data_ptr(),
                                                      int(pt.shape[0]), subdivs, dev, stream)
        torch.cuda.current_stream(pt.device).synchronize()    # calls on any stream may use the tree
        self._handle, self.device_index = handle, dev

    def intersect_rays(self, ray_o, ray_d, ray_near=0.0, ray_far=np.inf):
        """
        Compute intersection between a set of rays and the point cloud converted to circular patches oriented with the
        point normals

        Args:
            ray_o : array of shape (#rays, 3) of ray origins (one per row) or a single array of shape (3,) to use
                    (float32 / float64)
            ray_d : array of shape (#rays, 3) of ray directions (one per row) (ray_o's dtype)
            ray_near : an optional floating point value indicating the distance along each ray to start searching (default 0.0)
            ray_far : an optional floating point value indicating the maximum distance along each ray to search (default inf)

        Returns:
            pid : a (#rays,) shaped int32 array of the points hit (-1 for a ray miss)
            t : a (#rays,) shaped array (ray_o's dtype) of the distance along each ray to the hit (inf for missed rays)

        Rays given as CUDA tensors must live on the cloud's device; numpy arrays and CPU tensors are copied there.
        """
        return self._intersect(_pcu_internal._ray_surfel_prepared_device, [((), "int32"), ((), None)], ray_o, ray_d, ray_near,
                               ray_far)


def pointcloud_surfel_geometry(p, n, r=0.1, subdivs=7, *, device=None):
    """
    Generate geometry for a point cloud encoded as surfels (i.e. circular patches centered at each point and oriented
    perpendicularly to each normal)

    Args:
        p : \\#p by 3 array of vertex positions (each row is a vertex) (float32 / float64)
        n : \\#p by 3 array of vertex normals (each row is a vertex) (p's dtype)
        r : Array or Scalar describing the size of each geometry element (Either one radius per vertex, or a global size
            for the whole point cloud); cast to p's dtype
        subdivs : Number of times to subdivide the patch geometry for each point (i.e. # tris per circle), 4 to 2^24
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        verts : an array of shape (#p * (subdivs + 1), 3) (p's dtype): point i's rim vertex j at row i (subdivs + 1) + j,
                its centre at row i (subdivs + 1) + subdivs
        faces : an int32 array of shape (#p * subdivs, 3) indexing into verts: (centre, rim j, rim (j + 1) % subdivs)

    The reference's generate_splat_geometry ("circle") in p's dtype, with its mixed precision: the basis and the
    vertices in p's dtype, the rim offsets x0 and y0 rounded to float32 (DESIGN.md §3).  For float32 p the vertices are
    exactly the fans ray_surfel_intersection casts against.
    Divergence: subdivs < 4 raises ValueError as ray_surfel_intersection does (the reference's geometry function does
    not check it).
    """
    r = _validate_radius(p, r)
    form = _form([p, n], ["p", "n"])
    _check_float(p, "v")
    _check_match(n, "n", p, "v")
    subdivs = _validate_surfels(p, n, subdivs)
    torch = _torch()
    m = int(p.shape[0])
    if m == 0:
        if form == "numpy":
            return np.zeros((0, 3), dtype=p.dtype), np.zeros((0, 3), dtype=np.int32)
        if form == "cuda":
            _same_device(p, device)
        return torch.zeros((0, 3), dtype=p.dtype, device=p.device), torch.zeros((0, 3), dtype=torch.int32, device=p.device)
    if m * (subdivs + 1) >= 2 ** 31 - 1:
        raise ValueError("pointcloud_surfel_geometry: int32 faces index at most 2^31 - 2 vertices, got %d points of %d"
                         % (m, subdivs + 1))

    def body(pt, nt, rt, dev, stream):
        v = torch.empty((m * (subdivs + 1), 3), dtype=pt.dtype, device=pt.device)
        f = torch.empty((m * subdivs, 3), dtype=torch.int32, device=pt.device)
        _pcu_internal._surfel_geometry_device(pt.dtype == torch.float64, pt.data_ptr(), nt.data_ptr(), rt.data_ptr(), m, subdivs,
                                              v.data_ptr(), f.data_ptr(), dev, stream)
        return v, f

    return _run(form, [p, n, _radius_like(r, p, form)], device, body)


def pointcloud_sphere_geometry(p, r, num_stacks, num_slices, *, device=None):
    """
    Generate sphere geometry for a point cloud (i.e. one sphere per point)

    Args:
        p : \\#p by 3 array of vertex positions (each row is a vertex) (float32 / float64)
        r : Array or Scalar describing the radius along each axis (Either one radius per vertex, or a global size for
            the whole point cloud); cast to p's dtype
        num_stacks : Number of latitudal subdivisions (at least 1)
        num_slices : Number of longitudal subdivisions (at least 1)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        verts : an array of shape (#p * V, 3) (p's dtype), V = (num_stacks + 1)(num_slices + 1): point i's vertex
                (a, b) at row i V + a (num_slices + 1) + b
        faces : an int32 array of shape (#p * F, 3) indexing into verts, F = 2 (num_stacks - 1) num_slices

    The reference's generate_splat_geometry ("sphere", make_sphere_geometry) for each point, defined in DESIGN.md §3:
    stack a at angle pi / 2 - a (pi / num_stacks) and sector b at angle b (2 pi / num_slices), both in fp64, with the
    C library's cos and sin; xy = r cos(stack), z = r sin(stack), x = xy cos(sector), y = xy sin(sector), and each
    coordinate (p's type)(p_k + x_k) with the sum in fp64 (so float32 p rounds twice).  Faces per sector, stack by
    stack: (k1 + 1, k2, k2 + 1) on the first stack, (k1, k2, k1 + 1) on the last, both in that order in between.  The
    poles and the seam are duplicated, as in the reference.  Zero points give empty (0, 3) arrays.
    Divergences: num_stacks or num_slices below 1 raise ValueError (the reference sizes its faces negatively or writes
    NaN vertices), and so does a p that is not (n, 3); more than 2^31 - 2 vertices in all raise ValueError, where the
    reference's int indices would overflow.
    """
    r = _validate_radius(p, r)
    form = _form([p], ["p"])
    _check_float(p, "v")
    if len(p.shape) != 2 or p.shape[1] != 3:
        raise ValueError("Only 3D inputs are supported: p must have shape (n, 3). Got p.shape = %s." % (tuple(p.shape),))
    stacks, slices = int(num_stacks), int(num_slices)
    if stacks < 1 or slices < 1:
        raise ValueError("pointcloud_sphere_geometry: num_stacks and num_slices must be at least 1, got %d and %d" % (stacks, slices))
    torch = _torch()
    m = int(p.shape[0])
    if m == 0:
        if form == "numpy":
            return np.zeros((0, 3), dtype=p.dtype), np.zeros((0, 3), dtype=np.int32)
        if form == "cuda":
            _same_device(p, device)
        return torch.zeros((0, 3), dtype=p.dtype, device=p.device), torch.zeros((0, 3), dtype=torch.int32, device=p.device)
    nvp, nfp = (stacks + 1) * (slices + 1), 2 * (stacks - 1) * slices
    if m * nvp >= 2 ** 31 - 1:
        raise ValueError("pointcloud_sphere_geometry: int32 faces index at most 2^31 - 2 vertices, got %d points of %d" % (m, nvp))

    def body(pt, rt, dev, stream):
        v = torch.empty((m * nvp, 3), dtype=pt.dtype, device=pt.device)
        f = torch.empty((m * nfp, 3), dtype=torch.int32, device=pt.device)
        _pcu_internal._sphere_geometry_device(pt.dtype == torch.float64, pt.data_ptr(), rt.data_ptr(), m, stacks, slices, v.data_ptr(),
                                              f.data_ptr(), dev, stream)
        return v, f

    return _run(form, [p, _radius_like(r, p, form)], device, body)
