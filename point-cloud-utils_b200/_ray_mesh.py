"""ray_mesh_intersection and RayMeshIntersector -- the reference's names, arguments and outputs (the reference's
src/ray_mesh_intersection.cpp and point_cloud_utils/_ray_mesh_intersector.py), computed by csrc/raycast.cuh on the tree
of csrc/meshquery.cuh.

Input forms and validation follow _call.py: numpy arrays in -> numpy out; CUDA torch tensors in -> CUDA tensors
out; CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
import numpy as np

from . import _pcu_internal
from ._call import (_INDEX_KINDS, _call_args, _check_float, _check_index, _check_match, _dtype_name, _form, _matrix_shape,
                    _raise_bad, _run, _same_device, _torch, _upload, _validate_mesh)


def _validate_rays(ray_o, ray_d):
    """src/ray_mesh_intersection.cpp:117-135: a 3-element ray_o is one origin for every ray, else the row counts must
    match and ray_o must have 3 columns; ray_d must have 3 columns.  Returns (single origin, number of rays)."""
    single = int(np.prod(tuple(ray_o.shape))) == 3
    (orows, ocols), (drows, dcols) = _matrix_shape(ray_o), _matrix_shape(ray_d)
    if not single and orows != drows:
        raise ValueError("ray_o and ray_d must have the same number of rows (one ray origin per ray direction). "
                         "(Note: ray_o can have one row to use the same origin for all directions)")
    if not single and ocols != 3:
        raise ValueError("Invalid shape for ray_o must have shape (N, 3) but got (%d, %d)." % (orows, ocols))
    if dcols != 3:
        raise ValueError("Invalid shape for ray_d must have shape (N, 3) but got (%d, %d)." % (drows, dcols))
    return single, drows


def _bounds(ray_near, ray_far):
    """The reference hands both to Embree as float."""
    return float(np.float32(ray_near)), float(np.float32(ray_far))


def _origins(ot, single):
    """(origins, o_stride) of a contiguous ray_o: a single origin is its 3 elements in order, with stride 0."""
    return (ot.reshape(3), 0) if single else (ot, 3)


def _cast(form, scene, ray_o, ray_d, single, n, device, outs, call):
    """_run for rays.  `scene` holds the arrays that are uploaded with the rays (none for a prepared tree); `outs` gives
    one (shape after #rays, dtype name) per output, None standing for the rays' dtype; call(scene tensors, origins,
    o_stride, directions, outputs, device index, stream) makes the native call on contiguous CUDA tensors.  Zero rays
    return empty outputs without a launch."""
    torch = _torch()
    outs = [(tail, name or _dtype_name(ray_d)) for tail, name in outs]
    if n == 0:
        if form == "numpy":
            return tuple(np.zeros((0,) + tail, dtype=name) for tail, name in outs)
        if form == "cuda":
            _same_device(ray_d, device)
        return tuple(torch.zeros((0,) + tail, dtype=getattr(torch, name), device=ray_d.device) for tail, name in outs)

    def body(*args):
        *scene_t, ot, dt, dev, stream = args
        ot, o_stride = _origins(ot, single)
        dt = dt.reshape(n, 3)
        out = tuple(torch.empty((n,) + tail, dtype=getattr(torch, name), device=dt.device) for tail, name in outs)
        call(scene_t, ot, o_stride, dt, out, dev, stream)
        return out

    return _run(form, list(scene) + [ray_o, ray_d], device, body)


def ray_mesh_intersection(v, f, ray_o, ray_d, ray_near=0.0, ray_far=np.inf, *, device=None):
    """
    Compute intersection between a set of rays and a triangle mesh

    Args:
        v : \\#v by 3 array of vertex positions (each row is a vertex) (float32 / float64)
        f : \\#f by 3 Matrix of face (triangle) indices (int32 / int64 / uint32 / uint64)
        ray_o : array of shape (#rays, 3) of ray origins (one per row) or a single array of shape (3,) to use (v's dtype)
        ray_d : array of shape (#rays, 3) of ray directions (one per row) (v's dtype)
        ray_near : an optional floating point value indicating the distance along each ray to start searching (default 0.0)
        ray_far : an optional floating point value indicating the maximum distance along each ray to search (default inf)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        f_id : an array of shape (#rays,) representing the face id hit by each ray (f's dtype; -1 cast to it on a miss)
        bc : an array of shape (#rays, 3) where each row is the barycentric coordinates within each face of the ray
             intersection (v's dtype; 0 on a miss)
        t : the distance along each ray to the intersection, in units of |ray_d| (v's dtype; inf on a miss)

    Mirrors the reference's src/ray_mesh_intersection.cpp (Embree).  The result is a pure function of (v, f, o_i, d_i,
    ray_near, ray_far), defined in DESIGN.md §3: everything is rounded to float32 as the reference does, every face is
    tested with the watertight test of Woop, Benthin and Wald (2013) on both of its sides, and the chosen face is the
    lexicographic minimum of (t, face index) over the faces hit with ray_near < t <= ray_far.  bc = (1 - b1 - b2, b1, b2).
    Divergences: Embree's choice among tied faces and its arithmetic are not reproduced; a face corner outside [0, #v)
    raises ValueError (the reference reads out of bounds); a 3-element ray_o of any shape is taken in element order (the
    reference reads ray_o(0, 0), ray_o(1, 0), ray_o(2, 0)); a zero or non-finite origin or direction misses.
    """
    form = _form([v, f, ray_o, ray_d], ["v", "f", "ray_o", "ray_d"])
    _check_float(v, "v")
    _check_index(f, "f", _INDEX_KINDS)
    _check_match(ray_o, "ray_o", v, "v")
    _check_match(ray_d, "ray_d", v, "v")
    single, n = _validate_rays(ray_o, ray_d)
    _validate_mesh(v, f, tuple(_INDEX_KINDS))
    near, far = _bounds(ray_near, ray_far)
    torch = _torch()
    # numpy and CPU inputs: f_id travels as the signed type of f's width, as f does, and is viewed back as f's dtype
    fdt = _dtype_name(f) if form == "cuda" else _dtype_name(f).replace("u", "")

    def call(scene, ot, o_stride, dt, out, dev, stream):
        vt, ft = scene
        bad = torch.empty(1, dtype=torch.int64, device=vt.device)
        _pcu_internal._ray_mesh_intersection_device(vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(),
                                                    int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)], ot.data_ptr(), o_stride,
                                                    dt.data_ptr(), n, near, far, *(o.data_ptr() for o in out), bad.data_ptr(),
                                                    dev, stream)
        _raise_bad(bad)

    fidx, bc, t = _cast(form, [v, f], ray_o, ray_d, single, n, device, [((), fdt), ((3,), None), ((), None)], call)
    return fidx.view(f.dtype), bc, t


class _Prepared:
    """A tree built once and held through a native handle: what RayMeshIntersector and RaySurfelIntersector share.
    `_what` names the tree in messages; __init__ sets `_handle` and `device_index`."""
    _handle = 0

    def close(self):
        if self._handle:
            _pcu_internal._mesh_destroy(self._handle)
            self._handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:   # interpreter shutdown
            pass

    def _intersect(self, native, outs, ray_o, ray_d, ray_near, ray_far):
        """intersect_rays: the checks in the order their errors win, then `native` on the handle, outputs as `outs`."""
        if not self._handle:
            raise ValueError("the %s has been closed" % type(self).__name__)
        form = _form([ray_o, ray_d], ["ray_o", "ray_d"])
        _check_float(ray_o, "ray_o")
        _check_match(ray_d, "ray_d", ray_o, "ray_o")
        single, n = _validate_rays(ray_o, ray_d)
        near, far = _bounds(ray_near, ray_far)
        if form == "cuda" and (ray_o.device.index or 0) != self.device_index:
            raise ValueError("the rays live on %s, %s on cuda:%d" % (ray_o.device, self._what, self.device_index))

        def call(_, ot, o_stride, dt, out, dev, stream):
            native(dt.dtype == _torch().float64, self._handle, ot.data_ptr(), o_stride, dt.data_ptr(), n, near, far,
                   *(o.data_ptr() for o in out), dev, stream)

        return _cast(form, [], ray_o, ray_d, single, n, self.device_index, outs, call)


class RayMeshIntersector(_Prepared):
    """
    Class used to find the intersection between rays and a triangle mesh.

    The mesh's tree is built once, on the GPU, when the object is made; every `intersect_rays` call only casts its
    rays.  The results are those of `ray_mesh_intersection(mesh_v, mesh_f, ...)` (f_id as int32).  `close()` (or garbage
    collection) frees the device memory.
    """
    _what = "the mesh"

    def __init__(self, mesh_v, mesh_f, *, device=None):
        """
        Create a RayMeshIntersector object which can be used to do ray/mesh queries with a triangle mesh.

        Args:
          mesh_v : \\#v by 3 array of vertex positions (each row is a vertex) (float32 / float64)
          mesh_f : \\#f by 3 Matrix of face (triangle) indices (int32 / int64 / uint32 / uint64)
          device : (keyword only, not in the reference) the GPU of a numpy mesh, see `k_nearest_neighbors`; a mesh of
                   CUDA tensors stays on its device.

        Divergence: a face corner outside [0, #v) raises ValueError (the reference validates nothing here).
        """
        form = _form([mesh_v, mesh_f], ["mesh_v", "mesh_f"])
        _validate_mesh(mesh_v, mesh_f, tuple(_INDEX_KINDS))
        self.v = mesh_v
        self.f = mesh_f
        torch = _torch()
        vt, ft = _upload(form, [mesh_v, mesh_f], device)
        dev, stream = _call_args(vt)
        bad = torch.empty(1, dtype=torch.int64, device=vt.device)
        handle = _pcu_internal._mesh_prepare_device(vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(),
                                                    int(ft.shape[0]), _INDEX_KINDS[_dtype_name(mesh_f)], bad.data_ptr(), dev,
                                                    stream)
        try:
            _raise_bad(bad)      # also waits for the build, so calls on any stream may use the tree
        except ValueError:
            _pcu_internal._mesh_destroy(handle)
            raise
        self._handle, self.device_index = handle, dev

    def intersect_rays(self, ray_o, ray_d, ray_near=0.0, ray_far=np.inf):
        """
        Compute intersection between a set of rays and the triangle mesh enclosed in this class

        Args:
          ray_o : array of shape (\\#rays, 3) of ray origins (one per row) or a single array of shape (3,) to use
                  (float32 / float64)
          ray_d : array of shape (\\#rays, 3) of ray directions (one per row) (ray_o's dtype)
          ray_near : an optional floating point value indicating the distance along each ray to start searching (default 0.0)
          ray_far : an optional floating point value indicating the maximum distance along each ray to search (default inf)

        Returns:
          f_id : an array of shape (#rays,) representing the face id hit by each ray (int32; -1 on a miss)
          bc : an array of shape (#rays, 3) where each row is the barycentric coordinates within each face of the ray
               intersection (ray_o's dtype)
          t : the distance along each ray to the intersection (ray_o's dtype; inf on a miss)

        Rays given as CUDA tensors must live on the mesh's device; numpy arrays and CPU tensors are copied there.
        """
        return self._intersect(_pcu_internal._ray_mesh_prepared_device, [((), "int32"), ((3,), None), ((), None)], ray_o, ray_d,
                               ray_near, ray_far)
