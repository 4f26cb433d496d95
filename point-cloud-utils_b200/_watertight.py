"""make_mesh_watertight -- the reference's name, arguments and outputs (src/manifold.cpp), computed by
csrc/watertight.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
from . import _pcu_internal
from ._call import _INDEX_KINDS, _dtype_name, _form, _run, _torch, _validate_mesh


def make_mesh_watertight(v, f, resolution=20_000, seed=-1, *, device=None):
    """
    Convert a mesh into a watertight manifold using the [Manifold](https://arxiv.org/abs/1802.01698) algorithm.

    Args:
        v : (#v, 3)-shaped array of mesh vertex positions (one vertex position per row)
        f : (#f, 3)-shaped array of mesh face indexes into v (a row (fi, fj, fk) indicate the 3 vertices of a face)
        resolution : Resolution parameter proportional to the number of output faces. Default 20_000. (It represents the target number of leaf nodes in the octree).
        seed : A random seed to make make the algorithm deterministic. Pass -1 for random. (default -1)
        device: see `k_nearest_neighbors` (keyword only).
    Returns:
        vw : a (#vw, 3)-shaped array of vertices (one per row)
        fw : a (#fw, 3)-shaped array of face indices into vw (one face per row)

    Dtypes: v float32 / float64 (widened exactly to fp64; vw has v's dtype), f int32 / int64 / uint32 / uint64 (fw has
    f's dtype).  The reference's Manifold library is not available, so the result is defined in DESIGN.md §3 and
    computed deterministically: `seed` is accepted and ignored, and two calls give the same bits.  In short: v's
    bounding box, centred and enlarged to a cube 1.4 times its longest side, is split into 2^d voxels per side, d the
    smallest depth in [3, 10] at which at least `resolution` voxels meet a face (voxelize_triangle_mesh's test), else
    10.  The empty voxels connected to the grid's corner are the outside; marching cubes between voxel centres
    extracts the outside's boundary with a triangulation that makes every result a closed, consistently outward-oriented
    2-manifold; then 10 rounds move each vertex towards its closest point on the input, halving the step of every
    vertex of a face that the move would flip.
    The faces are exactly the pre-projection ones, and every vertex ends within s * sqrt(3/2) of the input (s the voxel
    size).  The result is not guaranteed to be free of self-intersections: near a hole wider than a voxel, an open
    input gives a double-sided shell whose two sides can meet after projection.
    Divergences: a non-finite vertex, a face corner outside [0, #v) or a mesh whose vertices all coincide raise
    ValueError.  At depth 10 the call needs about 5.4 GB of device scratch.
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    resolution = float(resolution)
    int(seed)
    torch = _torch()

    def body(vt, ft, dev, stream):
        handle, nv, nf, _ = _pcu_internal._make_mesh_watertight_prepare_device(
            vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)],
            resolution, dev, stream)
        try:
            vw = torch.empty((nv, 3), dtype=vt.dtype, device=vt.device)
            fw = torch.empty((nf, 3), dtype=ft.dtype, device=vt.device)
            _pcu_internal._make_mesh_watertight_emit_device(handle, vw.data_ptr(), fw.data_ptr(), dev, stream)
        finally:
            _pcu_internal._make_mesh_watertight_destroy(handle)
        return vw, fw

    return _run(form, [v, f], device, body, index=(f, [1]))
