"""voxelize_triangle_mesh, flood_fill_3d and voxel_grid_geometry -- the reference's names, arguments and outputs (the
reference's point_cloud_utils/_voxels.py, src/voxelize_triangle_mesh.cpp, src/flood_fill_3d.cpp,
point_cloud_utils/_point_cloud_geometry.py and src/mesh_for_voxels.cpp), computed by csrc/voxelize.cuh and
csrc/sparse_voxels.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages and in its order, before any
device call."""
import numpy as np

from . import _pcu_internal
from ._call import _INDEX_KINDS, _check_index, _dtype_name, _form, _matrix_shape, _run, _torch, _validate_mesh

_GRID_KINDS = {"int32": 0, "int64": 1, "float32": 2, "float64": 3}
_MAX_VOXELS = 2 ** 31
_MAX_CUBES = 2 ** 28                      # voxel_grid_geometry's int32 faces index 8 vertices per voxel


def _coord3d_to_array(coord, dtype=np.float64):
    """The reference's point_cloud_utils/_point_cloud_geometry.py:7-14."""
    if not hasattr(coord, "__len__") or len(coord) != 3:
        raise ValueError("expected 3D coordinate")
    if isinstance(coord, np.ndarray):
        return np.array([c.item() for c in coord], dtype=dtype)
    return np.array([c for c in coord], dtype=dtype)


def _number_or_coord3d_to_array(coord_or_number, dtype=np.float64):
    """The reference's point_cloud_utils/_point_cloud_geometry.py:17-21."""
    if isinstance(coord_or_number, (float, int)):
        return np.array([coord_or_number] * 3, dtype=dtype)
    return _coord3d_to_array(coord_or_number, dtype=dtype)


def flood_fill_3d(grid, start_coord, fill_value, *, device=None):
    """
    Flood fill a 3D grid starting from_start_coord with fill_value. This will return a
    copy of grid where the region in the input grid which is connected to start_coord
    and shares the value of start_coord is set to fill_value.

    Args:
        grid (np.ndarray): [w, h, d] array of scalars as input to the flood fill
        start_coord: (i, j, k) integer coordinate to start the flood fill
        fill_value: scalar value to flood fill
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        _type_: A flood filled copy of grid where all voxels which are connected to start_coord
                are set to fill_value

    Dtypes: grid int32 / int64 / float32 / float64; the result has grid's dtype and shape.  Bit for bit the reference's
    (src/flood_fill_3d.cpp): the region is the connected component of the seed among the voxels equal (IEEE ==) to the
    seed's value, so a NaN seed fills nothing and -0.0 matches 0.0.  Neighbours are those of the reference's linear
    offsets in the C-ordered grid: voxel o is adjacent to o +- 1, o +- d and o +- h d whenever that index lies in
    [0, w h d), so a step past z = d - 1 continues at z = 0 of the next y row, and past y = h - 1 at y = 0 of the next
    x slab.  The fill is float(fill_value) converted to the grid's dtype as the reference's x86 build converts it:
    integers truncate toward zero, and NaN or out-of-range values become INT32_MIN / INT64_MIN; float32 rounds to
    nearest.
    Divergences: when the converted fill equals the seed's value the result is an unchanged copy (the reference never
    returns); grids of 2^31 voxels or more raise ValueError (the reference's int offsets overflow).
    """
    start_coord = _coord3d_to_array(start_coord, np.int32)
    sizes = tuple(int(s) for s in grid.shape)
    if len(sizes) != 3:
        raise ValueError("grid must have shape [w, h, d]")
    form = _form([grid], ["grid"])
    _check_index(grid, "grid", _GRID_KINDS)
    if any(not (0 <= int(c) < s) for c, s in zip(start_coord, sizes)):
        raise ValueError("seed point must be inside grid")
    w, h, d = sizes
    if w * h * d >= _MAX_VOXELS:
        raise ValueError("flood_fill_3d: grids of at most 2^31 - 1 voxels are supported, got %d x %d x %d" % (w, h, d))
    fill = float(fill_value)
    torch = _torch()

    def body(gt, dev, stream):
        out = torch.empty_like(gt)
        _pcu_internal._flood_fill_3d_device(gt.data_ptr(), _GRID_KINDS[_dtype_name(grid)], w, h, d, int(start_coord[0]),
                                            int(start_coord[1]), int(start_coord[2]), fill, out.data_ptr(), dev, stream)
        return out

    return _run(form, [grid], device, body)


def voxelize_triangle_mesh(v, f, voxel_size, voxel_origin, *, device=None):
    """
    Return ijk coordinates of voxels which intersect the given mesh.
    Each voxel is assumed to have size voxel_size (scalar or triple of floats) and
    the (0, 0, 0) voxel is centred at voxel_origin

    Args:
        v (np.ndarray): [num_vertices, 3] array of triangle mesh vertices
        f (np.ndarray): [num_faces, 3] array of face indexes into v
        voxel_size: A float or triple specifying the size of each voxel
        voxel_origin: A float or triple specifying the position of the centre of the (0, 0, 0) voxel
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        ijk: [num_vox, 3] array of integer ijk coordinates for each voxel intersecting the mesh

    Dtypes: v float32 / float64 (widened exactly to fp64), f int32 / int64 / uint32 / uint64; ijk is int32.  Defined in
    DESIGN.md §3, as the reference computes it (src/voxelize_triangle_mesh.cpp): voxel (i, j, k) is the box centred
    at o + (i, j, k) * s (each product and sum rounded in fp64; the reference's docstring calls o the bottom-back-left
    corner, its code centres the box there) with half-size s / 2.  Each face tests the voxels of
    [floor((min - o) / s), ceil((max - o) / s)] per axis with the reference's triBoxOverlap, operation for operation in
    fp64.  The result is the reference wrapper's morton_decode(np.unique(morton_encode(ijk))): the distinct voxels in
    ascending 64-bit Morton order, so coordinates beyond 21 bits alias exactly as there.  When no voxel is accepted,
    the reference's morton_encode error is raised: "pts must be an array of shape [n, 3] but got an empty array".
    Divergence: the reference tests only x = floor((min_x - o_x) / s_x) of each face's candidates (its x loop runs
    from that bound to itself), so most faces lose voxels; here x runs over the whole range, as y and z do.  The
    result is a superset of the reference's, and equal to it when every face lies within the x extent of that voxel.
    Further divergences: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds); a
    non-finite vertex, or index bounds that are not finite or fall outside [INT32_MIN, INT32_MAX - 1], raise
    ValueError (the reference's int conversion is undefined there, and an upper bound of INT32_MAX never ends its
    loop); candidate counts are 64-bit and a total that overflows int64 raises ValueError.
    """
    voxel_origin = _coord3d_to_array(voxel_origin, np.float64)
    voxel_size = _number_or_coord3d_to_array(voxel_size, np.float64)
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    if voxel_size[0] <= 0.0 or voxel_size[1] <= 0.0 or voxel_size[2] <= 0.0:
        raise ValueError("Invalid voxel size")
    torch = _torch()

    def body(vt, ft, dev, stream):
        handle, n, _ = _pcu_internal._voxelize_prepare_device(vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]),
                                                              ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)],
                                                              voxel_size.tolist(), voxel_origin.tolist(), dev, stream)
        try:
            ijk = torch.empty((n, 3), dtype=torch.int32, device=vt.device)
            _pcu_internal._voxelize_emit_device(handle, ijk.data_ptr(), dev, stream)
        finally:
            _pcu_internal._voxelize_destroy(handle)
        return ijk

    return _run(form, [v, f], device, body)


def voxel_grid_geometry(ijk, voxel_size=np.array((1., 1., 1.)), voxel_origin=np.array((0., 0., 0.)), gap_fraction=0.0, *,
                        device=None):
    """
    Generate a triangle mesh of cubes for voxel coordinates ijk. The [0, 0, 0] voxel has its
    low corner at voxel_origin and each voxel has voxel_size.

    Args:
        ijk np.ndarray: [num_voxels, 3] array of integer voxel coordinates
        voxel_size: Float or triple representing the size of each voxel.
                    Defaults to np.array((1., 1., 1.)).
        voxel_origin: Low corner of the [0, 0, 0] voxel. Defaults to np.array((0., 0., 0.)).
        gap_fraction: Fraction of a voxel to leave as a gap between voxels (default 0.0)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v: Numpy array of vertices for the cube mesh
        f: Numpy array of faces for the cube mesh

    Dtypes: ijk int32 / int64 / uint32 / uint64; v float32 (8 n, 3), f int32 (12 n, 3).  Bit for bit the reference's
    (src/mesh_for_voxels.cpp): voxel i contributes 8 vertices and 12 faces in the order of the reference's tables;
    component k of table corner c (0 or 1) is float((((c * (1 - gap) + 0.5 gap) + ijk_k) * s_k) + o_k), each
    operation rounded in fp64 (uint64 indices convert as unsigned), and face j of voxel i is the table's face j plus
    8 i.  The origin is therefore the LOW corner of voxel (0, 0, 0), as the reference's code computes it (its
    description says the centre): cubes drawn for voxelize_triangle_mesh's output with the same origin, which centres
    voxel (i, j, k) at o + (i, j, k) s, sit half a voxel off.  A voxel size <= 0 raises ValueError("Voxel size must be
    positive") (NaN passes, as in the reference).  At most 2^28 voxels (the int32 face indices overflow beyond).
    """
    voxel_origin = _coord3d_to_array(voxel_origin, dtype=np.float64)
    voxel_size = _number_or_coord3d_to_array(voxel_size, dtype=np.float64)
    form = _form([ijk], ["ijk"])
    _check_index(ijk, "ijk", _INDEX_KINDS)
    gap_fraction = float(gap_fraction)
    rows, cols = _matrix_shape(ijk)
    if rows == 0:
        raise ValueError("Invalid input point cloud with zero points: points must have shape (n, 3) (n > 0). "
                         "Got points.shape =(%d, %d)." % (rows, cols))
    if cols != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). "
                         "Got points.shape =(%d, %d)." % (rows, cols))
    if voxel_size[0] <= 0.0 or voxel_size[1] <= 0.0 or voxel_size[2] <= 0.0:
        raise ValueError("Voxel size must be positive")
    if rows > _MAX_CUBES:
        raise ValueError("voxel_grid_geometry: at most 2^28 voxels are supported, got %d" % rows)
    torch = _torch()

    def body(it, dev, stream):
        v = torch.empty((8 * rows, 3), dtype=torch.float32, device=it.device)
        f = torch.empty((12 * rows, 3), dtype=torch.int32, device=it.device)
        _pcu_internal._voxel_grid_geometry_device(it.data_ptr(), rows, _INDEX_KINDS[_dtype_name(ijk)], voxel_size.tolist(),
                                                  voxel_origin.tolist(), gap_fraction, v.data_ptr(), f.data_ptr(), dev, stream)
        return v, f

    return _run(form, [ijk], device, body, squeeze=True)
