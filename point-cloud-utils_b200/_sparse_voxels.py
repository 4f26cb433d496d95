"""marching_cubes_sparse_voxel_grid and sparse_voxel_grid_boundary -- the reference's names, arguments and outputs (the
reference's src/marching_cubes.cpp and src/sparse_voxel_grid.cpp), computed by csrc/sparse_voxels.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
from . import _pcu_internal
from ._call import _INDEX_KINDS, _check_float, _check_index, _dtype_name, _form, _matrix_shape, _run, _torch

_MAX_ROWS = 2 ** 31 - 1
_OVERFLOW = "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small."


def _aligned(t):
    """t itself, or a copy when its data does not start on a 16-byte boundary (the kernels load cubes 16 bytes at a time)."""
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _validate_marching_cubes(grid_scalars, grid_coordinates, cube_indices):
    """The binding's dtype checks, then its shape checks in its order (src/marching_cubes.cpp:43-71; the rows-mismatch
    message prints grid_coordinates' shape twice, as the reference's does)."""
    _check_float(grid_scalars, "grid_scalars")
    _check_float(grid_coordinates, "grid_coordinates")
    _check_index(cube_indices, "cube_indices", _INDEX_KINDS)
    (cr, cc), (sr, sc), (ir, ic) = _matrix_shape(grid_coordinates), _matrix_shape(grid_scalars), _matrix_shape(cube_indices)
    if cr <= 0:
        raise ValueError("Invalid grid_coordinates has zero rows!")
    if cc != 3:
        raise ValueError("Invalid shape for grid_coordinates must have shape (N, 3) but got (%d, %d)" % (cr, cc))
    if sc != 1:
        raise ValueError("Invalid shape for grid_scalars must have shape (N,) or (N, 1) but got (%d, %d)" % (sr, sc))
    if sr != cr:
        raise ValueError("grid_coordinates and grid_scalars must have the same number of rows but got grid_coordinates.shape = "
                         "(%d, %d), and grid_scalars.shape = (%d, %d)" % (cr, cc, cr, cc))
    if ir == 0:
        raise ValueError("Invalid cube_indices has zero rows!")
    if ic != 8:
        raise ValueError("Invalid shape for cube_indices must have shape (N, 8) but got (%d, %d)" % (ir, ic))
    if cr >= _MAX_ROWS:
        raise ValueError("marching_cubes_sparse_voxel_grid: at most 2^31 - 2 grid vertices are supported, got %d" % cr)
    return cr, ir


def marching_cubes_sparse_voxel_grid(grid_scalars, grid_coordinates, cube_indices, isovalue, *, device=None):
    """
    Run marching cubes on a hex mesh representing a sparse voxel grid (see also sparse_voxel_grid_to_hex_mesh)

    Args:
        grid_scalars : An (n,) shaped array of scalar values at each hex mesh vertex
        grid_coordinates : An (n, 3) shaped array of hex mesh vertices
        cube_indices : An (m, 8) shaped array of indices into grid_coordinates where cube_indices[i, :] are the indices of the 8 points forming the i^th cube
                      Note the cube indices must be ordered as:
                      [[0, 0, 0],
                      [1, 0, 0],
                      [1, 1, 0],
                      [0, 1, 0],
                      [0, 0, 1],
                      [1, 0, 1],
                      [1, 1, 1],
                      [0, 1, 1]]
                      where [i, j, k] indicates the offset along the (x, y, z) axes from the bottom, back, left
                      corner of the cube
        isovalue : Which level set to extract
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v : A (#v, 3) array of triangle mesh vertices
        f : A (#f, 3) array of indices into v where f[i, :] are the indices into vof the 3 points forming the i^th triangle

    See Also:
        sparse_voxel_grid_to_hex_mesh

    Dtypes: grid_scalars float32 / float64 with shape (n,) or (n, 1); grid_coordinates float32 / float64 (v has its
    dtype); cube_indices int32 / int64 / uint32 / uint64 (f has its dtype).  The result is a pure function of the
    inputs, defined in DESIGN.md §3: iso = T(S(isovalue)) and corner k of a cube is above when T(scalar) > iso (NaN is
    not); one vertex per distinct unordered pair of corner indices on a crossing edge, numbered in order of first
    appearance (cube by cube, edge by edge), placed by t = (iso - s_i) / (s_j - s_i), v = g_i + t (g_j - g_i) in T on
    that first edge; faces cube by cube in the order of the generated case table, oriented towards the corners above
    (an SDF negative inside gives outward normals).  The triangles may use other diagonals than libigl's table.
    Raises ValueError("No level set found for isovalue ...") when no edge crosses.
    Divergence: a corner index outside [0, n) raises ValueError (the reference reads out of bounds).
    """
    form = _form([grid_scalars, grid_coordinates, cube_indices], ["grid_scalars", "grid_coordinates", "cube_indices"])
    n, m = _validate_marching_cubes(grid_scalars, grid_coordinates, cube_indices)
    isovalue = float(isovalue)
    torch = _torch()

    def body(st, ct, it, dev, stream):
        it = _aligned(it)
        handle, nv, nf = _pcu_internal._marching_cubes_prepare_device(
            ct.dtype == torch.float64, st.data_ptr(), st.dtype == torch.float64, ct.data_ptr(), n, it.data_ptr(), m,
            _INDEX_KINDS[_dtype_name(cube_indices)], isovalue, dev, stream)
        try:
            if nv == 0:
                raise ValueError("No level set found for isovalue %f" % isovalue)
            v = torch.empty((nv, 3), dtype=ct.dtype, device=ct.device)
            f = torch.empty((nf, 3), dtype=it.dtype, device=ct.device)
            _pcu_internal._marching_cubes_emit_device(handle, v.data_ptr(), f.data_ptr(), dev, stream)
        finally:
            _pcu_internal._marching_cubes_destroy(handle)
        return v, f

    return _run(form, [grid_scalars.reshape(n), grid_coordinates, cube_indices], device, body, index=(cube_indices, [1]))


def sparse_voxel_grid_boundary(grid_coordinates, *, device=None):
    """
    Find the indices of the voxels which lie on the boundary of a sparse voxel grid

    Args:
        grid_coordinates : An (n, 3) shaped integer array of voxels coordinates in the sparse voxel grid
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        boundary_voxels : An (m,) shaped array of indices into grid_coordinates encoding which voxels lie on the boundary

    Bit for bit the reference's (src/sparse_voxel_grid.cpp:463-522): int64 indices in ascending order of the voxels
    one of whose six face neighbours is missing, neighbours found through the reference's 64-bit Morton codes of the
    int32 coordinates (so coordinates alias beyond 21 bits exactly as there; duplicated voxels are each reported).
    Coordinates equal to INT32_MIN or INT32_MAX, beyond the int32 range, and every uint32 / uint64 grid raise
    ValueError("Invalid vertex leads to an overflow integer. ..."), as the reference's range check does.  The shape is
    the reference's (m, 1) squeezed as npe::move squeezes it: (m,), and a 0-d array when m = 1.
    """
    form = _form([grid_coordinates], ["grid_coordinates"])
    _check_index(grid_coordinates, "grid_coordinates", _INDEX_KINDS)
    rows, cols = _matrix_shape(grid_coordinates)
    if rows <= 0:
        raise ValueError("Invalid grid_coordinates has zero rows!")
    if cols != 3:
        raise ValueError("Invalid shape for grid_coordinates must have shape (N, 3) but got (%d, %d)" % (rows, cols))
    if _dtype_name(grid_coordinates) in ("uint32", "uint64"):
        raise ValueError(_OVERFLOW)
    if rows >= _MAX_ROWS:
        raise ValueError("sparse_voxel_grid_boundary: at most 2^31 - 2 voxels are supported, got %d" % rows)
    torch = _torch()

    def body(gt, dev, stream):
        out = torch.empty(rows, dtype=torch.int64, device=gt.device)
        counts = torch.empty(2, dtype=torch.int64, device=gt.device)
        _pcu_internal._sparse_voxel_grid_boundary_device(gt.data_ptr(), rows, _INDEX_KINDS[_dtype_name(grid_coordinates)],
                                                         out.data_ptr(), counts.data_ptr(), dev, stream)
        found, bad = (int(c) for c in counts.cpu().numpy())
        if bad:
            raise ValueError(_OVERFLOW)
        return out[:found].reshape(found, 1)        # the reference's (m, 1) result, squeezed as npe::move squeezes it

    return _run(form, [grid_coordinates], device, body, squeeze=True)
