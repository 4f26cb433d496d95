"""marching_cubes_sparse_voxel_grid, sparse_voxel_grid_boundary, sparse_voxel_grid_from_pointcloud,
dilate_sparse_voxel_grid, erode_sparse_voxel_grid and sparse_voxel_grid_to_hex_mesh -- the reference's names, arguments
and outputs (the reference's src/marching_cubes.cpp and src/sparse_voxel_grid.cpp, and the sparse-grid wrappers of its
trash/_sparse_voxels.py), computed by csrc/sparse_voxels.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
import numpy as np

from . import _pcu_internal
from ._call import _INDEX_KINDS, _check_float, _check_index, _dtype_name, _form, _matrix_shape, _run, _torch

_MAX_ROWS = 2 ** 31 - 1
_MAX_DILATE = (2 ** 31 - 2) // 26         # dilation ranks 26 neighbour flags per voxel in 32 bits
_MAX_HEX = (2 ** 31 - 2) // 8             # the hex mesh ranks 8 corners per voxel in 32 bits
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


def _size_and_origin(voxel_size, origin):
    """The checks of the reference's sparse-grid wrappers (trash/_sparse_voxels.py), in their order and with their
    messages; returns both as lists of three floats."""
    if np.isscalar(voxel_size):
        voxel_size = np.array([voxel_size] * 3)
    elif len(voxel_size) == 1:
        voxel_size = np.array([np.squeeze(voxel_size).reshape((1,))[0]] * 3)
    elif len(voxel_size) == 3:
        voxel_size = np.squeeze(voxel_size).reshape(3,)
    else:
        raise ValueError("voxel_size must be a scalar or an array/tuple/list of length 3")
    if not np.all(np.isreal(voxel_size)):
        raise ValueError("voxel_size must have a real numeric type")
    if len(origin) == 3:
        origin = np.squeeze(origin).reshape(3,)
    else:
        raise ValueError("origin must be an array/tuple/list of length 3")
    if not np.all(np.isreal(origin)):
        raise ValueError("origin must have a real numeric type")
    return [float(x) for x in voxel_size], [float(x) for x in origin]


def _validate_grid(grid_coordinates, most, name):
    """The dtype check, then validate_sparse_voxel_grid (src/sparse_voxel_grid.cpp:64-74), then the range check that
    every unsigned grid fails, then this package's size limit.  Returns the row count."""
    _check_index(grid_coordinates, "grid_coordinates", _INDEX_KINDS)
    rows, cols = _matrix_shape(grid_coordinates)
    if rows <= 0:
        raise ValueError("Invalid grid_coordinates has zero rows!")
    if cols != 3:
        raise ValueError("Invalid shape for grid_coordinates must have shape (N, 3) but got (%d, %d)" % (rows, cols))
    if _dtype_name(grid_coordinates) in ("uint32", "uint64"):
        raise ValueError(_OVERFLOW)
    if rows > most:
        raise ValueError("%s: at most %d voxels are supported, got %d" % (name, most, rows))
    return rows


def _next_round(t):
    """The rows of a round's result as the next round's binding sees them: npe::move squeezes a one-row result to (3,),
    an (3, 1) column there; a zero-row result fails validate_sparse_voxel_grid."""
    rows = int(t.shape[0])
    if rows == 0:
        raise ValueError("Invalid grid_coordinates has zero rows!")
    if rows == 1:
        raise ValueError("Invalid shape for grid_coordinates must have shape (N, 3) but got (3, 1)")
    return rows


def sparse_voxel_grid_from_pointcloud(points, voxel_size, origin=(0.0, 0.0, 0.0), *, device=None):
    """
    Construct a sparse voxel grid containing a point cloud, optionally returning the voxel index for each point.

    Args:
        points: An (n, 3) shaped array of points (one per row)
        voxel_size: Either a scalar representing the sidelength of a voxel or a triple representing the sidelength of a
                    voxel along each axis.
        origin: The origin of the point cloud corresponding to the bottom, back, left corner of the (0, 0, 0) voxel.
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        grid_coordinates: An (n, 3)-shaped array of integer grid coordinates corresponding to voxels in the sparse grid
        point_to_vox_idx: An (#points,)-shaped array where the i^th entry point_to_vox_idx[i] is the index into
                        grid_coordinates of of the voxel containing points[i]

    Dtypes: points float32 / float64; grid_coordinates int32, point_to_vox int64.  Defined in DESIGN.md §3, as the
    reference's binding computes it (src/sparse_voxel_grid.cpp:78-157): point i's voxel is round((p - o) / s) per axis,
    each operation rounded in fp64 and round() halving away from zero (so the origin is the CENTRE of voxel (0, 0, 0),
    whatever the description above says); an index above INT32_MAX - 1 or below INT32_MIN + 1, infinities included,
    raises ValueError("Invalid vertex leads to an overflow integer. ..."), and a NaN index becomes INT32_MIN, as the
    reference's x86-64 build converts it.  grid_coordinates are the distinct 64-bit Morton codes of the voxels in
    ascending order, decoded (so coordinates alias beyond 21 bits and a NaN axis lands at -2^20), and point_to_vox[i]
    the row of point i's voxel.  Both outputs are squeezed as npe::move squeezes them.  Fewer than 2^31 - 1 points.
    """
    size, origin = _size_and_origin(voxel_size, origin)
    form = _form([points], ["points"])
    _check_float(points, "points")
    rows, cols = _matrix_shape(points)
    if rows <= 0:
        raise ValueError("Invalid points has zero rows!")
    if cols != 3:
        raise ValueError("Invalid shape for points must have shape (N, 3) but got (%d, %d)" % (rows, cols))
    if rows >= _MAX_ROWS:
        raise ValueError("sparse_voxel_grid_from_pointcloud: at most 2^31 - 2 points are supported, got %d" % rows)
    torch = _torch()

    def body(pt, dev, stream):
        handle, u, _ = _pcu_internal._sparse_grid_from_points_device(pt.dtype == torch.float64, pt.data_ptr(), rows, size, origin,
                                                                     dev, stream)
        try:
            grid = torch.empty((u, 3), dtype=torch.int32, device=pt.device)
            point_to_vox = torch.empty(rows, dtype=torch.int64, device=pt.device)
            _pcu_internal._sparse_grid_emit_device(handle, grid.data_ptr(), point_to_vox.data_ptr(), dev, stream)
        finally:
            _pcu_internal._sparse_grid_destroy(handle)
        return grid, point_to_vox

    return _run(form, [points], device, body, squeeze=True)


def dilate_sparse_voxel_grid(grid_coordinates, count=1, *, device=None):
    """
    Perform binary dilation on a sparse voxel grid, using a 3x3 filter of ones applied count times.
    i.e. convolve the filter:
        [[1, 1, 1],
         [1, 1, 1],
         [1, 1, 1]]
    with the sparse voxel grid.

    Args:
        grid_coordinates: An (n, 3) shaped integer array of voxels coordinates in the sparse voxel grid
        count: The number of iterations of binary dilation to run
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        dilated_grid_coordinates: An (m, 3) integer array encoding the coordinates of the sparse voxel grid after dilation

    Dtypes: grid_coordinates int32 / int64 (uint32 / uint64 grids fail the range check); the result has its dtype.
    Defined in DESIGN.md §3: one round returns the input rows verbatim (duplicates included), then the distinct
    64-bit Morton codes code + offset, over every voxel and each of its 26 neighbour offsets, that are not among the
    input's codes, in ascending order, decoded.  count rounds feed each round's result to the next; count <= 0 returns
    grid_coordinates itself, unchecked.  Coordinates outside [INT32_MIN + 1, INT32_MAX - 1] raise ValueError("Invalid
    vertex leads to an overflow integer. ..."); neighbours wrap at +-2^20 and alias beyond 21 bits, as the reference's
    Morton arithmetic does.  At most 82 595 524 voxels per round.
    Divergence: the reference's offset table repeats (-1, 0, 1), (0, 0, 1) and (1, 0, 1) in place of (-1, 1, 1),
    (0, 1, 1) and (1, 1, 1), so it never adds those three neighbours; here all 26 are used (the 3 x 3 x 3 filter the
    description promises), and the result is a superset of the reference's.
    """
    if count <= 0:
        return grid_coordinates
    form = _form([grid_coordinates], ["grid_coordinates"])
    rows = _validate_grid(grid_coordinates, _MAX_DILATE, "dilate_sparse_voxel_grid")
    kind = _INDEX_KINDS[_dtype_name(grid_coordinates)]
    torch = _torch()

    def body(gt, dev, stream):
        n = rows
        for r in range(count):
            if r > 0:
                n = _next_round(gt)
                if n > _MAX_DILATE:
                    raise ValueError("dilate_sparse_voxel_grid: at most %d voxels are supported, got %d" % (_MAX_DILATE, n))
            handle, total, _ = _pcu_internal._sparse_grid_dilate_prepare_device(gt.data_ptr(), n, kind, dev, stream)
            try:
                out = torch.empty((total, 3), dtype=gt.dtype, device=gt.device)
                _pcu_internal._sparse_grid_emit_device(handle, out.data_ptr(), 0, dev, stream)
            finally:
                _pcu_internal._sparse_grid_destroy(handle)
            gt = out
        return gt

    return _run(form, [grid_coordinates], device, body, squeeze=True)


def erode_sparse_voxel_grid(grid_coordinates, count=1, *, device=None):
    """
    Perform binary erosion on a sparse voxel grid, using a 3x3 filter of ones applied count times.
    i.e. take the negation of the convolution of the filter:
        [[1, 1, 1],
         [1, 1, 1],
         [1, 1, 1]]
    with the sparse voxel grid.

    Args:
        grid_coordinates: An (n, 3) shaped integer array of voxels coordinates in the sparse voxel grid
        count: The number of iterations of binary erosion to run
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        eroded_grid_coordinates: An (m, 3) integer array encoding the coordinates of the sparse voxel grid after erosion

    Dtypes: grid_coordinates int32 / int64 (uint32 / uint64 grids fail the range check); the result has its dtype.
    Defined in DESIGN.md §3: one round keeps, verbatim and in input order, the rows all 26 of whose neighbours'
    64-bit Morton codes are among the input's codes.  count rounds feed each round's result to the next (a round on an
    empty result raises "Invalid grid_coordinates has zero rows!", as in the reference); count <= 0 returns
    grid_coordinates itself, unchecked.  Range check, wrap and aliasing as in dilate_sparse_voxel_grid.  Fewer than
    2^31 - 1 voxels.
    Divergence: the reference's offset table never tests (-1, 1, 1), (0, 1, 1) or (1, 1, 1) (see
    dilate_sparse_voxel_grid); here all 26 neighbours are required, and the result is a subset of the reference's.
    """
    if count <= 0:
        return grid_coordinates
    form = _form([grid_coordinates], ["grid_coordinates"])
    rows = _validate_grid(grid_coordinates, _MAX_ROWS - 1, "erode_sparse_voxel_grid")
    kind = _INDEX_KINDS[_dtype_name(grid_coordinates)]
    torch = _torch()

    def body(gt, dev, stream):
        n = rows
        counts = torch.empty(2, dtype=torch.int64, device=gt.device)
        for r in range(count):
            if r > 0:
                n = _next_round(gt)
            out = torch.empty((n, 3), dtype=gt.dtype, device=gt.device)
            _pcu_internal._sparse_grid_erode_device(gt.data_ptr(), n, kind, out.data_ptr(), counts.data_ptr(), dev, stream)
            kept, bad = (int(c) for c in counts.cpu().numpy())
            if bad:
                raise ValueError(_OVERFLOW)
            gt = out[:kept]
        return gt

    return _run(form, [grid_coordinates], device, body, squeeze=True)


def _numpy_dtype(dtype):
    """A numpy dtype, or the numpy dtype of a torch dtype."""
    torch = _torch()
    return torch.empty(0, dtype=dtype).numpy().dtype if isinstance(dtype, torch.dtype) else np.dtype(dtype)


def sparse_voxel_grid_to_hex_mesh(grid_coordinates, voxel_size=1.0, origin=(0.0, 0.0, 0.0), dtype=np.float64, *, device=None):
    """
    Convert a sparse voxel grid where the voxel indices represent the centers of each voxel coordinate into a
    hexahedral mesh.

    i.e. a pair of arrays (v, c) where v has shape (n, 3) and each row is a vertex position
         and c has shape (m, 8) where the i^th row c[i, :] are the indices into v of the 8 corners of the i^th cube

    Args:
        grid_coordinates: An (n, 3) shaped integer array of voxels coordinates in the sparse voxel grid
        voxel_size: Either a scalar encoding the length of one voxel along an axis or a triple encoding the length of a
                    voxel on each of 3 axes
        origin: A triple encoding a global offset for the hex mesh (i.e. all vertices will have origin added to them).
                Default is (0.0, 0.0, 0.0).
        dtype: The scalar type of vertices to return.
            Default is np.float64.
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        vertices: An (n, 3) shaped array where each row vertices[i, :] is a vertex position in the hex mesh
        cubes: An (m, 8) shaped array of indices into v where each row cubes[j, :] are indices of the 8 points forming
            the j^th cube

    See Also:
        marching_cubes_sparse_voxel_grid

    Dtypes: grid_coordinates int32 / int64 (uint32 / uint64 grids fail the range check); cubes int64; vertices in
    dtype (a numpy dtype, or a torch dtype for tensors).  Defined in DESIGN.md §3: voxel i's corners are the 64-bit
    Morton codes code_i + (0,0,0), (1,0,0), (1,1,0), (0,1,0), (0,0,1), (1,0,1), (1,1,1), (0,1,1) (the corner order
    marching_cubes_sparse_voxel_grid expects); the vertices are the distinct corner codes in ascending order, decoded
    to c and placed at ((double)c * s + o) - 0.5 * s per axis, each operation rounded in fp64, then converted to dtype
    (float32 and float64 by the kernel, with one rounding; any other dtype from the fp64 result, as numpy's astype
    converts it); cubes[i, k] is the row of voxel i's corner k.  A zero-row grid returns (0, 3) and (0, 8) arrays, as
    the reference's binding does; coordinates outside [INT32_MIN + 1, INT32_MAX - 1] raise ValueError("Invalid vertex
    leads to an overflow integer. ...").  Fewer than 2^28 voxels.  cubes is squeezed as npe::move squeezes it.
    Divergences: the reference subtracts half of the x voxel size on every axis; here each axis subtracts half its own
    size (the same bits whenever the three sizes are equal).  A grid whose column count is not 3 raises the shape
    ValueError (the reference reads out of bounds).
    """
    size, origin = _size_and_origin(voxel_size, origin)
    form = _form([grid_coordinates], ["grid_coordinates"])
    _check_index(grid_coordinates, "grid_coordinates", _INDEX_KINDS)
    dt = _numpy_dtype(dtype)
    torch = _torch()
    rows, _ = _matrix_shape(grid_coordinates)
    if rows <= 0:
        if form == "numpy":
            return np.zeros((0, 3), dt), np.zeros((0, 8), np.int64)
        tdt = torch.from_numpy(np.zeros(0, dt)).dtype
        dev = grid_coordinates.device
        return torch.empty((0, 3), dtype=tdt, device=dev), torch.empty((0, 8), dtype=torch.int64, device=dev)
    rows = _validate_grid(grid_coordinates, _MAX_HEX, "sparse_voxel_grid_to_hex_mesh")
    kind = _INDEX_KINDS[_dtype_name(grid_coordinates)]
    f32 = dt == np.float32

    def body(gt, dev, stream):
        handle, nv, _ = _pcu_internal._sparse_grid_hex_prepare_device(gt.data_ptr(), rows, kind, size, origin, not f32, dev, stream)
        try:
            v = torch.empty((nv, 3), dtype=torch.float32 if f32 else torch.float64, device=gt.device)
            cubes = torch.empty((rows, 8), dtype=torch.int64, device=gt.device)
            _pcu_internal._sparse_grid_emit_device(handle, v.data_ptr(), cubes.data_ptr(), dev, stream)
        finally:
            _pcu_internal._sparse_grid_destroy(handle)
        return v, cubes

    v, cubes = _run(form, [grid_coordinates], device, body, squeeze=True)
    if dt not in (np.float32, np.float64):
        # the reference's ret_v.astype(dtype), from the fp64 vertices, by numpy (a torch cast from fp64 to fp16 rounds
        # twice, through fp32)
        if form == "numpy":
            v = v.astype(dt)
        else:
            v = torch.from_numpy(v.cpu().numpy().astype(dt)).to(v.device)
    return v, cubes
