"""deduplicate_point_cloud / deduplicate_mesh_vertices -- the reference's names, arguments and return conventions
(/root/reference/src/remove_duplicates.cpp:85-176), computed by csrc/dedup.cuh (keys -> radix sort -> run heads).

Inputs and results take the forms of _call.py.  float32 / float64 points, int32 / int64 faces."""
import numpy as _np

from . import _pcu_internal
from ._call import _check_float, _check_index, _form, _is_tensor, _run, _same_device, _torch


def _dedup(points, faces, epsilon, device, pname):
    """(points, faces or None, svi, svj) of the deduplicated cloud or mesh."""
    if not _is_tensor(points):       # lists work, as in the reference
        points, faces = _np.asarray(points), None if faces is None else _np.asarray(faces)
    arrays = [points] if faces is None else [points, faces]
    form = _form(arrays, [pname, "f"])
    _check_float(points, pname)
    if len(points.shape) != 2 or points.shape[1] != 3:                    # validate_point_cloud, src/common/common.h:68-73
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =" + str(tuple(points.shape)) + ".")
    if faces is not None:
        _check_index(faces, "f", ("int32", "int64"))
        if len(faces.shape) != 2:
            raise ValueError("Invalid shape for faces, must be (m, c) but got " + str(tuple(faces.shape)))
    n = int(points.shape[0])
    torch = _torch()
    if n == 0:          # the reference accepts an empty cloud and returns empty arrays
        if form == "numpy":
            empty = _np.zeros(0, dtype=_np.int32)
            return points.copy(), None if faces is None else faces.copy(), empty, empty.copy()
        if form == "cuda":
            _same_device(points, device)
        empty = torch.zeros(0, dtype=torch.int32, device=points.device)
        return (points.detach().contiguous().clone(), None if faces is None else faces.detach().contiguous().clone(), empty,
                empty.clone())

    def body(pts, *rest):
        fcs, (dev, stream) = (rest[0] if faces is not None else None), rest[-2:]
        nf, cols = (fcs.shape[0], fcs.shape[1]) if fcs is not None else (0, 0)
        out_p = torch.empty((n, 3), dtype=pts.dtype, device=pts.device)
        svi = torch.empty(n, dtype=torch.int32, device=pts.device)
        svj = torch.empty(n, dtype=torch.int32, device=pts.device)
        out_f = torch.empty((nf, cols), dtype=fcs.dtype, device=pts.device) if fcs is not None else None
        counts = torch.empty(3, dtype=torch.int64, device=pts.device)
        _pcu_internal._deduplicate_device(pts.dtype == torch.float64, pts.data_ptr(), n, float(epsilon),
                                          fcs.data_ptr() if (fcs is not None and nf) else 0, nf, cols,
                                          bool(fcs is not None and fcs.dtype == torch.int64), out_p.data_ptr(), svi.data_ptr(),
                                          svj.data_ptr(), out_f.data_ptr() if (out_f is not None and nf) else 0, counts.data_ptr(),
                                          dev, stream)
        u, kept_f, bad = (int(v) for v in counts.tolist())
        if bad:
            raise ValueError("%d faces refer to vertices outside [0, %d)" % (bad, n))
        return (out_p[:u], svi[:u], svj) if fcs is None else (out_p[:u], out_f[:kept_f], svi[:u], svj)

    out = _run(form, arrays, device, body)
    return (out[0], None) + out[1:] if faces is None else out


def deduplicate_point_cloud(points, epsilon, return_index=True, *, device=None):
    """
    Removes duplicated points from a point cloud where two points are considered the same if their distance is below
    some threshold

    Args:
        x : #x by 3 Matrix of 3D positions
        epsilon: threshold below which two points are considered equal
        return_index: If true, return indices to map between input and output

    Returns:
        x_new : #x_new x 3 Point cloud with duplicates removed
        if return indices is set, this function also returns:
            svi : #x_new x 1 indices so that x_new = x[svi]
            svj : #x x 1 indices so that x = x_new[svj]

    Mirrors /root/reference/src/remove_duplicates.cpp:85-126 (libigl round + unique_rows): with epsilon > 0 two points
    are merged when round(p / epsilon) agrees on every axis, otherwise when they are equal; unique rows come in ascending
    lexicographic order.  svi names the FIRST input row of each cluster (libigl's choice among equal rows is unspecified).
    `device` (keyword only): see `k_nearest_neighbors`.
    """
    x_new, _, svi, svj = _dedup(points, None, epsilon, device, "points")
    if return_index:
        return x_new, svi, svj
    return x_new


def deduplicate_mesh_vertices(v, f, epsilon, return_index=True, *, device=None):
    """
    Removes duplicated vertices from a triangle mesh two vertices are considered the same if their distance is below
    some threshold

    Args:
        v : #v by 3 Matrix of mesh vertex 3D positions
        f : #f by 3 Matrix of face (triangle) indices
        epsilon: threshold below which two points are considered equal
        return_index: If true, return indices to map between input and output

    Returns:
        v_out : #v x 3 array of mesh vertices with duplicates removed
        f_out : #f x 3 array of mesh faces corresponding to the deduplicated mesh
        svi : #v_out x 1 indices so that v_out = v[svi] (only returned if return_index is True)
        svj : #v x 1 indices so that v = v_out[svj] (only returned if return_index is True)

    Mirrors /root/reference/src/remove_duplicates.cpp:129-176 and :36-77: faces are re-indexed through svj; a face two of
    whose corners end up on the same vertex is dropped; the others keep their order.
    """
    if f is None:
        raise ValueError("f must be an (m, 3) array of face indices")
    v_out, f_out, svi, svj = _dedup(v, f, epsilon, device, "v")
    if return_index:
        return v_out, f_out, svi, svj
    return v_out, f_out
