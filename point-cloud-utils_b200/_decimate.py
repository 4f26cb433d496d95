"""decimate_triangle_mesh -- the reference's name, arguments and outputs (src/mesh_decimate.cpp), computed by
csrc/decimate.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
from . import _pcu_internal
from ._call import _INDEX_KINDS, _dtype_name, _form, _run, _torch, _validate_mesh


def decimate_triangle_mesh(v, f, max_faces, decimation_heuristic="shortest_edge", *, device=None):
    """
    Decimate a (manifold) triangle mesh by collapsing edges

    Args:
        v : (#v, 3)-shaped array of mesh vertex positions
        f : (#f, 3)-shaped array of triangle face indices
        max_faces : The maximum number of faces in the decimated output mesh (must be between 0 and #f)
        decimation_heuristic : Which decimation heuristic to use. Currently only supports "shortest_edge".
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v_out : (#v_out, 3)-shaped array of vertex positions for the decimated mesh
        f_out : (#f_out, 3)-shaped array of triangle face indices for the decimated mesh
        v_correspondences : (#v_out,)-shaped array where v_correspondences[i] is the index of the vertex in v which generated v_out[i]
        f_correspondences : (#f_out,)-shaped array where f_correspondences[i] is the index of the face in f which generated f_out[i]

    Dtypes: v float32 / float64 (widened exactly to fp64; v_out has v's dtype), f int32 / int64 / uint32 / uint64 (f_out
    and both correspondences have f's dtype).  The reference's libigl is not available, so the result is defined in
    DESIGN.md §3 and computed deterministically in fp64.  In short: rounds of edge collapses.  Each round ranks the
    edges that pass the link condition (on the mesh with its boundary joined to a virtual vertex) by squared length,
    ties by vertex ids; takes those ranked below #alive - max_faces whose neighbourhoods meet no lower-ranked one's;
    applies them in rank order while the faces they remove stay below #alive - max_faces; and merges the higher id into
    the lower at the edge's midpoint.  Rounds repeat until at most max_faces faces remain or no edge passes.
    f_out keeps the surviving faces in input order (f_correspondences), v_out the vertices they use in ascending id
    (v_correspondences).  The result has max_faces or max_faces - 1 faces, unless a component cannot shrink further
    (a lone tetrahedron, say): then it has more than max_faces faces and is returned as it is.
    A mesh with a repeated corner in a face, an edge in three or more faces, or a vertex with other than zero or two
    boundary edges raises the reference's "produced an empty mesh" ValueError.
    Divergences: a non-finite vertex or a face corner outside [0, #v) raise ValueError.
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    max_faces = int(max_faces)
    nf = int(f.shape[0])
    if max_faces <= 0:
        raise ValueError("max_faces must be greater than 0, got %d." % max_faces)
    if max_faces > nf:
        raise ValueError("max_faces must be less than or equal to the number of input faces (%d), got %d." % (nf, max_faces))
    if decimation_heuristic != "shortest_edge":
        raise ValueError("Invalid decimation heuristic, must be 'shortest_edge'. Others will be implemented"
                         " in future versions of Point Cloud Utils.")
    torch = _torch()

    def body(vt, ft, dev, stream):
        handle, nv_out, nf_out, _ = _pcu_internal._decimate_triangle_mesh_prepare_device(
            vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(), nf, _INDEX_KINDS[_dtype_name(f)],
            max_faces, dev, stream)
        try:
            v_out = torch.empty((nv_out, 3), dtype=vt.dtype, device=vt.device)
            f_out = torch.empty((nf_out, 3), dtype=ft.dtype, device=vt.device)
            v_corr = torch.empty((nv_out,), dtype=ft.dtype, device=vt.device)
            f_corr = torch.empty((nf_out,), dtype=ft.dtype, device=vt.device)
            _pcu_internal._decimate_triangle_mesh_emit_device(handle, v_out.data_ptr(), f_out.data_ptr(), v_corr.data_ptr(),
                                                              f_corr.data_ptr(), dev, stream)
        finally:
            _pcu_internal._decimate_triangle_mesh_destroy(handle)
        return v_out, f_out, v_corr, f_corr

    return _run(form, [v, f], device, body, index=(f, [1, 2, 3]))
