"""connected_components, remove_mesh_vertices, remove_unreferenced_mesh_vertices, orient_mesh_faces and adjacency_list
-- the reference's names, arguments and outputs (the reference's src/connected_components.cpp,
src/remove_mesh_vertices.cpp, src/remove_unreferenced_mesh_vertices.cpp, src/orient_mesh_faces.cpp and
src/adjacency_list.cpp), computed by csrc/mesh_topology.cuh, csrc/orient.cuh and csrc/laplacian.cuh.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages and in its order, before any
device call.  Shapes are the reference's through npe::move, which squeezes them as numpy does: an (m, 1) result is
(m,), a single entry is a 0-d array and a single (1, 3) row is (3,)."""
from . import _pcu_internal
from ._call import (_INDEX_KINDS, _check_float, _check_index, _dtype_name, _form, _matrix_shape, _run, _torch, _validate_mesh,
                    _validate_mesh_faces)

_MAX_ROWS = 2 ** 31 - 1


def connected_components(v, f, *, device=None):
    """
    Determine the connected components of a mesh

    Args:
      v : (#v, 3)-shaped array of mesh vertex positions (one vertex position per row)
      f : (#f, 3)-shaped array of mesh face indexes into v (a row (fi, fj, fk) indicate the 3 vertices of a face)
      device: see `k_nearest_neighbors` (keyword only).

    Returns:
      cv : a (#vertices,)-shaped array of integer indexes (starting from 0) indicating which component each vertex belongs to. i.e. cv[i] is the component of the vertex v[i].
      nv : the number of vertices in each connected component. i.e. nv[j] is the number of vertices in component j
      cf : a (#faces,)-shaped array of integer indexes (starting from 0) indicating which component each face belongs to. i.e. cf[i] is the component of the face f[i].
      nf : the number of faces in each connected component. i.e. nf[j] is the number of faces in component j

    Dtypes: v float32 / float64 (checked, never read: the result depends on f alone), f int32 / int64 / uint32 / uint64
    of shape (m, c), m, c >= 1 (a 1-D f is one column); all four outputs have f's dtype.  Defined in DESIGN.md §3 as
    the reference computes it: the graph's vertices are [0, n) with n = max(f) + 1 (libigl's adjacency_matrix sizes it
    so), not #v, so cv is shorter than #v when the last vertices are unreferenced and longer when f refers past #v;
    the corners of a row are joined to each other (so edge lists and tets work), and every index no face names is a
    component of one vertex.  Component j is the j-th in ascending order of its smallest vertex, the order in which the
    reference starts its BFS runs; cf[i] = cv[f[i, 0]].  Shapes squeezed as npe::move squeezes them: one face gives a
    0-d cf, one component 0-d nv and nf.
    Divergences, where the reference is undefined: an f with zero rows or zero columns, a negative index or an index
    above 2^31 - 2 raise ValueError.
    """
    form = _form([v, f], ["v", "f"])
    _check_float(v, "v")
    _check_index(f, "f", _INDEX_KINDS)
    if len(f.shape) not in (1, 2):
        raise ValueError("connected_components: f must be a 1-D or 2-D array, got shape %s" % (tuple(f.shape),))
    rows, cols = _matrix_shape(f)
    if rows == 0 or cols == 0:
        raise ValueError("connected_components: f must have at least one row and one column, got shape %s" % (tuple(f.shape),))
    if rows >= _MAX_ROWS:
        raise ValueError("connected_components: at most 2^31 - 2 faces are supported, got %d" % rows)
    torch = _torch()

    def body(ft, dev, stream):
        handle, n, k = _pcu_internal._connected_components_prepare_device(ft.data_ptr(), rows, cols, _INDEX_KINDS[_dtype_name(f)], dev,
                                                                           stream)
        try:
            cv = torch.empty(n, dtype=ft.dtype, device=ft.device)
            nv = torch.empty(k, dtype=ft.dtype, device=ft.device)
            cf = torch.empty(rows, dtype=ft.dtype, device=ft.device)
            nf = torch.empty(k, dtype=ft.dtype, device=ft.device)
            _pcu_internal._connected_components_emit_device(handle, cv.data_ptr(), nv.data_ptr(), cf.data_ptr(), nf.data_ptr(), dev, stream)
        finally:
            _pcu_internal._connected_components_destroy(handle)
        return cv, nv, cf, nf

    return _run(form, [f], device, body, index=(f, [0, 1, 2, 3]), squeeze=True)


def remove_mesh_vertices(v, f, mask, *, device=None):
    """
    Removes vertices specified by a mask from a triangle mesh and updates the face indices accordingly.

    Args:
        v : #v by 3 Matrix of mesh vertex 3D positions
        f : #f by 3 Matrix of face (triangle) indices
        mask: A boolean mask of shape (#v,) indicating which vertices to keep (True) or remove (False)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v_out : (#v, 3)-shaped array of mesh vertices with the mask applied
        f_out : (#f, 3)-shaped array of mesh faces corresponding to mesh with removed vertices

    Dtypes: v float32 / float64, f int32 / int64, mask bool of shape (#v,) or (#v, 1); v_out has v's dtype, f_out f's.
    As the reference computes it (src/remove_mesh_vertices.cpp): v_out holds the kept vertices in input order, f_out
    the faces whose three corners are all kept, in input order, re-indexed to the new numbering.  Shapes squeezed as
    npe::move squeezes them: one kept vertex gives v_out of shape (3,), one kept face f_out of shape (3,).
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    form = _form([v, f, mask], ["v", "f", "mask"])
    _check_float(v, "v")
    _check_index(f, "f", {"int32": 0, "int64": 1})
    _check_index(mask, "mask", {"bool": 0})
    _validate_mesh(v, f, _INDEX_KINDS)
    mrows, mcols = _matrix_shape(mask)
    if mrows != v.shape[0]:
        raise ValueError("mask should have the same number of rows as v")
    if mcols != 1:
        raise ValueError("mask should have only one column")
    nvert, nface = int(v.shape[0]), int(f.shape[0])
    if nvert >= _MAX_ROWS or nface >= _MAX_ROWS:
        raise ValueError("remove_mesh_vertices: at most 2^31 - 2 vertices and faces are supported, got %d and %d" % (nvert, nface))
    torch = _torch()

    def body(vt, ft, mt, dev, stream):
        v_out = torch.empty((nvert, 3), dtype=vt.dtype, device=vt.device)
        f_out = torch.empty((nface, 3), dtype=ft.dtype, device=vt.device)
        kv, kf = _pcu_internal._remove_mesh_vertices_device(vt.dtype == torch.float64, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                                            _INDEX_KINDS[_dtype_name(f)], mt.data_ptr(), v_out.data_ptr(), f_out.data_ptr(),
                                                            dev, stream)
        return v_out[:kv], f_out[:kf]

    return _run(form, [v, f, mask.reshape(-1)], device, body, index=(f, [1]), squeeze=True)


def remove_unreferenced_mesh_vertices(v, f, *, device=None):
    """
    Removes the vertices of a triangle mesh that no face references.

    Args:
        v : (#v, 3)-shaped array of mesh vertex 3D positions
        f : (#f, 3)-shaped array of face (triangle) indices
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        v_new : (#v_new, 3)-shaped array of mesh vertex positions without unreferenced vertices
        f_new : (#f, 3)-shaped array of mesh faces indexing into v_new
        correspondences_v : (#v_new,)-shaped array J of old vertex indices, so that v_new = v[J]
        correspondences_f : (#v,)-shaped array I of new vertex indices, so that f_new = I[f]; -1 (converted to f's
                            dtype, so all ones for uint32 / uint64) for the unreferenced vertices

    Dtypes: v float32 / float64, f int32 / int64 / uint32 / uint64; the index outputs have f's dtype.  As the reference
    computes it (igl::remove_unreferenced(V, F, NV, NF, I, J), returned as (NV, NF, J, I)): a vertex is referenced
    when some face corner names it; J lists the referenced vertices in ascending order, and every face is kept.  The
    reference's own docstring describes the two correspondence arrays otherwise ("(#v, 1)-shaped ... v_new =
    correspondences_v[svi]", "(#f, 1)-shaped ... f_new = correspondences_f[svj]"); the shapes and meanings above are what
    it returns.  Shapes squeezed as npe::move squeezes them: one referenced vertex gives v_new of shape (3,) and a 0-d
    correspondences_v, one face f_new of shape (3,), one vertex a 0-d correspondences_f.
    Divergence: a face corner outside [0, #v) raises ValueError, -1 included (libigl's handling of it depends on its
    version).
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, _INDEX_KINDS)
    nvert, nface = int(v.shape[0]), int(f.shape[0])
    if nvert >= _MAX_ROWS or nface >= _MAX_ROWS:
        raise ValueError("remove_unreferenced_mesh_vertices: at most 2^31 - 2 vertices and faces are supported, got %d and %d"
                         % (nvert, nface))
    torch = _torch()

    def body(vt, ft, dev, stream):
        v_out = torch.empty((nvert, 3), dtype=vt.dtype, device=vt.device)
        f_out = torch.empty((nface, 3), dtype=ft.dtype, device=vt.device)
        corr_v = torch.empty(nvert, dtype=ft.dtype, device=vt.device)
        corr_f = torch.empty(nvert, dtype=ft.dtype, device=vt.device)
        kept = _pcu_internal._remove_unreferenced_device(vt.dtype == torch.float64, vt.data_ptr(), nvert, ft.data_ptr(), nface,
                                                         _INDEX_KINDS[_dtype_name(f)], v_out.data_ptr(), f_out.data_ptr(), corr_v.data_ptr(),
                                                         corr_f.data_ptr(), dev, stream)
        return v_out[:kept], f_out, corr_v[:kept], corr_f

    return _run(form, [v, f], device, body, index=(f, [1, 2, 3]), squeeze=True)


_MAX_ORIENT_FACES = 2 ** 30 - 1


def orient_mesh_faces(f, weighting_type="uniform", *, device=None):
    """
    Consistently orient faces of a mesh within each connected component

    Args:
        f : (#f, 3)-shaped NumPy array of face (triangle) indices
        weighting_type : accepted for the reference's signature and ignored (the reference never reads it)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        oriented_faces  : (#f, 3)-shaped NumPy array of faces which are consistently oriented
        face_components : (#f,)-shaped NumPy array of connected component ids (i.e. face_components[i] is the component id of facef[i])

    Dtypes: f int32 / int64 / uint32 / uint64; both outputs have f's dtype.  Defined in DESIGN.md §3 as libigl's
    bfs_orient computes it: two faces are adjacent when they share an undirected edge that no third face has, and the
    components are the patches this adjacency connects, numbered in ascending order of their smallest face.  Each patch
    is walked breadth-first from its smallest face, which is never flipped; a neighbour is reversed ((a, b, c) becomes
    (c, b, a)) whenever one of its directed edges equals one of the current face's.  Ids are only compared for
    equality, never used as indices, so any value (negative ones included) is legal and no vertex array is needed.
    Shapes squeezed as npe::move squeezes them: one face gives oriented_faces of shape (3,) and a 0-d face_components.
    A CUDA-tensor call never synchronises the host.
    Divergence: more than 2^30 - 1 faces raise ValueError.
    """
    form = _form([f], ["f"])
    _check_index(f, "f", _INDEX_KINDS)
    if len(f.shape) not in (1, 2):
        raise ValueError("orient_mesh_faces: f must be a 1-D or 2-D array, got shape %s" % (tuple(f.shape),))
    rows = _validate_mesh_faces(f)
    if rows > _MAX_ORIENT_FACES:
        raise ValueError("orient_mesh_faces: at most 2^30 - 1 faces are supported, got %d" % rows)
    torch = _torch()

    def body(ft, dev, stream):
        out_f = torch.empty((rows, 3), dtype=ft.dtype, device=ft.device)
        out_c = torch.empty(rows, dtype=ft.dtype, device=ft.device)
        _pcu_internal._orient_mesh_faces_device(ft.data_ptr(), rows, _INDEX_KINDS[_dtype_name(f)], out_f.data_ptr(), out_c.data_ptr(),
                                                dev, stream)
        return out_f, out_c

    return _run(form, [f], device, body, index=(f, [0, 1]), squeeze=True)


_MAX_ADJACENCY_FACES = (2 ** 31 - 1) // 6


def adjacency_list(f, *, return_csr=False, device=None):
    """
    Compute the adjacency list given a set of mesh faces.

    Args:
        f : \\#f by 3 Matrix of face (triangle) indices
        return_csr : (keyword only, not in the reference) return the lists as two flat arrays instead of Python lists
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        adj_list : a list of lists such that adj_list[i] contains the indexes of vertices adjacent to vertex i
        or, with return_csr=True, (offsets, neighbors): arrays in f's dtype and form of shape (n + 1,) and
            (offsets[-1],), list i being neighbors[offsets[i]:offsets[i + 1]]; a CUDA input gives CUDA tensors on its
            device, ready for torch's or scipy's sparse constructors

    Dtypes: f int32 / int64.  Defined in DESIGN.md §3 as libigl's adjacency_list(F, A, sorted=false) computes it: there
    are n = max(f) + 1 lists (not #v: there is no v); every face (a, b, c) adds a<->b, b<->c and c<->a in both
    directions, and each list is then sorted ascending without duplicates.  So list i holds every vertex that shares a
    face with i, i itself when some face names i at two or more corners, and an index no face names gets an empty
    list.  The default result holds Python ints whatever f's form; both results come from one device computation.
    Divergences: a negative index or an index above 2^31 - 2 raises ValueError (in the reference the outcome depends on
    the other indices), and so do more than 357913941 faces.
    """
    form = _form([f], ["f"])
    _check_index(f, "f", {"int32": 0, "int64": 1})
    if len(f.shape) not in (1, 2):
        raise ValueError("adjacency_list: f must be a 1-D or 2-D array, got shape %s" % (tuple(f.shape),))
    rows = _validate_mesh_faces(f)
    if rows > _MAX_ADJACENCY_FACES:
        raise ValueError("adjacency_list: at most %d faces are supported, got %d" % (_MAX_ADJACENCY_FACES, rows))
    torch = _torch()

    def body(ft, dev, stream):
        handle, n, nnz = _pcu_internal._adjacency_list_prepare_device(ft.data_ptr(), rows, _INDEX_KINDS[_dtype_name(f)], dev, stream)
        try:
            offsets = torch.empty(n + 1, dtype=ft.dtype, device=ft.device)
            neighbors = torch.empty(nnz, dtype=ft.dtype, device=ft.device)
            _pcu_internal._adjacency_list_emit_device(handle, offsets.data_ptr(), neighbors.data_ptr(), dev, stream)
        finally:
            _pcu_internal._adjacency_list_destroy(handle)
        return offsets, neighbors

    offsets, neighbors = _run(form, [f], device, body, index=(f, [0, 1]))
    if return_csr:
        return offsets, neighbors
    o, nb = offsets.tolist(), neighbors.tolist()
    return [nb[o[i]:o[i + 1]] for i in range(len(o) - 1)]
