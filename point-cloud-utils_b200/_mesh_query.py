"""closest_points_on_mesh -- the reference's name, arguments and outputs (the reference's src/closest_point_on_mesh.cpp),
computed by csrc/meshquery.cuh.

Input forms and validation follow _mesh_sampling.py: numpy arrays in -> numpy out; CUDA torch tensors in -> CUDA tensors
out; CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
from . import _pcu_internal
from ._mesh_sampling import _INDEX_KINDS, _back, _call_args, _dtype_name, _form, _to_device, _torch, _validate_mesh


def _validate_points(p, v, f):
    """The binding's dtype checks (npe_arg(v, npe_matches(p)) among them), then validate_point_cloud(p), which allows
    zero rows (src/common/common.h).  validate_mesh follows."""
    if _dtype_name(p) not in ("float32", "float64"):
        raise ValueError("Invalid scalar type (%s) for argument 'p'. Expected one of ['float32', 'float64']." % _dtype_name(p))
    if _dtype_name(v) != _dtype_name(p):
        raise ValueError("Invalid scalar type (%s) for argument 'v'. Expected it to match argument 'p' which is of type %s."
                         % (_dtype_name(v), _dtype_name(p)))
    if _dtype_name(f) not in _INDEX_KINDS:
        raise ValueError("Invalid scalar type (%s) for argument 'f'. Expected one of %s." % (_dtype_name(f), list(_INDEX_KINDS)))
    if len(p.shape) != 2 or p.shape[1] != 3:
        raise ValueError("Only 3D inputs are supported: v must have shape (n, 3) (n > 0). Got points.shape =%s."
                         % (tuple(p.shape),))


def closest_points_on_mesh(p, v, f, *, device=None):
    """
    Compute distances from a set of points p to a triangle mesh (v, f)

    Args:
        p : (#p, 3)-shaped array of query point positions (float32 / float64)
        v : (#v, 3)-shaped array of mesh vertex positions (p's dtype)
        f : (#f, 3)-shaped array of triangle face indices (int32 / int64 / uint32 / uint64)
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        d : a (#p,)-shaped array of shortest distances for each query point p (p's dtype)
        f_idx : a (#p,)-shaped array of indices into f of the face containing the closest point to each query point
                (f's dtype)
        bc : a (#p, 3)-shaped array of barycentric coordinates for each query point (p's dtype)

    Mirrors the reference's src/closest_point_on_mesh.cpp (igl::point_mesh_squared_distance).  The result is a pure
    function of (p, v, f), defined in DESIGN.md §3: for every face, Ericson's Voronoi-region closest point in p's
    precision with every operation rounded on its own (a face whose corners are collinear or coincident is the union of
    its edges, as in libigl); the chosen face is the lexicographic minimum of (squared distance, face index), so among
    faces at exactly the same distance the lowest index wins.  d = sqrt(d^2), and bc are the chosen face's coordinates
    of the closest point.
    Divergences: libigl's choice among tied faces depends on its tree and is not reproduced; a face corner outside
    [0, #v) raises ValueError (the reference reads out of bounds).
    """
    from . import _same_device
    form = _form([p, v, f], ["p", "v", "f"])
    _validate_points(p, v, f)
    _validate_mesh(v, f, ("int32", "int64", "uint32", "uint64"))
    torch = _torch()
    if form == "cpu":
        out = closest_points_on_mesh(p.detach().numpy(), v.detach().numpy(), f.detach().numpy(), device=device)
        return tuple(torch.from_numpy(o) for o in out)
    n = int(p.shape[0])
    if n == 0:
        if form == "numpy":
            import numpy as np
            return np.zeros(0, dtype=p.dtype), np.zeros(0, dtype=f.dtype), np.zeros((0, 3), dtype=p.dtype)
        _same_device(p, device)
        return (torch.zeros(0, dtype=p.dtype, device=p.device), torch.zeros(0, dtype=f.dtype, device=p.device),
                torch.zeros((0, 3), dtype=p.dtype, device=p.device))
    if form == "cuda":
        _same_device(p, device)
        pt, vt, ft = p.detach().contiguous(), v.detach().contiguous(), f.detach().contiguous()
    else:
        pt, vt, ft = _to_device([p, v, f], device)
    dev, stream = _call_args(pt)
    d = torch.empty(n, dtype=pt.dtype, device=pt.device)
    fidx = torch.empty(n, dtype=ft.dtype, device=pt.device)
    bc = torch.empty((n, 3), dtype=pt.dtype, device=pt.device)
    bad = torch.empty(1, dtype=torch.int64, device=pt.device)
    _pcu_internal._closest_points_on_mesh_device(pt.dtype == torch.float64, pt.data_ptr(), n, vt.data_ptr(), int(vt.shape[0]),
                                                 ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)], d.data_ptr(),
                                                 fidx.data_ptr(), bc.data_ptr(), bad.data_ptr(), dev, stream)
    nbad = int(bad.item())
    if nbad:
        raise ValueError("Invalid face indices: %d faces have a corner outside [0, #v)" % nbad)
    if form == "numpy":
        return (d.cpu().numpy(),) + _back(fidx, bc, f, form)
    return d, fidx, bc
