"""sample_mesh_random, sample_mesh_poisson_disk and interpolate_barycentric_coords -- the reference's names, arguments
and defaults (the reference's src/sample_mesh.cpp and point_cloud_utils/__init__.py:203-217), computed by
csrc/meshsample.cuh (and, for the Poisson-disk selection, csrc/poisson.cuh).

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors.  Arguments are validated, with the reference's messages, before any device call."""
import math

import numpy as _np

from . import _pcu_internal
from ._call import _INDEX_KINDS, _check_float, _check_index, _dtype_name, _form, _raise_bad, _run, _same_device, _torch, _validate_mesh


def _seed(random_seed):
    """A 32-bit seed; 0 draws one from NumPy's global random state (the reference uses the time)."""
    seed = int(random_seed) & 0xFFFFFFFF
    return int(_np.random.randint(2 ** 31 - 1)) if seed == 0 else seed


def _read_area(area):
    """{W, S, bad faces} from the 24-byte device record (synchronises), with the errors they imply."""
    host = area.cpu().numpy()
    W = int(host[:1].view(_np.uint64)[0])
    S = float(host[1:2].view(_np.float64)[0])
    _raise_bad(host[2])
    if W == 0:
        raise ValueError("Mesh has zero area")
    return W, S


def sample_mesh_random(v, f, num_samples, random_seed=0, *, device=None):
    """
    Generate uniformly distributed random point samples on a mesh

    Args:
        v : (#v, 3)-shaped array of mesh vertex positions (float32 / float64)
        f : (#f, 3)-shaped array of mesh face indices (int32 / int64 / uint32 / uint64)
        num_samples : The number of samples to generate
        random_seed : A random seed used to generate the samples (a 32-bit integer).  Passing in 0 draws the seed from
                      NumPy's global random state (the reference uses the current time): seed NumPy for reproducible
                      results.
        device: see `k_nearest_neighbors` (keyword only).
    Returns:
        f_idx : (num_samples,) shaped array of face indices into f, of f's dtype
        bc : (num_samples, 3) shaped array of barycentric coordinates, of v's dtype

    Mirrors the reference's src/sample_mesh.cpp (igl::random_points_on_mesh).  The reference draws with std::rand; here
    sample s is a pure function of (v, f, seed), defined in DESIGN.md §3: faces are drawn in proportion to an exact
    fixed-point cumulative area, s's face is the first whose cumulative weight exceeds mulhi64(h(0), W), and its
    coordinates are (1 - sqrt(u1), sqrt(u1) (1 - u2), sqrt(u1) u2) with u1, u2 from h(1), h(2), h(j) = mix64(mix64(3 s +
    j) ^ seed).  Faces of zero area are never drawn.
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, ("int32", "int64", "uint32", "uint64"))
    if int(num_samples) <= 0:
        raise ValueError("num_samples must be positive")
    n = int(num_samples)
    seed = _seed(random_seed)
    torch = _torch()

    def body(vt, ft, dev, stream):
        kind = _INDEX_KINDS[_dtype_name(f)]
        fidx = torch.empty(n, dtype=ft.dtype, device=vt.device)
        bc = torch.empty((n, 3), dtype=vt.dtype, device=vt.device)
        area = torch.empty(3, dtype=torch.int64, device=vt.device)
        _pcu_internal._sample_mesh_random_device(vt.dtype == torch.float64, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(),
                                                 int(ft.shape[0]), kind, n, seed, fidx.data_ptr(),
                                                 bc.data_ptr(), area.data_ptr(), dev, stream)
        _read_area(area)
        return fidx, bc

    return _run(form, [v, f], device, body, index=(f, [0]))


def dense_plan(W, S, num_samples, radius, oversampling_factor):
    """(radius, number of dense samples) of sample_mesh_poisson_disk from the mesh's {W, S} (DESIGN.md §3)."""
    total_area = float(W) / S / 2.0
    if radius <= 0.0 and num_samples > 0:                                    # src/sample_mesh.cpp:57-63
        radius = math.sqrt(total_area / (0.7 * math.pi * num_samples))
    n_est = float(num_samples) if num_samples > 0 else total_area / (0.7 * math.pi * (radius * radius))
    dense = oversampling_factor * n_est
    if not dense < 2 ** 31:
        raise ValueError("oversampling_factor * num_samples = %g dense samples: at most 2^31 - 1 are supported" % dense)
    return float(radius), max(1, int(math.ceil(dense)))


def sample_mesh_poisson_disk(v, f, num_samples, radius=0.0, use_geodesic_distance=True, best_choice_sampling=True,
                             random_seed=0, sample_num_tolerance=0.04, oversampling_factor=40.0, *, device=None):
    """
    Downsample a mesh's surface so that samples are approximately evenly spaced.

    Args:
        v : #v by 3 array of mesh vertex positions (float32 / float64)
        f : #f by 3 array of mesh face indices (int32 / int64)
        num_samples: desired number of Poisson Disk samples.  If this value <= 0, then the parameter radius is used to
                     decide the number of samples.
        radius : desired separation between points; when positive it is used even if num_samples > 0.  Otherwise it is
                 sqrt(total_area / (0.7 pi num_samples)), as in the reference.
        use_geodesic_distance : accepted and ignored, as in the reference (which does not pass it on).
        best_choice_sampling : accepted and ignored, as in the reference.
        random_seed : a 32-bit seed; 0 draws one from NumPy's global random state (the reference uses the time).
        sample_num_tolerance: accepted and ignored as in the reference, but validated like it: must be in (0, 1].
        oversampling_factor: the dense uniform sample has ceil(oversampling_factor * num_samples) rows (num_samples is
                             estimated from the area and the radius when not given).  Must be >= 1.
        device: see `k_nearest_neighbors` (keyword only).
    Returns:
        f_idx : a (m,)-shaped array of face indices into f (f's dtype), m the number of Poisson-disk samples
        bc : a (m, 3)-shaped array of barycentric coordinates (v's dtype)

    Mirrors the reference's src/sample_mesh.cpp (igl::blue_noise).  The reference's subset cannot be reproduced; here
    it is defined exactly (DESIGN.md §3): n_dense samples of sample_mesh_random with the same seed, their positions
    p_s = fl((bc0 a + bc1 b) + bc2 c) (fp64 from the unrounded coordinates), and downsample_point_cloud_poisson_disk(p,
    radius, random_seed=seed) on those: the kept samples in ascending dense order.  No two kept dense positions are
    closer than the radius; positions a caller re-interpolates in v's dtype can differ from them in the last bit.
    The total area is W / S / 2 from the fixed-point face weights: it differs from a floating-point sum of the areas by
    at most a few ulps plus m * 2^-(62 - ceil(log2 m)) of the largest face's area.
    Divergences: distances are Euclidean between dense positions (the reference's are too: it does not use geodesics);
    a face corner outside [0, #v) raises ValueError.
    """
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, ("int32", "int64"))
    num_samples, radius = int(num_samples), float(radius)
    if num_samples <= 0 and radius <= 0.0:                                   # src/sample_mesh.cpp:49-51
        raise ValueError("Cannot have both num_samples <= 0 and radius <= 0")
    tol = float(_np.float32(sample_num_tolerance))                           # the binding takes a float
    if tol > 1.0 or tol <= 0.0:                                              # :52-54
        raise ValueError("sample_num_tolerance must be in (0, 1]")
    osf = float(_np.float32(oversampling_factor))
    if not osf >= 1.0:
        raise ValueError("oversampling_factor must be >= 1.0 (got %r)" % (oversampling_factor,))
    seed = _seed(random_seed)
    torch = _torch()

    def body(vt, ft, dev, stream):
        is_f64, nv, nf, kind = vt.dtype == torch.float64, int(vt.shape[0]), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)]
        area = torch.empty(3, dtype=torch.int64, device=vt.device)
        _pcu_internal._mesh_area_device(is_f64, vt.data_ptr(), nv, ft.data_ptr(), nf, kind, area.data_ptr(), dev, stream)
        W, S = _read_area(area)
        r, n_dense = dense_plan(W, S, num_samples, radius, osf)
        fidx = torch.empty(n_dense, dtype=ft.dtype, device=vt.device)
        bc = torch.empty((n_dense, 3), dtype=vt.dtype, device=vt.device)
        count = torch.empty(1, dtype=torch.int64, device=vt.device)
        _pcu_internal._sample_mesh_poisson_disk_device(is_f64, vt.data_ptr(), nv, ft.data_ptr(), nf, kind, r, n_dense, seed,
                                                       fidx.data_ptr(), bc.data_ptr(), count.data_ptr(), dev, stream)
        m = int(count.item())
        return fidx[:m], bc[:m]

    return _run(form, [v, f], device, body, index=(f, [0]))


def interpolate_barycentric_coords(f, fi, bc, attribute, *, device=None):
    """
    Interpolate an attribute stored at each vertex of a mesh across the faces of a triangle mesh using
    barycentric coordinates

    Args:
        f : a (#faces, 3)-shaped array of mesh faces (int32 / int64 / uint32 / uint64, indexing into some vertex array).
        fi: a (#attribs,)-shaped integer array of indexes into f indicating which face each attribute lies within.
        bc: a (#attribs, 3)-shaped float32 / float64 array of barycentric coordinates for each attribute
        attribute: a (#vertices, dim)-shaped float32 / float64 array of attributes at each of the mesh vertices
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        A (#attribs, dim)-shaped array of interpolated attributes, float64 if bc or attribute is, else float32.

    Bit for bit the reference's (attribute[f[fi]] * bc[:, :, np.newaxis]).sum(1) (point_cloud_utils/__init__.py:217):
    ((x0 b0 + x1 b1) + x2 b2) with every product and sum rounded in the promoted dtype.  Negative indices wrap as in
    numpy; an index out of range raises IndexError (for numpy inputs before any device call).
    Divergence: attribute must be 2-D; a 1-D attribute raises ValueError (numpy's broadcasting makes the reference's
    result an unrelated (#attribs, 3) array).
    """
    form = _form([f, fi, bc, attribute], ["f", "fi", "bc", "attribute"])
    _check_index(f, "f", _INDEX_KINDS)
    _check_index(fi, "fi", _INDEX_KINDS)
    _check_float(bc, "bc")
    _check_float(attribute, "attribute")
    if attribute.ndim != 2:
        raise ValueError("attribute must have shape (#vertices, dim), got %s" % (tuple(attribute.shape),))
    if f.ndim != 2 or f.shape[1] != 3:
        raise ValueError("f must have shape (#faces, 3), got %s" % (tuple(f.shape),))
    if fi.ndim != 1 or bc.ndim != 2 or bc.shape[1] != 3 or bc.shape[0] != fi.shape[0]:
        raise ValueError("fi and bc must have shapes (n,) and (n, 3), got %s and %s" % (tuple(fi.shape), tuple(bc.shape)))
    torch = _torch()
    out_f64 = "float64" in (_dtype_name(bc), _dtype_name(attribute))
    n, dim, nv, nf = int(fi.shape[0]), int(attribute.shape[1]), int(attribute.shape[0]), int(f.shape[0])
    if form != "cuda":
        hf, hfi = (f, fi) if form == "numpy" else (f.detach().numpy(), fi.detach().numpy())
        corners = hf[hfi]                                 # numpy's own IndexError for fi out of range
        if corners.size and (int(corners.max()) >= nv or (corners.dtype.kind == "i" and int(corners.min()) < -nv)):
            raise IndexError("index out of bounds for attribute with %d rows" % nv)
    if n == 0 or dim == 0:
        if form == "numpy":
            return _np.zeros((n, dim), dtype=_np.float64 if out_f64 else _np.float32)
        if form == "cuda":
            _same_device(f, device)
        return torch.zeros((n, dim), dtype=torch.float64 if out_f64 else torch.float32, device=f.device)

    def body(ft, fit, bct, at, dev, stream):
        if nf == 0 or nv == 0:
            raise IndexError("index out of bounds: f has %d rows and attribute %d" % (nf, nv))
        out = torch.empty((n, dim), dtype=torch.float64 if out_f64 else torch.float32, device=ft.device)
        bad = torch.empty(1, dtype=torch.int64, device=ft.device)
        _pcu_internal._interpolate_barycentric_device(ft.data_ptr(), nf, _INDEX_KINDS[_dtype_name(f)], fit.data_ptr(), n,
                                                      _INDEX_KINDS[_dtype_name(fi)], bct.data_ptr(), bct.dtype == torch.float64,
                                                      at.data_ptr(), at.dtype == torch.float64, nv, dim, out.data_ptr(),
                                                      bad.data_ptr(), dev, stream)
        if int(bad.item()):
            raise IndexError("index out of bounds: %d rows of fi name a face or a vertex out of range" % int(bad.item()))
        return out

    return _run(form, [f, fi, bc, attribute], device, body)
