"""voronoi_centroids_unit_cube, lloyd_3d, lloyd_2d and sample_mesh_lloyd -- the reference's names, arguments, defaults
and messages (the reference's src/lloyd.cpp:166-401), computed by csrc/voronoi.cuh and csrc/rvd.cuh.

The reference computes its cells with geogram's restricted Voronoi diagram and relaxes with geogram's initial sampling
and HLBFGS Newton iterations, none of which is available; DESIGN.md §3 defines the results exactly instead (cells,
restricted cells, centroid rows, the initial samples, the Lloyd step and the L-BFGS Newton phase)."""
import numpy as _np

from . import _pcu_internal
from ._call import (_INDEX_KINDS, _call_args, _dtype_name, _form, _ordinal, _run, _same_device, _to_device, _torch,
                    _validate_mesh)

# Cells (for restricted cells: (face, seed) pairs) handled by each pass (first pass, longer neighbour lists, all seeds)
# in the last call of this module's functions, in any thread (a plain module global, for tests and tools): the fallback
# passes are otherwise invisible.
last_pass_counts = (0, 0, 0)
# The CVT energy of the starting point and of every accepted Newton step of the last lloyd_3d / lloyd_2d /
# sample_mesh_lloyd call.
last_newton_energies = []


def voronoi_centroids_unit_cube(centers, *, device=None):
    """
    Compute the centroids of a 3d voronoi diagram restricted to the unit cube [0, 1]^3

    Args:
      centers : A [n, 3] array where each row is a point in a voronoi diagram restricted to
               the unit cube [0, 1]^3 (float32 / float64 numpy array, CUDA tensor or CPU tensor)
      device: see `k_nearest_neighbors` (keyword only).

    Returns:
      voronoi_ctrs : a [n, 3] float64 array of centroids where each row is the centroid of the corresponding voronoi
                     cell in the input centers (a CUDA tensor for a CUDA tensor, a CPU tensor for a CPU tensor).

    Row i is the centroid of {x in [0,1]^3 : |x - c_i| <= |x - c_j| for every c_j != c_i} when that cell's volume is
    above 1e-30.  Seeds at one position share one cell, which the lowest index owns; every other row (an empty cell)
    is the seed itself -- the reference leaves such rows uninitialised.
    """
    form = _form([centers], ["centers"])
    if _dtype_name(centers) not in ("float32", "float64"):
        raise ValueError("Invalid scalar type (%s) for argument 'centers'. Expected one of ['float32', 'float64']."
                         % _dtype_name(centers))
    shape = tuple(centers.shape)
    if len(shape) != 2 or shape[1] != 3:
        raise ValueError("Invalid shape for centers, must be (n, 3) but got " + str(shape))
    n = shape[0]
    torch = _torch()
    if n == 0:
        if form == "numpy":
            return _np.zeros((0, 3), dtype=_np.float64)
        if form == "cuda":
            _same_device(centers, device)
        return torch.zeros((0, 3), dtype=torch.float64, device=centers.device)
    if form != "cuda":
        host = centers if form == "numpy" else centers.detach().numpy()
        if ((host < 0) | (host > 1) | _np.isnan(host)).any():
            raise ValueError("Centers of voronoi diagram must lie in the unit cube [0, 1]^3")

    def body(x, dev, stream):
        global last_pass_counts
        x = x.to(torch.float64).contiguous()                            # float32 widens exactly
        if form == "cuda" and bool(((x < 0) | (x > 1) | torch.isnan(x)).any().item()):
            raise ValueError("Centers of voronoi diagram must lie in the unit cube [0, 1]^3")
        out = torch.empty_like(x)
        last_pass_counts = tuple(_pcu_internal._voronoi_centroids_device(x.data_ptr(), n, 3, out.data_ptr(), 0, dev, stream))
        return out

    return _run(form, [centers], device, body)


def _cell_moments(centers, *, device=None):
    """(centroid rows, moments) of a float64 numpy array of (n, 2) or (n, 3) seeds in the unit square / cube, n >= 1,
    as numpy arrays; moments (n, 5): volume, first moment about the seed (x, y, z; z = 0 in 2-D) and second moment
    about the seed of every cell.  Not part of the public interface: the cells the relaxations see, for tests."""
    global last_pass_counts
    torch = _torch()
    host = _np.ascontiguousarray(centers, dtype=_np.float64)
    n, dim = host.shape
    x, = _to_device([host], device)
    out = torch.empty_like(x)
    mom = torch.empty((n, 5), dtype=torch.float64, device=x.device)
    last_pass_counts = tuple(_pcu_internal._voronoi_centroids_device(x.data_ptr(), n, dim, out.data_ptr(), mom.data_ptr(),
                                                                     *_call_args(x)))
    return out.cpu().numpy(), mom.cpu().numpy()


def _lloyd(n, num_lloyd, num_newton, dim, device):
    global last_pass_counts, last_newton_energies
    n = int(n)
    if n <= 0:
        raise ValueError("n must be a positive integer. Got n = %d" % n)
    seed = int(_np.random.randint(2 ** 31 - 1))
    torch = _torch()
    out = torch.empty((n, dim), dtype=torch.float64, device=torch.device("cuda", _ordinal(device)))
    energies, passes = _pcu_internal._lloyd_device(n, dim, seed, int(num_lloyd), int(num_newton), out.data_ptr(),
                                                   *_call_args(out))
    last_pass_counts = tuple(passes)
    last_newton_energies = list(energies)
    return out.cpu().numpy()


_LLOYD_DEFINITION = """
    The initial sample is a pure function of (n, seed, dimension), the seed drawn as int(np.random.randint(2**31 - 1))
    (seed NumPy for reproducible results); num_lloyd steps then move every point to its cell's centroid, and at most
    num_newton L-BFGS steps (memory 7, Armijo backtracking inside the unit cube) decrease the CVT energy
    sum_i int_{V_i} |y - x_i|^2 dy.  num_lloyd <= 0 / num_newton <= 0 skip their phase.  DESIGN.md §3 states the
    definitions; geogram's initial sampling and HLBFGS, which the reference uses, cannot be reproduced.
"""


def lloyd_2d(n, num_lloyd=10, num_newton=10, *, device=None):
    return _lloyd(n, num_lloyd, num_newton, 2, device)


def lloyd_3d(n, num_lloyd=10, num_newton=10, *, device=None):
    return _lloyd(n, num_lloyd, num_newton, 3, device)


lloyd_2d.__doc__ = """
    Generate n samples in the unit square, [0, 1]^2 using Lloyd's algorithm
    (https://en.wikipedia.org/wiki/Lloyd%27s_algorithm).

    Args:
      n : The number of 2d point samples to generate
      num_lloyd : The number of Lloyd iterations to do (default 10)
      num_newton : The number of Newton iterations to do when computing Voronoi diagrams (default 10)
      device: see `k_nearest_neighbors` (keyword only).

    Returns:
      lloyd_points : a (n, 2)-shaped float64 numpy array of point samples in the unit square [0, 1]^2
""" + _LLOYD_DEFINITION

lloyd_3d.__doc__ = """
    Generate n samples in the unit cube, [0, 1]^3 using Lloyd's algorithm
    (https://en.wikipedia.org/wiki/Lloyd%27s_algorithm).

    Args:
      n : The number of 3d point samples to generate
      num_lloyd : The number of Lloyd iterations to do (default 10)
      num_newton : The number of Newton iterations to do when computing Voronoi diagrams (default 10)
      device: see `k_nearest_neighbors` (keyword only).

    Returns:
      lloyd_pts : a (n, 3)-shaped float64 numpy array of point samples in the unit cube [0, 1]^3
""" + _LLOYD_DEFINITION


def _restricted_cell_moments(seeds, v, f, *, device=None):
    """Moments (n, 5) of the cells of (n, 3) seeds restricted to the mesh (v, f), numpy arrays in and out (v float32 or
    float64, widened exactly; f of any of the four index dtypes), n >= 1: area, first moment about the seed (x, y, z)
    and second moment about the seed of every cell.  Not part of the public interface: the cells sample_mesh_lloyd
    sees, for tests."""
    global last_pass_counts
    torch = _torch()
    seeds = _np.ascontiguousarray(seeds, dtype=_np.float64)
    _validate_mesh(v, f, tuple(_INDEX_KINDS))
    n = seeds.shape[0]
    result = {}

    def body(vt, ft, st, dev, stream):
        vt = vt.to(torch.float64).contiguous()
        mom = torch.empty((n, 5), dtype=torch.float64, device=vt.device)
        result["passes"] = _pcu_internal._restricted_voronoi_moments_device(
            st.data_ptr(), n, vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(), int(ft.shape[0]), _INDEX_KINDS[_dtype_name(f)],
            mom.data_ptr(), dev, stream)
        return mom

    mom = _run("numpy", [v, f, seeds], device, body)
    last_pass_counts = tuple(result["passes"])
    return mom


def sample_mesh_lloyd(v, f, num_samples, num_lloyd=10, num_newton=10, return_mesh=False, *, device=None):
    """
    Sample points on a mesh surface using Lloyd's algorithm

    Args:
      v : (#v, 3)-shaped array of mesh vertex positions (float32 / float64)
      f : (#f, 3)-shaped array of mesh face indices (int32 / int64 / uint32 / uint64)
      num_samples : the number of samples to generate (> 0)
      num_lloyd : the number of Lloyd iterations to do (default 10)
      num_newton : the number of Newton iterations to do when computing Voronoi diagrams (default 10)
      return_mesh : accepted and ignored, as in the reference (whose binding does not use it)
      device: see `k_nearest_neighbors` (keyword only).

    Returns:
      points : a (num_samples, 3)-shaped float64 array of samples (numpy for numpy inputs, a CUDA tensor for CUDA
               tensors, a CPU tensor for CPU tensors)

    All arithmetic is fp64 (float32 v is widened exactly first).  The cell of sample x_i is the part of the surface
    nearer to x_i than to any other sample, R_i = {y on the faces : |y - x_i|^2 <= |y - x_j|^2 for every x_j != x_i}
    (samples at one position share one cell, owned by the lowest index; faces of zero area contribute nothing).  The
    initial sample is the first num_samples samples of sample_mesh_random on the fp64 vertices with the seed
    int(np.random.randint(2**31 - 1)) (seed NumPy for reproducible results), at positions fl((b0 a + b1 b) + b2 c) per
    axis; num_lloyd steps then move every point to its cell's centroid (a point whose cell has area <= 1e-30 stays),
    and at most num_newton L-BFGS steps (memory 7, Armijo backtracking, no domain test) decrease the energy
    sum_i int_{R_i} |y - x_i|^2 dA.  Centroids are not projected onto the surface: the centroid of a cell on a curved
    surface lies slightly off it.  Two calls with the same NumPy state give bit-identical points.  DESIGN.md §3 states
    the definitions; geogram's initial sampling and HLBFGS, which the reference uses, cannot be reproduced.
    Divergence: a face corner outside [0, #v) raises ValueError (the reference reads out of bounds).
    """
    global last_pass_counts, last_newton_energies
    form = _form([v, f], ["v", "f"])
    _validate_mesh(v, f, tuple(_INDEX_KINDS))
    n = int(num_samples)
    if n <= 0:
        raise ValueError("num_samples must be > 0")
    seed = int(_np.random.randint(2 ** 31 - 1))
    torch = _torch()
    kind = _INDEX_KINDS[_dtype_name(f)]
    result = {}

    def body(vt, ft, dev, stream):
        vt = vt.to(torch.float64).contiguous()
        out = torch.empty((n, 3), dtype=torch.float64, device=vt.device)
        result["energies"], result["passes"] = _pcu_internal._sample_mesh_lloyd_device(
            vt.data_ptr(), int(vt.shape[0]), ft.data_ptr(), int(ft.shape[0]), kind, n, seed, int(num_lloyd), int(num_newton),
            out.data_ptr(), dev, stream)
        return out

    out = _run(form, [v, f], device, body)
    last_pass_counts = tuple(result["passes"])
    last_newton_energies = list(result["energies"])
    return out
