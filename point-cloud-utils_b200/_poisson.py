"""downsample_point_cloud_poisson_disk -- the reference's name, arguments and defaults
(/root/reference/src/sample_point_cloud.cpp:240-333), computed by csrc/poisson.cuh.

Inputs and results take the forms of _call.py; the cloud is uploaded once, whatever the number of radii the
target-count search tries."""
import numpy as _np

from . import _pcu_internal
from ._call import _dtype_name, _form, _run, _same_device, _torch


def target_search(sample, dtype, bbsize, target, tolerance):
    """The reference's search for a radius whose sample has about `target` rows (:285-326), with sample(radius) -> row
    count.  Radii are the cloud's scalar type T, updated as the reference computes them: `range /= 2.0` and
    `range *= 2.0` in double, then narrowed to T; the midpoint `(lo + hi) / 2.0` adds in T first.  The sample of the
    last call is the result.  bbsize == 0 (every row the same point) is the caller's: there the reference's doubling
    loop never ends."""
    T = _np.dtype(dtype).type
    tol = _np.float32(tolerance)                                   # the binding takes a float (:258)
    num_min = int(T(target) * T(_np.float32(1.0) - tol))           # int(T(target) * (1.0f - tol)) (:285-286)
    num_max = int(T(target) * T(_np.float32(1.0) + tol))
    lo = hi = T(float(bbsize) / 50.0)
    while True:                                                    # :296-301
        lo = T(float(lo) / 2.0)
        count = sample(lo)
        if not count < target:
            break
    while True:                                                    # :303-308
        hi = T(float(hi) * 2.0)
        count = sample(hi)
        if not count > target:
            break
    it = 0
    while it < 20 and (count < num_min or count > num_max):        # :311-326
        it += 1
        cur = T(float(T(lo + hi)) / 2.0)
        count = sample(cur)
        if count > target:
            lo = cur
        if count < target:
            hi = cur
    return count


def _box_size(lo, hi, T):
    """(bmax - bmin).norm() in the cloud's scalar type (:288-290)."""
    d = (_np.asarray(hi, dtype=T) - _np.asarray(lo, dtype=T)).astype(T)
    with _np.errstate(over="ignore"):
        return T(_np.sqrt(T(T(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])))


def downsample_point_cloud_poisson_disk(v, radius, target_num_samples=-1, random_seed=0, sample_num_tolerance=0.04, *,
                                        device=None):
    """
    Downsample a point set so that samples are approximately evenly spaced.

    Args:
        v: #v by 3 array of vertex positions (float32 / float64 numpy array or CUDA tensor)
        radius: desired separation between points.
        target_num_samples: If set to a positive value, iterate to generate points as close to this target as possible
                            (determined by sample_num_tolerance).
        random_seed: A random seed used to generate the samples (a 32-bit integer).  Passing in 0 draws the seed from
                     NumPy's global random state (the reference uses the current time): seed NumPy for reproducible
                     results.
        sample_num_tolerance: If you requested a target number of samples, by passing num_samples > 0, then this
                              function will return between (1 - sample_num_tolerance) * num_samples and
                              (1 + sample_num_tolerance) * num_samples, unless 20 bisection steps do not get there (as
                              in the reference).  Must be in (0, 1].
        device: see `k_nearest_neighbors` (keyword only).

    Returns:
        p_idx : A (m,) shaped int32 array of indices into v where m is the number of Poisson-disk samples, ascending.

    Mirrors /root/reference/src/sample_point_cloud.cpp:240-333 (and blue_noise_downsample, :14-109).  The reference's
    subset comes from libigl's blue-noise helpers, std::mt19937 and the iteration order of a hash map, none of which
    can be reproduced, so the sample is defined exactly instead, as a pure function of (v, radius, seed):
      - r is radius in v's precision and rr = r * r rounded in that precision (the reference's `const double rr =
        r*r` with r of that type).  Rows p and q conflict when their squared distance, ((dx^2 + dy^2) + dz^2) with
        every operation rounded in v's precision, is below rr.  Whether a pair at exactly rr conflicts in the reference
        depends on libigl's distance expression, which is not available: parity is unpinned there.
      - Every row has the priority (h(row), row), h(row) = mix32(seed ^ mix32(row * 0x9E3779B9 + 0x85EBCA6B)).
      - The sample is the greedy maximal independent set in priority order: rows are visited by ascending priority
        and kept when they conflict with no kept row.  No two samples are closer than r, and every row is a sample or
        conflicts with one.
    With target_num_samples > 0 the radius is searched as in the reference (:278-326) and radius is ignored; the
    result is the sample of the last radius tried.  target_num_samples >= len(v) returns arange(len(v)).
    Divergences: rows come back ascending (the reference's order is its hash map's); when every row is the same point
    and target_num_samples < len(v), the reference's search never ends (its radius stays 0), while here the one sample
    any positive radius gives -- the row of smallest priority -- is returned.
    """
    target = int(target_num_samples)
    if target <= 0 and radius <= 0.0:                                       # :265-267
        raise ValueError("Cannot have both num_samples <= 0 and radius <= 0")
    if float(_np.float32(sample_num_tolerance)) > 1.0 or float(_np.float32(sample_num_tolerance)) <= 0.0:   # :268-270
        raise ValueError("sample_num_tolerance must be in (0, 1]")
    form = _form([v], ["v"])
    if _dtype_name(v) not in ("float32", "float64"):
        raise ValueError("Invalid scalar type (%s) for argument 'v'. Expected one of ['float32', 'float64']." % v.dtype)
    if len(v.shape) != 2 or v.shape[1] != 3:
        raise ValueError("Invalid shape for v, must be (n, 3) but got " + str(tuple(v.shape)))
    n = int(v.shape[0])
    if n == 0 or 0 < n <= target:                                            # :279-283
        if form == "numpy":
            return _np.arange(n, dtype=_np.int32)
        if form == "cuda":
            _same_device(v, device)
        torch = _torch()
        return torch.arange(n, dtype=torch.int32, device=v.device)
    seed = int(random_seed) & 0xFFFFFFFF
    if seed == 0:
        seed = int(_np.random.randint(2 ** 31 - 1))
    T = _np.float64 if _dtype_name(v) == "float64" else _np.float32
    torch = _torch()

    def body(pts, dev, stream):
        idx = torch.empty(n, dtype=torch.int32, device=pts.device)
        count = torch.empty(1, dtype=torch.int64, device=pts.device)

        def sample(r):
            _pcu_internal._poisson_disk_device(pts.dtype == torch.float64, pts.data_ptr(), n, float(r), seed, idx.data_ptr(),
                                               count.data_ptr(), 0, dev, stream)
            return int(count.item())

        if target <= 0:
            return idx[:sample(radius)]         # radius narrowed to T by the library
        lo, hi = torch.stack((pts.amin(dim=0), pts.amax(dim=0))).cpu().numpy()
        if _box_size(lo, hi, T) == 0:
            return idx[:sample(T(1))]           # every row conflicts with every other: one sample
        return idx[:target_search(sample, T, _box_size(lo, hi, T), target, sample_num_tolerance)]

    return _run(form, [v], device, body)
