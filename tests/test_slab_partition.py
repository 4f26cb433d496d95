"""GPU: the slab partition stages a tile in slab order when its slabs are few enough (about one point per
slab per tile or more) and stores point by point otherwise.  A cloud on each side of that choice, binned
by the slab build (options.binning = 3), gives what the cell-wise passes (binning = 1) give."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


# 1e6 fp32 points cut into 489 slabs (staged); 3e6 fp64 points into 2930 slabs (point by point)
@pytest.mark.parametrize("dtype,n", [(np.float32, 1_000_000), (np.float64, 3_000_000)])
def test_both_partition_paths_match_the_cell_wise_build(pcu, dtype, n):
    rng = np.random.default_rng(2024)
    big = rng.random((n, 3)).astype(dtype)
    small = rng.random((100_000, 3)).astype(dtype)
    got = {}
    for mode in (1, 3):
        pcu._pcu_internal._set_defaults(binning=mode)
        try:
            got[mode] = (pcu.k_nearest_neighbors(small, big, 4), pcu.k_nearest_neighbors(big, small, 1),
                         float(pcu.chamfer_distance(big, small)))
        finally:
            pcu._pcu_internal._set_defaults()
    for a, b in zip(got[1][:2], got[3][:2]):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])
    assert abs(got[3][2] - got[1][2]) <= 1e-6 * abs(got[1][2])
