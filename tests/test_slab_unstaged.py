"""GPU: a cloud with more slabs than a partition tile has points (kSlabTile = 2048) takes the point-by-point
partition.  At a mean slab of 3/4 of the staging buffer that needs more than 2048 * 3072 fp32 points (the 10^7-point
cloud of the k = 16 benchmark has 3256 slabs); 7e6 points make 2279 slabs.  The slab build (options.binning = 3)
gives what the cell-wise passes (binning = 1) give."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_point_by_point_partition_matches_the_cell_wise_build(pcu):
    rng = np.random.default_rng(7)
    big = rng.random((7_000_000, 3), dtype=np.float32)
    small = rng.random((50_000, 3), dtype=np.float32)
    got = {}
    for mode in (1, 3):
        pcu._pcu_internal._set_defaults(binning=mode)
        try:
            got[mode] = (pcu.k_nearest_neighbors(small, big, 4), float(pcu.chamfer_distance(big, small)))
        finally:
            pcu._pcu_internal._set_defaults()
    (d1, i1), (d3, i3) = got[1][0], got[3][0]
    assert np.array_equal(i1, i3) and np.array_equal(d1, d3)
    assert abs(got[3][1] - got[1][1]) <= 1e-6 * abs(got[1][1])
