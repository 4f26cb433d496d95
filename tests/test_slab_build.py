"""GPU: the slab build of the grid (options.binning = 3) gives the reference's results, on the goldens,
on the inputs of the other builds' parity test, and where a slab holds more points than one CTA can
stage in shared memory."""
import numpy as np
import pytest

import test_gpu_parity as parity
from conftest import knn_golden_names, metric_golden_names

pytestmark = pytest.mark.gpu
REL = 1e-6


@pytest.fixture
def slab_build(pcu):
    pcu._pcu_internal._set_defaults(binning=3)
    try:
        yield
    finally:
        pcu._pcu_internal._set_defaults()


def test_slab_build_gives_the_reference_results(pcu, oracle, slab_build):
    parity.test_both_grid_builds_give_the_reference_results(pcu, oracle, 3)


@pytest.mark.parametrize("name", knn_golden_names())
def test_slab_build_knn_goldens(pcu, slab_build, name):
    parity.test_knn_matches_reference_goldens(pcu, name)


@pytest.mark.parametrize("name", metric_golden_names())
def test_slab_build_metric_goldens(pcu, slab_build, name):
    parity.test_metrics_match_reference_goldens(pcu, name)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("clustered_side", ["queries", "dataset"])
def test_oversized_slab(pcu, oracle, dtype, clustered_side):
    """40 000 distinct points inside a cube 1e-4 wide all fall into one cell, so their slab holds far
    more points than the shared-memory staging buffer; 60 000 uniform points fill the rest of the box."""
    rng = np.random.default_rng(77)
    cluster = 0.3 + 1e-4 * rng.random((40000, 3))
    cloud = np.concatenate([cluster, rng.random((60000, 3))]).astype(dtype)
    cloud = cloud[rng.permutation(len(cloud))]
    other = rng.random((50000, 3)).astype(dtype)
    q, d = (cloud, other) if clustered_side == "queries" else (other, cloud)
    for mode in (0, 3):   # automatic mode takes the slab build for a single pair too
        pcu._pcu_internal._set_defaults(binning=mode)
        try:
            for k in (1, 4):
                got = pcu.k_nearest_neighbors(q, d, k)
                ref = oracle.k_nearest_neighbors(q, d, k)
                assert np.array_equal(got[1], ref[1]) and np.array_equal(got[0], ref[0]), (mode, k)
            ref = float(oracle.chamfer_distance(q, d))
            assert abs(float(pcu.chamfer_distance(q, d)) - ref) <= REL * ref
            assert pcu.hausdorff_distance(q, d, return_index=True) == oracle.hausdorff_distance(q, d, return_index=True)
        finally:
            pcu._pcu_internal._set_defaults()
