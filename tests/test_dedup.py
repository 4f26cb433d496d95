"""Duplicate removal (SURVEY.md 8f, N2; /root/reference/src/remove_duplicates.cpp:11-79, :108-176).

Integer work apart from the rounding division: unique rows, their order, both index maps and the re-indexed faces are
compared bit for bit with the oracle's numpy restatement of libigl's round + unique_rows (libigl is not in the reference
tree: parity unpinned, anchored on the published algorithm and on the properties the reference's own tests assert,
tests/test_examples.py:509-531)."""
import numpy as np
import pytest


def _cloud_with_duplicates(rng, n, dtype, dup_share=0.3):
    base = rng.random((n, 3)).astype(dtype)
    pick = rng.integers(0, n, int(n * dup_share))
    pts = np.concatenate([base, base[pick]])
    return pts[rng.permutation(len(pts))]


def test_oracle_conventions(oracle):
    rng = np.random.default_rng(0)
    v = _cloud_with_duplicates(rng, 2000, np.float64)
    v2, i_v_to_v2, i_v2_to_v = oracle.deduplicate_point_cloud(v, 1e-11, return_index=True)
    assert v2.shape[0] == 2000 and v2.shape[0] < v.shape[0]                  # tests/test_examples.py:517-520
    assert np.all(np.equal(v2[i_v2_to_v], v)) and np.all(np.equal(v[i_v_to_v2], v2))
    assert i_v_to_v2.dtype == np.int32 and i_v2_to_v.dtype == np.int32
    assert np.all(np.lexsort(v2.T[::-1])[:] == np.arange(len(v2)))           # ascending lexicographic rows
    # std::round: halves away from zero, in the cloud's precision
    p = np.array([[0.5, -0.5, 1.5], [2.5, -2.5, 0.49999997], [1.4999999, 0.0, -0.0]], dtype=np.float32)
    sv, svi, svj = oracle.deduplicate_point_cloud(p, 1.0)
    assert len(sv) == 3
    q = np.array([[0.5, 0.5, 0.5], [1.4, 1.2, 0.6], [0.6, 0.7, 1.49]], dtype=np.float32)    # all round to (1, 1, 1)
    sv, svi, svj = oracle.deduplicate_point_cloud(q, 1.0)
    assert len(sv) == 1 and svi[0] == 0 and np.array_equal(svj, [0, 0, 0]) and np.array_equal(sv[0], q[0])
    # mesh: a face with two merged corners disappears
    vv = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [1, 1, 0]], dtype=np.float64)
    ff = np.array([[0, 1, 2], [3, 1, 4], [0, 3, 1]], dtype=np.int32)
    v2, f2, svi, svj = oracle.deduplicate_mesh_vertices(vv, ff, 0.0)
    assert len(v2) == 4 and f2.shape == (2, 3) and np.array_equal(v2[f2], vv[ff[:2]])


def test_argument_errors(pcu):
    with pytest.raises(ValueError, match="3D"):
        pcu.deduplicate_point_cloud(np.zeros((10, 2)), 0.1)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.deduplicate_point_cloud(np.zeros((10, 3), dtype=np.int32), 0.1)
    with pytest.raises(ValueError, match="scalar type"):
        pcu.deduplicate_mesh_vertices(np.zeros((10, 3)), np.zeros((4, 3)), 0.1)
    with pytest.raises(ValueError):
        pcu.deduplicate_mesh_vertices(np.zeros((10, 3)), None, 0.1)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("eps", [0.0, 1e-11, 1e-3, 0.05])
def test_points_match_the_oracle(pcu, oracle, dtype, eps):
    rng = np.random.default_rng(17)
    v = _cloud_with_duplicates(rng, 30000, dtype) - dtype(0.4)               # negative coordinates too
    v[rng.integers(0, len(v), 50)] = 0.0
    v[rng.integers(0, len(v), 50), 1] = -0.0
    ref = oracle.deduplicate_point_cloud(v, eps)
    got = pcu.deduplicate_point_cloud(v, eps)
    assert [a.dtype for a in got] == [dtype, np.int32, np.int32]
    for g, r in zip(got, ref):
        assert g.shape == r.shape and np.array_equal(g, r)
    v2, i_v_to_v2, i_v2_to_v = got
    assert np.all(np.equal(v[i_v_to_v2], v2))
    if eps <= 1e-11:
        assert np.all(np.equal(v2[i_v2_to_v], v))                            # the reference's own assertion
    only = pcu.deduplicate_point_cloud(v, eps, return_index=False)
    assert isinstance(only, np.ndarray) and np.array_equal(only, v2)


@pytest.mark.gpu
def test_sort_sizes_and_patterns(pcu, oracle):
    """Tile boundaries of the radix sort (4096 records per CTA), all-equal and all-distinct clouds, constant digits."""
    rng = np.random.default_rng(3)
    for n in (1, 2, 31, 4095, 4096, 4097, 8193, 70001):
        v = np.round(rng.random((n, 3)) * 7).astype(np.float32)              # few distinct values: long runs of equal rows
        for g, r in zip(pcu.deduplicate_point_cloud(v, 0.0), oracle.deduplicate_point_cloud(v, 0.0)):
            assert np.array_equal(g, r), n
    same = np.tile(np.array([[0.25, -3.0, 7.5]]), (10000, 1))
    sv, svi, svj = pcu.deduplicate_point_cloud(same, 0.0)
    assert sv.shape == (1, 3) and svi[0] == 0 and not svj.any()
    big = (rng.random((300000, 3)) * 1e6).astype(np.float64)                 # wide exponent range: every digit pass is live
    for g, r in zip(pcu.deduplicate_point_cloud(big, 0.0), oracle.deduplicate_point_cloud(big, 0.0)):
        assert np.array_equal(g, r)
    many = np.round(rng.random((1100000, 3)) * 200).astype(np.float32)      # 269 tiles: the scan over a digit's tile counts takes two rounds
    for g, r in zip(pcu.deduplicate_point_cloud(many, 0.0), oracle.deduplicate_point_cloud(many, 0.0)):
        assert np.array_equal(g, r)
    x, i, j = pcu.deduplicate_point_cloud(np.zeros((0, 3), dtype=np.float32), 0.1)
    assert x.shape == (0, 3) and i.shape == (0,) and j.shape == (0,)


@pytest.mark.gpu
@pytest.mark.parametrize("itype", [np.int32, np.int64])
def test_mesh_matches_the_oracle(pcu, oracle, itype):
    import torch
    rng = np.random.default_rng(5)
    v = _cloud_with_duplicates(rng, 20000, np.float32)
    f = rng.integers(0, len(v), (50000, 3)).astype(itype)
    f[::7, 1] = f[::7, 0]                                                     # degenerate already
    ref = oracle.deduplicate_mesh_vertices(v, f, 1e-11)
    got = pcu.deduplicate_mesh_vertices(v, f, 1e-11)
    assert got[1].dtype == itype and got[1].shape[1] == 3 and 0 < len(got[1]) < len(f)
    for g, r in zip(got, ref):
        assert g.shape == r.shape and np.array_equal(g, r)
    v2, f2 = pcu.deduplicate_mesh_vertices(v, f, 1e-11, return_index=False)
    assert np.array_equal(v2, got[0]) and np.array_equal(f2, got[1])
    with pytest.raises(ValueError, match="outside"):
        bad = f.copy(); bad[3, 2] = len(v)
        pcu.deduplicate_mesh_vertices(v, bad, 1e-11)
    # CUDA tensors in, CUDA tensors out
    tv, tf = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    out = pcu.deduplicate_mesh_vertices(tv, tf, 1e-11)
    assert all(t.is_cuda for t in out)
    for t, r in zip(out, ref):
        assert np.array_equal(t.cpu().numpy(), r)
    # quads (the reference loops over F.cols())
    q = rng.integers(0, len(v), (4000, 4)).astype(itype)
    for g, r in zip(pcu.deduplicate_mesh_vertices(v, q, 0.0), oracle.deduplicate_mesh_vertices(v, q, 0.0)):
        assert np.array_equal(g, r)
