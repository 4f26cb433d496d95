"""The Hausdorff witness of the fused Chamfer sweeps, taken from whichever pass answered the maximal query.

The main pass (3 x 3 x 3 cells per query) tracks distances only; queries it cannot settle go to the far pass
(the whole 5 x 5 x 5 window in one round) and from there to the very-far pass (occupancy pyramid).  The far
and very-far passes carry the neighbour and tie flag of their maximum into the statistics; a maximum answered
by the main pass gets its witness from one more round over its 27 cells.

The dataset is a jittered lattice (spacing s, about 1.1 s per cell at the k = 1 cell occupancy), so every
query inside it is settled by the main pass.  One query sits at the centre of a spherical hole cut out of the
lattice, near the middle of a cell: with no hole the maximum comes from the main pass, a hole of radius
2.2 s - 2.5 s puts it beyond the 27 cells (1.5 cells away) but inside the 125-cell window (2.5 cells away), and
one of 8 s puts it on the very-far list.  Variants place exactly two points at the hole's rim, equidistant from
the query (a tie decided in the far pass), and make every distance a tie (a query lattice at the dataset
lattice's cell centres).  Coordinates are multiples of 2^-10, so every squared distance is exact in both precisions.

Each case checks the raw statistics records (argmax_data = lowest tied index, witness_tied) against numpy,
the public Hausdorff results against the oracle, and the k = 1 neighbours of every query (the far pass of the
k-NN sweep) against the oracle, through plain CUDA-tensor calls, host calls, a prepared target and the batch.
"""
import numpy as np
import pytest

F32, F64 = np.float32, np.float64
STATS_WORDS = 10
SPACING = 32        # lattice spacing in units of 2^-10
SIDE = 20           # dataset lattice points per axis


def decode_records(words):
    w = np.asarray(words, dtype=np.int64).reshape(-1, STATS_WORDS)
    f = w.view(np.float64)
    return [{"max_sq_dist": float(f[r, 2]), "argmax_query": int(w[r, 3]), "argmax_data": int(w[r, 4]),
             "n_far": int(w[r, 7]), "witness_tied": int(w[r, 8])} for r in range(len(w))]


def make_case(kind, dtype):
    """(x, y): queries and dataset, coordinates k / 1024."""
    rng = np.random.default_rng({"main": 1, "far22": 2, "far24": 3, "vfar": 4, "tie": 5, "lattice": 6}[kind])
    g = np.arange(SIDE)
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) * SPACING + SPACING // 2
    if kind == "lattice":   # every query at a lattice cell centre: eight neighbours at one distance
        c = np.arange(SIDE - 1)
        x = np.stack(np.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3) * SPACING + SPACING
        y = lat
    else:
        y = lat + rng.integers(-3, 4, lat.shape)
        x = rng.integers(2 * SPACING, (SIDE - 2) * SPACING, (6000, 3))
        centre = np.array([312, 347, 312])   # near the middle of a cell (about 35 units wide, starting at 13)
        radius = {"main": 0, "far22": 2.2, "far24": 2.4, "vfar": 8.0, "tie": 2.5}[kind] * SPACING
        if radius:
            y = y[np.linalg.norm(y - centre, axis=1) > radius + 4]
            x = np.concatenate([x[np.linalg.norm(x - centre, axis=1) > radius + 4], centre[None]])
        if kind == "tie":   # two points on the rim, equidistant from the centre query, nearer than any other
            rim = int(radius)
            y = np.concatenate([y, centre + [[rim, 0, 0], [0, -rim, 0]]])
        x = x[rng.permutation(len(x))]
        y = y[rng.permutation(len(y))]
    return np.ascontiguousarray(x / 1024.0, dtype=dtype), np.ascontiguousarray(y / 1024.0, dtype=dtype)


def witness(q, d, dtype):
    """Lowest index of q's nearest points in d (the metric's rounding, in the input precision) and whether tied."""
    q = q.astype(dtype)
    diff = q[None, :] - d
    d2 = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
    at = np.flatnonzero(d2 == d2.min())
    return int(at[0]), int(len(at) > 1), float(d2.min())


def check_record(rec, x, y, dtype, oracle_h):
    """One direction's raw record against the oracle's maximum and numpy's witness of the maximal query."""
    value, row, _ = oracle_h
    assert rec["argmax_query"] == row, (rec["argmax_query"], row)
    j, tied, d2 = witness(x[row], y, dtype)
    assert rec["max_sq_dist"] == d2
    assert (rec["argmax_data"], rec["witness_tied"]) == (j, tied), (rec, j, tied)


KINDS = ["main", "far22", "far24", "vfar", "tie", "lattice"]
WITNESS = ("max_sq_dist", "argmax_query", "argmax_data", "witness_tied")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("kind", KINDS)
def test_witness_from_each_pass(pcu, oracle, kind, dtype):
    import torch
    x, y = make_case(kind, dtype)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    hxy = oracle.one_sided_hausdorff_distance(x, y, True)
    hyx = oracle.one_sided_hausdorff_distance(y, x, True)

    buf, _ = pcu._stats_device(xt, yt, True, 10)
    recs = decode_records(buf.cpu().numpy())
    check_record(recs[0], x, y, dtype, hxy)
    check_record(recs[1], y, x, dtype, hyx)
    if kind == "main":
        assert recs[0]["n_far"] == 0   # every query of the lattice's interior settles in its 27 cells
    elif kind != "lattice":
        assert recs[0]["n_far"] >= 1
    if kind in ("tie", "lattice"):
        assert recs[0]["witness_tied"] == 1

    # the host call hands back its records with tied witnesses already replayed in the reference's tie order
    _, sxy, syx = pcu._pcu_internal._chamfer_stats(x, y)
    for got, want, h in ((sxy, recs[0], hxy), (syx, recs[1], hyx)):
        assert (got["max_sq_dist"], got["argmax_query"]) == (want["max_sq_dist"], want["argmax_query"])
        assert got["argmax_data"] == h[2]

    target = pcu.prepare_cloud(yt)
    try:
        _, _, _, (pbuf, _) = pcu._prepared_stats(xt, target, True, 10, None)
        prec = decode_records(pbuf.cpu().numpy())
        for got, want in zip(prec, recs):
            assert {k: got[k] for k in WITNESS} == {k: want[k] for k in WITNESS}
        assert pcu.one_sided_hausdorff_distance(xt, target, return_index=True) == hxy
    finally:
        target.close()

    # public results: the witness after the library's tie-order replay is the reference's
    assert pcu.one_sided_hausdorff_distance(x, y, return_index=True) == hxy
    assert pcu.one_sided_hausdorff_distance(yt, xt, return_index=True) == hyx
    assert pcu.hausdorff_distance(x, y, return_index=True) == oracle.hausdorff_distance(x, y, return_index=True)
    assert float(pcu.chamfer_distance(xt, yt)) == pytest.approx(float(oracle.chamfer_distance(x, y)), rel=1e-6)

    # the k = 1 k-NN sweep's far pass answers the same queries with per-point outputs
    d, i = pcu.k_nearest_neighbors(xt, yt, 1)
    rd, ri = oracle.k_nearest_neighbors(x, y, 1)
    assert np.array_equal(i.cpu().numpy().reshape(-1), ri.reshape(-1))
    assert np.array_equal(d.cpu().numpy().reshape(-1), rd.reshape(-1))


@pytest.mark.gpu
def test_witness_in_the_batch(pcu, oracle):
    """Every case as one pair of a batch (fp32), each padded to the batch's sizes by repeating its last point; the
    records are checked against the padded pairs."""
    import torch
    pairs = [make_case(kind, F32) for kind in KINDS]
    n = max(len(a) for a, _ in pairs)
    m = max(len(b) for _, b in pairs)
    pad = lambda a, k: np.concatenate([a, np.repeat(a[-1:], k - len(a), 0)])
    xs = np.stack([pad(a, n) for a, _ in pairs])
    ys = np.stack([pad(b, m) for _, b in pairs])
    B = len(pairs)
    xt, yt = torch.from_numpy(xs).cuda(), torch.from_numpy(ys).cuda()
    stats = torch.empty(2 * B * STATS_WORDS, dtype=torch.int64, device=xt.device)
    per_pair = torch.empty(B, dtype=torch.float32, device=xt.device)
    pcu._pcu_internal._batched_chamfer_stats_device(xt.data_ptr(), yt.data_ptr(), B, n, m, stats.data_ptr(),
                                                    per_pair.data_ptr(), 10, xt.device.index or 0,
                                                    torch.cuda.current_stream(xt.device).cuda_stream)
    recs = decode_records(stats.cpu().numpy())
    for p in range(B):
        x, y = xs[p], ys[p]
        check_record(recs[2 * p], x, y, F32, oracle.one_sided_hausdorff_distance(x, y, True))
        check_record(recs[2 * p + 1], y, x, F32, oracle.one_sided_hausdorff_distance(y, x, True))
    assert np.array_equal(pcu.batched_chamfer_distance(xt, yt).cpu().numpy(), per_pair.cpu().numpy())
