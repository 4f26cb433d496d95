"""The point-cloud functions take their input forms and their device from one call path: numpy in -> numpy out, CUDA
tensors in -> CUDA tensors out on their device, CPU tensors in -> CPU tensors out.  The nearest-neighbour family (k-NN,
the Hausdorff distances, Chamfer, prepared clouds, batched Chamfer and the normal estimators) checks its arguments on
that path too, with plain and prepared second arguments alike, before its numpy arrays and CPU tensors go to the
binding's host entry points.
On the CPU: every argument error comes before any device call, numpy arrays and CPU tensors raise the same message for
the same mistake, and device= is read the one way the package reads it.  On the GPU, CUDA tensors raise those messages
too, before any device call.
On the GPU: numpy, CUDA-tensor and CPU-tensor calls of every function give results of the right form, dtype and
device that are bit-identical (voxel means and the EMD value, fp64 sums in the order the device's atomics take: to
rounding), and CUDA tensors with a contradicting device= raise."""
import numpy as np
import pytest


def _boom(*args, **kwargs):
    raise AssertionError("a device call was made before the argument error")


@pytest.fixture
def no_device(monkeypatch):
    """The package with every way to the device replaced by an assertion: uploads (once device= has been checked), and
    the binding's host and device entry points."""
    import pcu_b200 as pcu
    from pcu_b200 import _call

    def upload(device):
        _call._dev(device)
        _boom()

    monkeypatch.setattr(_call, "_ordinal", upload)
    for name in dir(pcu._pcu_internal):
        if name.endswith(("_device", "_internal", "_host")) or name == "_chamfer_stats":
            monkeypatch.setattr(pcu._pcu_internal, name, _boom)
    return pcu


# ---- CPU: argument errors before any device call -------------------------------------------------------------------
def _cases(pcu, torch):
    rng = np.random.default_rng(0)
    p = rng.random((50, 3))
    t = torch.from_numpy(p)
    w = np.ones(5) / 5
    M = rng.random((5, 5))
    f = np.array([[0, 1, 2], [2, 3, 4]])
    return [
        # dense metrics
        (pcu.pairwise_distances, (p[0], p), {}, "Invalid shape for a"),
        (pcu.pairwise_distances, (p[None], np.stack([p, p])), {}, "operands could not be broadcast"),
        (pcu.pairwise_distances, (p.astype(np.int32), p.astype(np.int32)), {}, "Invalid scalar type (int32). Expected one of"),
        (pcu.pairwise_distances, (p, p.astype(np.float32)), {}, "a and b must have the same dtype"),
        (pcu.pairwise_distances, (p, p), {"p": "fro"}, "Invalid norm order"),
        (pcu.pairwise_distances, (p, t), {}, "Invalid type for b"),
        (pcu.pairwise_distances, (t, t.float()), {}, "a and b must have the same dtype"),
        (pcu.sinkhorn, (w, w, M.astype(np.float32), 1e-3), {}, "Tensors a, b, and M must have the same dtype"),
        (pcu.sinkhorn, (np.ones(4) / 4, w, M, 1e-3), {}, "Got unexpected shape for tensor a"),
        (pcu.sinkhorn, (np.ones((2, 5)) / 5, w, M, 1e-3), {}, "Invalid shape for a"),
        (pcu.sinkhorn, (torch.from_numpy(w), torch.from_numpy(w), torch.from_numpy(M).long(), 1e-3), {},
         "Tensors a, b, and M must have the same dtype"),
        (pcu.earth_movers_distance, (p.astype(np.float32), p.astype(np.float32)), {}, "Tensors a, b, and M must have the same dtype"),
        (pcu.earth_movers_distance, (t.float(), t.float()), {}, "Tensors a, b, and M must have the same dtype"),
        # duplicate removal
        (pcu.deduplicate_point_cloud, (p[:, :2], 0.1), {}, "Only 3D inputs are supported"),
        (pcu.deduplicate_point_cloud, (p.astype(np.int32), 0.1), {}, "Invalid scalar type (int32) for argument 'points'"),
        (pcu.deduplicate_point_cloud, (t.int(), 0.1), {}, "Invalid scalar type (int32) for argument 'points'"),
        (pcu.deduplicate_point_cloud, (p, 0.1), {"device": "cuda:99"}, "out of range"),
        (pcu.deduplicate_point_cloud, (p, 0.1), {"device": torch.device("cuda", 99)}, "out of range"),
        (pcu.deduplicate_point_cloud, (t, 0.1), {"device": torch.device("cuda", 99)}, "out of range"),
        (pcu.deduplicate_point_cloud, (p, 0.1), {"device": "gpu"}, "device must be"),
        (pcu.deduplicate_mesh_vertices, (p, f.astype(np.float64), 0.1), {}, "Invalid scalar type (float64) for argument 'f'"),
        (pcu.deduplicate_mesh_vertices, (p, f.ravel(), 0.1), {}, "Invalid shape for faces"),
        (pcu.deduplicate_mesh_vertices, (p, None, 0.1), {}, "f must be an (m, 3) array"),
        (pcu.deduplicate_mesh_vertices, (t, f, 0.1), {}, "Invalid type for v"),
        (pcu.deduplicate_mesh_vertices, (t, torch.from_numpy(f).double(), 0.1), {}, "Invalid scalar type (float64) for argument 'f'"),
        # Poisson disk
        (pcu.downsample_point_cloud_poisson_disk, (p, 0.0), {}, "Cannot have both num_samples <= 0 and radius <= 0"),
        (pcu.downsample_point_cloud_poisson_disk, (p, 0.1), {"sample_num_tolerance": 0.0}, "sample_num_tolerance must be in (0, 1]"),
        (pcu.downsample_point_cloud_poisson_disk, (p.astype(np.int32), 0.1), {}, "Invalid scalar type (int32) for argument 'v'"),
        (pcu.downsample_point_cloud_poisson_disk, (t.int(), 0.1), {}, "for argument 'v'"),
        (pcu.downsample_point_cloud_poisson_disk, (p[:, :2], 0.1), {}, "Invalid shape for v"),
        (pcu.downsample_point_cloud_poisson_disk, (t[:, :2], 0.1), {}, "Invalid shape for v"),
        (pcu.downsample_point_cloud_poisson_disk, (p.tolist(), 0.1), {}, "Invalid type for v, must be a NumPy array"),
        # voxel grid
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, p.tolist()), {}, "points must be a numpy array but got type"),
        (pcu.downsample_point_cloud_on_voxel_grid, ((0.1, 0.1), p), {}, "3-tuple"),
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, p, p[:10]), {}, "first dimension"),
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, p), {"min_bound": (0, 0, 0), "max_bound": (1, 0, 1)}, "max_bound must be greater"),
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, p.astype(np.int32)), {}, "Invalid scalar type (int32) for argument 'v'"),
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, p, p.astype(np.int32)), {}, "Invalid scalar type (int32) for argument 'attrib'"),
        (pcu.downsample_point_cloud_on_voxel_grid, (0.1, t, t.int()), {}, "Invalid scalar type (int32) for argument 'attrib'"),
        (pcu._voxel_internal, (p, p[:10], [0.1] * 3, [0] * 3, [1] * 3, 1, None), {}, "Invalid number of attributes (10)"),
        # normals
        (pcu.estimate_point_cloud_normals_knn, (p[:, :2], 5), {}, "Invalid shape for points"),
        (pcu.estimate_point_cloud_normals_knn, (p.tolist(), 5), {}, "Invalid type for points"),
        (pcu.estimate_point_cloud_normals_knn, (t.half(), 5), {}, "Invalid scalar type (float16) for argument 'points'"),
        (pcu.estimate_point_cloud_normals_knn, (t[:, :2], 5), {}, "Invalid shape for points"),
        (pcu.estimate_point_cloud_normals_knn, (t[:0], 5), {}, "Invalid point set with zero elements"),
        (pcu.estimate_point_cloud_normals_knn, (t, 0), {}, "Invalid number of neighbors (0)"),
        (pcu.estimate_point_cloud_normals_knn, (t, 5), {"view_directions": t[:10]}, "Invalid view directions"),
        (pcu.estimate_point_cloud_normals_ball, (p[:, :2], 0.1), {}, "Invalid shape for points"),
        (pcu.estimate_point_cloud_normals_ball, (t.half(), 0.1), {}, "Invalid scalar type (float16) for argument 'points'"),
        (pcu.estimate_point_cloud_normals_ball, (t, 0.1), {"view_directions": p}, "Invalid type for points, must be a NumPy array"),
        (pcu.estimate_point_cloud_normals_ball, (p, 0.1), {"view_directions": p.tolist()}, "Invalid type for view_directions"),
        # nearest neighbours: numpy arrays and tensors do not mix (the rest is in _nn_cases)
        (pcu.k_nearest_neighbors, (p, t, 1), {}, "Invalid type for dataset_points, must be a NumPy array"),
        (pcu.chamfer_distance, (t, p), {}, "Invalid type for x, must be a NumPy array"),
        (pcu.one_sided_hausdorff_distance, (t, p), {}, "Invalid type for source, must be a NumPy array"),
        (pcu.batched_chamfer_distance, (torch.zeros((2, 5, 3)), np.zeros((2, 5, 3), np.float32)), {}, "Invalid type for x"),
        # Voronoi centroids
        (pcu.voronoi_centroids_unit_cube, (p.astype(np.int32),), {}, "Invalid scalar type (int32) for argument 'centers'"),
        (pcu.voronoi_centroids_unit_cube, (p[:, :2],), {}, "Invalid shape for centers"),
        (pcu.voronoi_centroids_unit_cube, (p.tolist(),), {}, "Invalid type for centers"),
        (pcu.voronoi_centroids_unit_cube, (p + 1.0,), {}, "Centers of voronoi diagram must lie in the unit cube [0, 1]^3"),
        (pcu.voronoi_centroids_unit_cube, (t + 1.0,), {}, "Centers of voronoi diagram must lie in the unit cube [0, 1]^3"),
    ]


def _fake_cloud(pcu, handle, device_index=0):
    """A PreparedCloud of 40 float64 points on cuda:device_index that holds no device memory (handle 0: closed)."""
    class Fake(pcu.PreparedCloud):
        def close(self):
            self._handle = 0
    return Fake(handle, 40, True, device_index, False)


def _nn_cases(pcu, make):
    """Argument errors of the nearest-neighbour family, with the arrays made by `make` from numpy arrays, and the message
    each raises: the reference's checks in its order (k, dtypes, shapes), then a prepared cloud's."""
    rng = np.random.default_rng(1)
    a, b = rng.random((50, 3)), rng.random((40, 3))
    cloud, closed = _fake_cloud(pcu, 1), _fake_cloud(pcu, 0)
    ab = "query_points and dataset_points must have shape (n, 3) and (m, 3). Got query_points.shape = "
    f32 = "Invalid scalar type (float64) for argument 'dataset_points'. Expected it to match argument 'query_points' which is of type float32."
    batch = rng.random((2, 5, 3)).astype(np.float32)
    cases = [
        (pcu.k_nearest_neighbors, (a, b, 0), {}, "Invalid value for k (0) must be greater than 0."),
        (pcu.k_nearest_neighbors, (a, cloud, -1), {}, "Invalid value for k (-1) must be greater than 0."),
        (pcu.k_nearest_neighbors, (a.astype(np.int64), b, 1), {},
         "Invalid scalar type (int64) for argument 'query_points'. Expected one of ['float32', 'float64']."),
        (pcu.k_nearest_neighbors, (a.astype(np.float32), b, 1), {}, f32),
        (pcu.k_nearest_neighbors, (a.astype(np.float32), cloud, 1), {}, f32),
        (pcu.k_nearest_neighbors, (a[:, :2], b, 1), {}, "Only 3D inputs are supported: " + ab + "(50, 2), dataset_points.shape = (40, 3)."),
        (pcu.k_nearest_neighbors, (a[:, :2], cloud, 1), {}, "Only 3D inputs are supported: " + ab + "(50, 2), dataset_points.shape = (40, 3)."),
        (pcu.k_nearest_neighbors, (a[0], b, 1), {}, "Only 3D inputs are supported: " + ab + "(3), dataset_points.shape = (40, 3)."),
        (pcu.k_nearest_neighbors, (a, b[:0], 1), {}, "Invalid input set with zero elements: " + ab + "(50, 3), dataset_points.shape = (0, 3)."),
        (pcu.k_nearest_neighbors, (a[:0, :2], cloud, 1), {}, "Invalid input set with zero elements: " + ab + "(0, 2), dataset_points.shape = (40, 3)."),
        (pcu.k_nearest_neighbors, (a, closed, 1), {}, "the PreparedCloud has been closed"),
        (pcu.k_nearest_neighbors, (a, cloud, 1), {"device": 1}, "device=1 contradicts the prepared cloud, which lives on cuda:0"),
        (pcu.k_nearest_neighbors, (a, b, 1), {"device": "cuda:99"}, "out of range"),
        (pcu.one_sided_hausdorff_distance, (a, b[:, :1]), {}, "Only 3D inputs are supported: source and target must have shape"),
        (pcu.one_sided_hausdorff_distance, (a[:0], cloud), {}, "Invalid input set with zero elements: source and target must"),
        (pcu.one_sided_hausdorff_distance, (a, closed), {}, "the PreparedCloud has been closed"),
        (pcu.one_sided_hausdorff_distance, (a, cloud), {"device": "cuda:1"}, "device='cuda:1' contradicts the prepared cloud"),
        (pcu.hausdorff_distance, (a, b.astype(np.float32)), {}, "Invalid scalar type (float32) for argument 'y'. Expected it to match"),
        (pcu.hausdorff_distance, (a.astype(np.float32), cloud), {}, "Invalid scalar type (float64) for argument 'y'. Expected it to match"),
        (pcu.chamfer_distance, (a.astype(np.float16), b), {}, "Invalid scalar type (float16) for argument 'x'"),
        (pcu.chamfer_distance, (a, closed), {}, "the PreparedCloud has been closed"),
        (pcu.chamfer_distance, (a, cloud), {"device": 1}, "device=1 contradicts the prepared cloud"),
        (pcu.chamfer_distance, (a, b[:, :2]), {"p_norm": 1}, "Only 3D inputs are supported: query_points and dataset_points"),
        (pcu.chamfer_distance, (a, cloud), {"return_index": True}, "a PreparedCloud serves the fused metrics"),
        (pcu.prepare_cloud, (a.astype(np.int32),), {}, "Invalid scalar type (int32) for argument 'points'"),
        (pcu.prepare_cloud, (a[:0],), {}, "Invalid input set with zero elements: points must have shape (n, 3). Got points.shape = (0, 3)."),
        (pcu.prepare_cloud, (a[:, :2],), {}, "Only 3D inputs are supported: points must have shape (n, 3). Got points.shape = (50, 2)."),
        (pcu.prepare_cloud, (a,), {"k": 0}, "Invalid value for k (0) must be greater than 0."),
        (pcu.batched_chamfer_distance, (batch, batch.astype(np.float64)), {}, "batched_chamfer_distance: x and y must both be float32"),
        (pcu.batched_chamfer_distance, (batch, batch[:1]), {}, "must have shape (B, n, 3) and (B, m, 3)"),
        (pcu.batched_chamfer_distance, (batch, batch[:, :0]), {}, "Invalid input set with zero elements"),
        (pcu.estimate_point_cloud_normals_knn, (a.astype(np.int64), 5), {}, "Invalid scalar type (int64) for argument 'points'"),
        (pcu.estimate_point_cloud_normals_knn, (a[:0], 5), {},
         "Invalid point set with zero elements: points must have shape (n, 3), but got points.shape = (0, 3)."),
        (pcu.estimate_point_cloud_normals_knn, (a, 5), {"view_directions": a.astype(np.float32)},
         "Invalid scalar type (float32) for argument 'view_dirs'. Expected it to match argument 'points' which is of type float64."),
        (pcu.estimate_point_cloud_normals_knn, (a, 5), {"view_directions": a[:10]},
         "Invalid view directions does not match the number of points. If view directions are passed in, they must have the "
         "same shape as points. Got points.shape = (50, 3), and view_dirs.shape = (10, 3)."),
        (pcu.estimate_point_cloud_normals_ball, (a, 0.1), {"view_directions": a[:, 0]}, "Invalid shape for view_directions"),
    ]
    return [(fn, tuple(make(x) if isinstance(x, np.ndarray) else x for x in args),
             {k: make(v) if isinstance(v, np.ndarray) else v for k, v in kwargs.items()}, msg) for fn, args, kwargs, msg in cases]


def _raises(fn, args, kwargs, msg):
    with pytest.raises(ValueError) as e:
        fn(*args, **kwargs)
    assert msg in str(e.value), (fn.__name__, msg, str(e.value))
    return str(e.value)


def test_nearest_neighbour_errors_come_before_any_device_call(no_device, monkeypatch):
    """numpy arrays and CPU tensors: every argument error before any device call, and one message for one mistake."""
    import torch
    monkeypatch.setattr(no_device._pcu_internal, "_device_count", lambda: 2)   # device=1 names a device, not a range error
    numpy = [_raises(*case) for case in _nn_cases(no_device, lambda a: a)]
    cpu = [_raises(*case) for case in _nn_cases(no_device, torch.from_numpy)]
    assert cpu == numpy


@pytest.mark.gpu
def test_nearest_neighbour_errors_on_cuda_tensors(no_device, monkeypatch):
    """CUDA tensors: the same messages, before any device call; and a prepared cloud on another device."""
    import torch
    monkeypatch.setattr(no_device._pcu_internal, "_device_count", lambda: 2)
    numpy = [_raises(*case) for case in _nn_cases(no_device, lambda a: a)]
    cuda = [_raises(*case) for case in _nn_cases(no_device, lambda a: torch.from_numpy(a).cuda())]
    assert cuda == numpy
    x = torch.zeros((5, 3), dtype=torch.float64, device="cuda")
    _raises(no_device.chamfer_distance, (x, _fake_cloud(no_device, 1, device_index=1)), {},
            "x lives on cuda:0, the prepared cloud on cuda:1")


def test_argument_errors_come_before_any_device_call(no_device):
    import torch
    for fn, args, kwargs, msg in _cases(no_device, torch):
        with pytest.raises(ValueError) as e:
            fn(*args, **kwargs)
        assert msg in str(e.value), (fn.__name__, msg, str(e.value))


def test_empty_inputs_need_no_device(no_device):
    import torch
    pcu = no_device
    for make in (lambda a: a, torch.from_numpy):
        e = make(np.zeros((0, 3)))
        x, svi, svj = pcu.deduplicate_point_cloud(e, 0.1, device="cuda:99")
        v, f, _, _ = pcu.deduplicate_mesh_vertices(e, make(np.zeros((0, 3), dtype=np.int64)), 0.1)
        idx = pcu.downsample_point_cloud_poisson_disk(e, 0.1)
        few = pcu.downsample_point_cloud_poisson_disk(make(np.ones((4, 3))), 0.0, target_num_samples=9)
        c = pcu.voronoi_centroids_unit_cube(e)
        for o, dtype, shape in ((x, "float64", (0, 3)), (svi, "int32", (0,)), (svj, "int32", (0,)), (v, "float64", (0, 3)),
                                (f, "int64", (0, 3)), (idx, "int32", (0,)), (few, "int32", (4,)), (c, "float64", (0, 3))):
            assert type(o) is type(e) and str(o.dtype).endswith(dtype) and tuple(o.shape) == shape
        assert np.array_equal(np.asarray(few), np.arange(4))


# ---- GPU: one result in every form ---------------------------------------------------------------------------------
def _bits(x):
    import torch
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    return a.dtype, a.shape, np.ascontiguousarray(a).tobytes()


def _in_forms(call, arrays, seed=None, exact=True):
    """call(*arrays) with numpy arrays, CUDA tensors and CPU tensors (NumPy's global state seeded to `seed` before each,
    when given); every result must come back in its inputs' form and be bit-identical across the three.  exact=False:
    floating-point values may differ in the last bits (sums whose order the device does not fix)."""
    import torch
    ref = None
    for form in ("numpy", "cuda", "cpu"):
        ins = [a if form == "numpy" else torch.from_numpy(a).to("cuda" if form == "cuda" else "cpu") for a in arrays]
        if seed is not None:
            np.random.seed(seed)
        out = call(*ins)
        out = out if isinstance(out, tuple) else (out,)
        for o in out:
            if form == "numpy":
                assert isinstance(o, (np.ndarray, np.generic)), (form, type(o))
            else:
                assert isinstance(o, torch.Tensor) and o.is_cuda == (form == "cuda"), (form, type(o))
                assert form == "cpu" or o.device == ins[0].device
        got = [_bits(o) for o in out]
        if ref is None:
            ref, values = got, [np.asarray(o.detach().cpu().numpy() if isinstance(o, torch.Tensor) else o) for o in out]
        elif exact:
            assert got == ref, form
        else:
            assert [g[:2] for g in got] == [r[:2] for r in ref], form
            for o, v in zip(out, values):
                o = o.detach().cpu().numpy() if isinstance(o, torch.Tensor) else o
                assert np.allclose(o, v, rtol=4 * np.finfo(v.dtype).eps, atol=0) if v.dtype.kind == "f" else np.array_equal(o, v)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_every_function_in_every_form(pcu, dtype):
    rng = np.random.default_rng(5)
    a = rng.random((300, 3)).astype(dtype)
    b = rng.random((200, 3)).astype(dtype)
    _in_forms(pcu.pairwise_distances, [a, b])
    _in_forms(lambda x, y: pcu.pairwise_distances(x, y, p=1), [a.reshape(3, 100, 3), b[:150].reshape(3, 50, 3)])
    M = np.asarray(pcu.pairwise_distances(a[:60], b[:40]))
    _in_forms(lambda u, v, m: pcu.sinkhorn(u, v, m, 1e-2), [np.ones(60, dtype) / 60, np.ones(40, dtype) / 40, M])
    if dtype == np.float64:
        _in_forms(lambda x, y: pcu.earth_movers_distance(x, y, eps=1e-2), [a[:80], b[:70]], exact=False)   # the cost: a device sum
    dup = np.concatenate([a, a[:100] + dtype(1e-4), a[::7]])
    _in_forms(lambda x: pcu.deduplicate_point_cloud(x, 1e-3), [dup])
    f = rng.integers(0, len(dup), (400, 3)).astype(np.int32)
    _in_forms(lambda v, g: pcu.deduplicate_mesh_vertices(v, g, 1e-3), [dup, f])
    _in_forms(lambda v, g: pcu.deduplicate_mesh_vertices(v, g, 1e-3), [dup, f.astype(np.int64)])
    cloud = rng.random((5000, 3)).astype(dtype)
    _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.05, random_seed=3), [cloud])
    _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.0, target_num_samples=700, random_seed=3), [cloud])
    _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.05), [cloud], seed=11)
    _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.05, target_num_samples=5000), [cloud])
    _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.05), [cloud[:0]])
    colors = rng.random((5000, 3)).astype(np.float32)
    scalar = rng.random(5000)
    # voxel means are fp64 sums in the order the device's atomics take: rows, counts and dtypes exact, means to rounding
    _in_forms(lambda x, c, s: pcu.downsample_point_cloud_on_voxel_grid(0.07, x, c, s, min_points_per_voxel=2),
              [cloud, colors, scalar], exact=False)
    _in_forms(lambda x: pcu.downsample_point_cloud_on_voxel_grid((0.05, 0.1, 0.2), x), [cloud], exact=False)
    view = np.tile(np.array([[0.0, 0.0, 1.0]], dtype), (5000, 1))
    _in_forms(lambda x: pcu.estimate_point_cloud_normals_knn(x, 12), [cloud])
    _in_forms(lambda x, d: pcu.estimate_point_cloud_normals_knn(x, 12, d), [cloud, view])
    _in_forms(lambda x: pcu.estimate_point_cloud_normals_ball(x, 0.01, max_pts_per_ball=8), [cloud], seed=4)
    _in_forms(lambda x, d: pcu.estimate_point_cloud_normals_ball(x, 0.01, d), [cloud, view], seed=4)
    _in_forms(pcu.voronoi_centroids_unit_cube, [a])
    _in_forms(pcu.voronoi_centroids_unit_cube, [a[:0]])


@pytest.mark.gpu
def test_poisson_target_box_of_non_finite_clouds(pcu, monkeypatch):
    """The target search's bounding box, taken on the device for every form, is numpy's min and max: the same box size
    with +-inf and NaN coordinates, and the same error when the radius it gives is NaN."""
    from pcu_b200 import _poisson
    rng = np.random.default_rng(6)
    clouds = []
    for fill in ([(0, 0, np.inf), (1, 1, -np.inf)], [(0, 2, np.nan)], [(slice(None), 1, np.inf)], [(3, 0, -np.inf), (4, 1, np.nan)]):
        c = rng.random((64, 3))
        for i, j, x in fill:
            c[i, j] = x
        clouds.append(c)
    boxes = []
    monkeypatch.setattr(_poisson, "target_search", lambda sample, T, bbsize, target, tol: boxes.append(bbsize) or 0)
    for dtype in (np.float32, np.float64):
        for c in clouds:
            boxes.clear()
            _in_forms(lambda x: pcu.downsample_point_cloud_poisson_disk(x, 0.0, target_num_samples=10, random_seed=1),
                      [c.astype(dtype)])
            assert len(boxes) == 3 and len({np.asarray(x).tobytes() for x in boxes}) == 1, boxes
            assert not np.isfinite(boxes[0])
    monkeypatch.undo()
    import torch
    nan_cloud = clouds[3]
    for x in (nan_cloud, torch.from_numpy(nan_cloud).cuda(), torch.from_numpy(nan_cloud)):
        with pytest.raises(ValueError, match="Invalid radius"):
            pcu.downsample_point_cloud_poisson_disk(x, 0.0, target_num_samples=10, random_seed=1)


@pytest.mark.gpu
def test_device_keyword(pcu, monkeypatch):
    import torch
    from pcu_b200 import _pcu_internal
    rng = np.random.default_rng(7)
    pts = np.concatenate([rng.random((500, 3))] * 2)
    ref = pcu.deduplicate_point_cloud(pts, 1e-3)
    for device in (0, "cuda", "cuda:0", torch.device("cuda"), torch.device("cuda", 0)):
        got = pcu.deduplicate_point_cloud(pts, 1e-3, device=device)
        assert all(np.array_equal(g, r) for g, r in zip(got, ref)), device
    # a second GPU as far as device= can tell: CUDA tensors on cuda:0 contradict device=1
    monkeypatch.setattr(_pcu_internal, "_device_count", lambda: 2)
    x = torch.from_numpy(pts).cuda()
    w = torch.ones(4, dtype=torch.float64, device="cuda") / 4
    M = torch.rand((4, 4), dtype=torch.float64, device="cuda")
    for call in (lambda: pcu.pairwise_distances(x, x, device=1), lambda: pcu.sinkhorn(w, w, M, 1e-2, device=1),
                 lambda: pcu.earth_movers_distance(x[:50], x[:40], device=1),
                 lambda: pcu.downsample_point_cloud_on_voxel_grid(0.1, x, x, device=1),
                 lambda: pcu.deduplicate_point_cloud(x, 1e-3, device=1),
                 lambda: pcu.deduplicate_mesh_vertices(x, torch.zeros((1, 3), dtype=torch.int64, device="cuda"), 1e-3,
                                                       device="cuda:1")):
        with pytest.raises(ValueError, match="contradicts the inputs, which live on cuda:0"):
            call()
