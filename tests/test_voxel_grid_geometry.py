"""voxel_grid_geometry: a numpy restatement pinned to a loop-by-loop transcription of the reference's
generate_cube_mesh (src/mesh_for_voxels.cpp, fp64 with a float32 cast); argument errors in the reference's order; on
the GPU, bit-for-bit equality in every form and index dtype, and the half-voxel offset against voxelize_triangle_mesh
that the reference's own documented pairing produces."""
import numpy as np
import pytest

from meshes import to_form, to_numpy

# the reference's tables (src/mesh_for_voxels.cpp)
FACES = np.array([2, 7, 6, 2, 3, 7, 0, 4, 5, 0, 5, 1, 0, 2, 6, 0, 6, 4, 1, 7, 3, 1, 5, 7, 0, 3, 2, 0, 1, 3, 4, 6, 7, 4, 7, 5],
                 np.int32).reshape(12, 3)
CORNERS = np.array([0, 0, 1, 1, 0, 1, 0, 1, 1, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 1, 1, 0], np.float32).reshape(8, 3)


def transcription(ijk, size, origin, gap):
    """generate_cube_mesh, loop by loop, on Python floats (IEEE fp64, no FMA)."""
    v = np.empty((8 * len(ijk), 3), np.float32)
    f = np.empty((12 * len(ijk), 3), np.int32)
    for i, row in enumerate(ijk.tolist()):
        for vi in range(8):
            vert = [float(CORNERS[vi, k]) * (1.0 - gap) + 0.5 * gap for k in range(3)]
            vert = [vert[k] + float(row[k]) for k in range(3)]
            vert = [vert[k] * size[k] for k in range(3)]
            vert = [vert[k] + origin[k] for k in range(3)]
            v[8 * i + vi] = np.array(vert, np.float64).astype(np.float32)
        for fi in range(12):
            f[12 * i + fi] = FACES[fi] + 8 * i
    return v, f


def restate(ijk, size, origin, gap):
    base = CORNERS.astype(np.float64) * (1.0 - gap) + 0.5 * gap                       # (8, 3)
    x = (base[None, :, :] + ijk.astype(np.float64)[:, None, :]) * np.asarray(size, np.float64) + np.asarray(origin, np.float64)
    f = FACES[None, :, :] + 8 * np.arange(len(ijk), dtype=np.int32)[:, None, None]
    return x.reshape(-1, 3).astype(np.float32), f.reshape(-1, 3)


def cases():
    rng = np.random.default_rng(0)
    yield rng.integers(-50, 50, (40, 3)).astype(np.int32), (1.0, 1.0, 1.0), (0.0, 0.0, 0.0), 0.0
    yield rng.integers(-2 ** 31, 2 ** 31 - 1, (30, 3)).astype(np.int64), (0.1, 0.25, 3.0), (1.5, -2.0, 1e-3), 0.1
    yield rng.integers(0, 2 ** 64 - 1, (30, 3), dtype=np.uint64), (0.37, 0.37, 0.37), (0.0, 5.0, -5.0), 0.5
    yield rng.integers(0, 2 ** 32 - 1, (30, 3), dtype=np.uint64).astype(np.uint32), (2.0, 1.0, 0.5), (0.0, 0.0, 0.0), 0.9
    yield np.array([[2 ** 53 + 1, -(2 ** 62), 7]], np.int64), (0.3, 0.3, 0.3), (0.1, 0.2, 0.3), 0.25
    yield rng.integers(-1000, 1000, (25, 3)).astype(np.int64), (0.013, 0.017, 0.019), (10.0, -3.0, 7.5), 1.5


def test_restatement_is_the_transcription():
    for ijk, size, origin, gap in cases():
        v, f = restate(ijk, size, origin, gap)
        tv, tf = transcription(ijk, size, origin, gap)
        assert np.array_equal(v, tv) and np.array_equal(f, tf)
        assert v.dtype == np.float32 and f.dtype == np.int32


def test_argument_errors():
    import pcu_b200 as pcu
    ijk = np.zeros((4, 3), np.int32)
    with pytest.raises(ValueError, match="expected 3D coordinate"):
        pcu.voxel_grid_geometry(ijk.astype(np.float64), 1.0, (0.0, 0.0))            # the wrapper's arguments first
    with pytest.raises(ValueError, match="expected 3D coordinate"):
        pcu.voxel_grid_geometry(ijk, (1.0, 1.0))
    with pytest.raises(ValueError, match=r"Invalid scalar type \(float64\) for argument 'ijk'"):
        pcu.voxel_grid_geometry(ijk.astype(np.float64))
    with pytest.raises(ValueError, match=r"Invalid input point cloud with zero points: points must have shape \(n, 3\) "
                                         r"\(n > 0\)\. Got points.shape =\(0, 3\)\."):
        pcu.voxel_grid_geometry(ijk[:0], -1.0)
    with pytest.raises(ValueError, match=r"Only 3D inputs are supported: v must have shape \(n, 3\) \(n > 0\)\. "
                                         r"Got points.shape =\(4, 2\)\."):
        pcu.voxel_grid_geometry(ijk[:, :2], -1.0)
    for size in (0.0, -1.0, (1.0, 0.0, 1.0)):
        with pytest.raises(ValueError, match="Voxel size must be positive"):
            pcu.voxel_grid_geometry(ijk, size)
    import inspect
    sig = inspect.signature(pcu.voxel_grid_geometry)
    assert list(sig.parameters) == ["ijk", "voxel_size", "voxel_origin", "gap_fraction", "device"]
    assert sig.parameters["gap_fraction"].default == 0.0
    assert np.array_equal(sig.parameters["voxel_size"].default, [1.0, 1.0, 1.0])


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["numpy", "cuda", "cpu"])
def test_equals_restatement(form):
    import pcu_b200 as pcu
    rng = np.random.default_rng(1)
    all_cases = list(cases()) + [(rng.integers(-300, 300, (10 ** 6, 3)).astype(np.int32), (0.01, 0.02, 0.03), (1.0, 2.0, 3.0), 0.05)]
    for ijk, size, origin, gap in all_cases:
        v, f = pcu.voxel_grid_geometry(to_form(form, ijk), size, origin, gap)
        wv, wf = restate(ijk, size, origin, gap)
        v, f = to_numpy(v, form), to_numpy(f, form)
        assert v.dtype == np.float32 and f.dtype == np.int32
        assert np.array_equal(v, wv) and np.array_equal(f, wf)
    v, f = pcu.voxel_grid_geometry(to_form(form, np.array([[1, 2, 3]], np.int64)), 2.0)
    assert to_numpy(v, form).shape == (8, 3) and to_numpy(f, form).shape == (12, 3)
    v, _ = pcu.voxel_grid_geometry(to_form(form, np.array([[0, 0, 0]], np.int32)), float("nan"))   # NaN passes, as there
    assert np.isnan(to_numpy(v, form)).all()


@pytest.mark.gpu
def test_pairing_with_voxelize_is_half_a_voxel_off():
    """The reference's documented example: voxelize_triangle_mesh centres voxel (i, j, k) at o + (i, j, k) s;
    voxel_grid_geometry with the same origin puts that voxel's LOW corner there, so each cube sits half a voxel off."""
    import pcu_b200 as pcu
    v = np.array([[0.1, 0.2, 0.3], [1.7, 0.4, 0.2], [0.5, 1.9, 1.1]])
    f = np.array([[0, 1, 2]], np.int32)
    s, o = 0.25, np.array([0.0, 0.0, 0.0])
    ijk = pcu.voxelize_triangle_mesh(v, f, s, o)
    cv, _ = pcu.voxel_grid_geometry(ijk, s, o)
    cv = cv.reshape(-1, 8, 3).astype(np.float64)
    centres = o + ijk * s
    assert np.allclose(cv.min(1), centres, atol=1e-6)                # the box's low corner at the voxel's centre
    assert np.allclose(cv.mean(1), centres + 0.5 * s, atol=1e-6)     # offset by half a voxel on every axis
