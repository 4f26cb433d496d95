"""adjacency_list: the result of DESIGN.md §3 restated with numpy (one unique over the directed face edges) and pinned
to a literal transcription of libigl's adjacency_list (push_back both ways, then sort and unique) on random small
meshes with repeated corners, duplicate faces and unreferenced indices; the argument errors and the signature; on the
GPU, both return forms equal to the restatement over every dtype and input form, the bunny, a 1.31 * 10^6-face
icosphere, a 10^5-face fan, all-degenerate faces, a max(f) far above the referenced vertices, rejected indices, and
an input left as it was."""
import inspect
import os

import numpy as np
import pytest

from meshes import icosphere, to_form, to_numpy

IDX = [np.int32, np.int64]
FORMS = ["numpy", "cuda", "cpu"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- the restatement ------------------------------------------------------------------------------------------------
def restate(f):
    """(offsets (n + 1,), neighbors (offsets[-1],)) in f's dtype, n = max(f) + 1: the distinct directed pairs of the
    face edges a->b, b->c, c->a and their reverses, in ascending (row, column) order."""
    a = np.asarray(f)
    e = a.reshape(-1, 3).astype(np.int64)
    n = int(e.max()) + 1
    src, dst = e.ravel(), e[:, [1, 2, 0]].ravel()
    key = np.unique(np.concatenate([src * n + dst, dst * n + src]))
    rows, cols = key // n, key % n
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(rows, minlength=n))
    return offsets.astype(a.dtype), cols.astype(a.dtype)


def as_lists(offsets, neighbors):
    o, nb = np.asarray(offsets).tolist(), np.asarray(neighbors).tolist()
    return [nb[o[i]:o[i + 1]] for i in range(len(o) - 1)]


def literal(f):
    """libigl's adjacency_list(F, A, sorted=false): A.resize(F.maxCoeff() + 1); for every face and corner j,
    s = F(i, j), d = F(i, (j + 1) % 3), A[s].push_back(d), A[d].push_back(s); then every list sorted and made unique."""
    F = [[int(x) for x in row] for row in np.asarray(f).reshape(-1, 3)]
    A = [[] for _ in range(max(max(row) for row in F) + 1)]
    for row in F:
        for j in range(3):
            s, d = row[j], row[(j + 1) % 3]
            A[s].append(d)
            A[d].append(s)
    out = []
    for lst in A:
        lst = sorted(lst)
        out.append([x for k, x in enumerate(lst) if k == 0 or x != lst[k - 1]])
    return out


def random_faces(rng, m, hi, dtype):
    """Random faces over [0, hi) with repeated corners, duplicated (and reversed) faces and indices no face names."""
    f = rng.integers(0, hi, (m, 3))
    k = max(1, m // 8)
    f[rng.integers(0, m, k), 1] = f[rng.integers(0, m, k), 0]             # (a, a, b)
    f[rng.integers(0, m, k)] = f[rng.integers(0, m, k)]                    # duplicate faces
    f[rng.integers(0, m, k)] = f[rng.integers(0, m, k)][:, ::-1]           # reversed duplicates
    f[rng.integers(0, m, 1)] = f[rng.integers(0, m, 1), :1]                # (a, a, a)
    f[f % 5 == 3] += 1                                                     # leaves holes in the numbering
    return f.astype(dtype)


@pytest.mark.parametrize("seed", range(12))
def test_restatement_equals_literal(seed):
    rng = np.random.default_rng(seed)
    for m, hi in [(1, 3), (2, 5), (7, 6), (40, 30), (200, 90)]:
        f = random_faces(rng, m, hi, IDX[seed % 2])
        o, nb = restate(f)
        assert o.dtype == f.dtype and nb.dtype == f.dtype and o.shape == (int(f.max()) + 2,)
        assert as_lists(o, nb) == literal(f)


def test_restatement_cases():
    f = np.array([[0, 1, 2], [2, 2, 4]], np.int32)
    assert literal(f) == [[1, 2], [0, 2], [0, 1, 2, 4], [], [2]]
    assert as_lists(*restate(f)) == literal(f)
    assert as_lists(*restate(np.array([[3, 3, 3]], np.int64))) == [[], [], [], [3]]


# ---- CPU: interface and argument errors ---------------------------------------------------------------------------
def test_signature(pcu):
    ps = list(inspect.signature(pcu.adjacency_list).parameters.values())
    assert [p.name for p in ps] == ["f", "return_csr", "device"]
    assert ps[0].kind == inspect.Parameter.POSITIONAL_OR_KEYWORD
    assert ps[1].kind == inspect.Parameter.KEYWORD_ONLY and ps[1].default is False
    assert ps[2].kind == inspect.Parameter.KEYWORD_ONLY and ps[2].default is None
    assert "adjacency_list" in pcu.__all__


def test_argument_errors(pcu):
    f = np.array([[0, 1, 2], [2, 3, 0]], np.int32)
    cases = [
        (f.astype(np.float32), "Invalid scalar type (float32) for argument 'f'. Expected one of ['int32', 'int64']."),
        (f.astype(np.uint32), "Invalid scalar type (uint32) for argument 'f'"),
        (f[:0].astype(np.float64), "Invalid scalar type (float64) for argument 'f'"),       # the dtype first
        (f[:0], "Invalid input faces with zero elements: f must have shape (n, 3) where n > 0. Got f.shape =(0, 3)."),
        (np.zeros((2, 4), np.int64), "Only triangle inputs are supported: f must have shape (n, 3) where n > 0. Got f.shape =(2, 4)."),
        (np.zeros((0, 4), np.int64), "Invalid input faces with zero elements"),               # rows before columns
        (np.arange(3, dtype=np.int32), "Only triangle inputs are supported"),                 # a 1-D f is one column
        (np.zeros((1, 3, 1), np.int32), "f must be a 1-D or 2-D array"),
        (f.tolist(), "Invalid type for f"),
        (np.broadcast_to(np.zeros((1, 3), np.int32), (357913942, 3)), "at most 357913941 faces are supported"),
    ]
    for arg, msg in cases:
        with pytest.raises(ValueError) as e:
            pcu.adjacency_list(arg)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(TypeError):
        pcu.adjacency_list(f, True)                          # return_csr is keyword only


# ---- GPU ------------------------------------------------------------------------------------------------------------
def check(pcu, f, form="numpy"):
    """Both return forms of adjacency_list(f) against the restatement; returns the CSR."""
    import torch
    want = restate(f)
    ft = to_form(form, f)
    got = pcu.adjacency_list(ft, return_csr=True)
    assert isinstance(got, tuple) and len(got) == 2
    for g, w in zip(got, want):
        if form == "numpy":
            assert isinstance(g, np.ndarray)
        else:
            assert isinstance(g, torch.Tensor) and g.is_cuda == (form == "cuda")
        g = to_numpy(g)
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g, w)
    lists = pcu.adjacency_list(ft)
    assert isinstance(lists, list) and lists == as_lists(*want)
    assert all(type(x) is int for lst in lists[:50] for x in lst)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("idt", IDX)
def test_forms_and_dtypes(pcu, form, idt):
    rng = np.random.default_rng(3)
    for m, hi in [(1, 3), (5, 4), (300, 120), (5000, 1500)]:
        f = random_faces(rng, m, hi, idt)
        check(pcu, f, form)
        if m <= 300:
            assert pcu.adjacency_list(to_form(form, f)) == literal(f)


@pytest.mark.gpu
def test_bunny(pcu):
    f = np.load(os.path.join(GOLDEN, "bunny_faces.npy"))
    o, nb = check(pcu, f)
    check(pcu, f.astype(np.int64), "cuda")
    assert len(o) == f.max() + 2 and np.all(np.diff(o) >= 3)


@pytest.mark.gpu
def test_icosphere_level_8(pcu):
    import torch
    _, f = icosphere(8)
    assert len(f) == 1310720
    ft = torch.from_numpy(f).cuda()
    o, nb = pcu.adjacency_list(ft, return_csr=True)
    wo, wnb = restate(f)
    assert torch.equal(o.cpu(), torch.from_numpy(wo)) and torch.equal(nb.cpu(), torch.from_numpy(wnb))
    deg = np.diff(wo)
    assert deg.min() == 5 and deg.max() == 6 and (deg == 5).sum() == 12     # a closed icosphere: 12 valence-5 vertices
    lists = pcu.adjacency_list(ft)
    assert len(lists) == len(wo) - 1 and lists[0] == wnb[wo[0]:wo[1]].tolist() and lists[-1] == wnb[wo[-2]:].tolist()


@pytest.mark.gpu
def test_fan(pcu):
    k = 100000
    i = np.arange(k, dtype=np.int64)
    f = np.stack([np.zeros(k, np.int64), i + 1, i + 2], 1)
    o, nb = check(pcu, f, "cuda")
    assert o[1] - o[0] == k + 1 and np.array_equal(nb[:k + 1], np.arange(1, k + 2))


@pytest.mark.gpu
def test_degenerate_faces(pcu):
    f = np.array([[2, 2, 2], [5, 5, 5], [2, 2, 2]], np.int32)
    o, nb = check(pcu, f)
    assert pcu.adjacency_list(f) == [[], [], [2], [], [], [5]]


@pytest.mark.gpu
def test_max_index_far_above_the_mesh(pcu):
    f = np.array([[0, 1, 2], [1, 2, 3], [3, 4, 3_000_000]], np.int64)
    o, nb = check(pcu, f, "cuda")
    assert len(o) == 3_000_002 and o[-1] == len(nb) == 16
    lists = pcu.adjacency_list(f.astype(np.int32))
    assert lists[3] == [1, 2, 4, 3_000_000] and lists[5:3_000_000] == [[]] * 2_999_995


@pytest.mark.gpu
def test_rejected_indices(pcu):
    for f in (np.array([[0, 1, -1]], np.int32), np.array([[0, 2 ** 31 - 1, 1], [2, 3, 4]], np.int64),
              np.array([[0, -(2 ** 40), 1]], np.int64)):
        with pytest.raises(ValueError, match="negative or above 2\\^31 - 2"):
            pcu.adjacency_list(f)


@pytest.mark.gpu
def test_input_is_not_modified(pcu):
    import torch
    f = random_faces(np.random.default_rng(9), 20000, 4000, np.int64)
    ft = torch.from_numpy(f).cuda()
    before = ft.clone()
    check(pcu, f, "numpy")
    pcu.adjacency_list(ft, return_csr=True)
    pcu.adjacency_list(ft)
    assert torch.equal(ft, before)
