"""Test inputs shared by the test modules and the timing tools: seeded meshes, and the conversions between numpy arrays
and the input forms a function accepts."""
import numpy as np


def icosphere(level, jitter=0.0, seed=0, dtype=np.float64):
    """The icosahedron subdivided `level` times, each edge split at its midpoint, projected onto the unit sphere:
    (vertices (n, 3) in dtype, faces (m, 3) int64).  Each level appends the new vertices in ascending order of their
    edge (smaller index, larger index).  jitter > 0 adds seeded normal noise of that standard deviation to the
    projected vertices."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    for _ in range(level):
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        uk, inv = np.unique(np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1]), return_inverse=True)
        mid = len(v) + inv.reshape(3, -1).T
        v = np.concatenate([v, 0.5 * (v[uk >> 32] + v[uk & 0xFFFFFFFF])])
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        f = np.concatenate([np.stack([a, mid[:, 0], mid[:, 2]], 1), np.stack([b, mid[:, 1], mid[:, 0]], 1),
                            np.stack([c, mid[:, 2], mid[:, 1]], 1), mid])
    v = v / np.linalg.norm(v, axis=1, keepdims=True)
    if jitter:
        v = v + jitter * np.random.default_rng(seed).standard_normal(v.shape)
    return v.astype(dtype), f


def noisy_icosphere(level, seed=0, amp=0.05):
    """icosphere(level) with every vertex scaled by 1 + amp * (seeded standard normal)."""
    v, f = icosphere(level)
    rng = np.random.default_rng(seed)
    return v * (1.0 + amp * rng.standard_normal((len(v), 1))), f


def torus(nu, nv, r=0.35, dtype=np.float64):
    """A closed torus about the z axis, major radius 1 and minor radius r, on an nu x nv grid of its two angles: two
    triangles per grid cell, (vertices in dtype, faces int64)."""
    u, w = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    v = np.stack([(1.0 + r * np.cos(w)) * np.cos(u), (1.0 + r * np.cos(w)) * np.sin(u), r * np.sin(w)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return v.astype(dtype), f


def to_form(form, a):
    """The numpy array a as the input form "numpy", "cpu" (a CPU tensor) or "cuda" (a CUDA tensor)."""
    import torch
    if form == "numpy":
        return a
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.cuda() if form == "cuda" else t


def to_numpy(x, form=None):
    """A result (numpy array or tensor) as a numpy array.  With form given, first check that the result came back in
    that input form."""
    if form is not None:
        assert isinstance(x, np.ndarray) if form == "numpy" else x.is_cuda == (form == "cuda")
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()
