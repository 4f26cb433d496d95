"""Writes tests/golden/bunny_vertices.npy: the (2885, 3) float32 vertices of the reference's data/bunny.ply, whose faces
are tests/golden/bunny_faces.npy.  The file is binary little-endian PLY with float x, y, z per vertex and int-counted
int faces; the faces it holds are checked against the committed ones.

    python tools/bunny_golden.py /path/to/point-cloud-utils/data/bunny.ply"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii", "replace").splitlines()
    assert "format binary_little_endian 1.0" in header
    nv = next(int(h.split()[2]) for h in header if h.startswith("element vertex"))
    nf = next(int(h.split()[2]) for h in header if h.startswith("element face"))
    props = [h.split()[2] for h in header if h.startswith("property float")]
    assert props == ["x", "y", "z"], props
    assert "property list int int vertex_indices" in header
    v = np.frombuffer(data, "<f4", 3 * nv, end).reshape(nv, 3)
    rows = np.frombuffer(data, "<i4", 4 * nf, end + 12 * nv).reshape(nf, 4)
    assert (rows[:, 0] == 3).all()
    return v.copy(), rows[:, 1:].copy()


if __name__ == "__main__":
    v, f = read_ply(sys.argv[1])
    golden = os.path.join(ROOT, "tests", "golden")
    assert np.array_equal(f, np.load(os.path.join(golden, "bunny_faces.npy"))), "faces differ from bunny_faces.npy"
    np.save(os.path.join(golden, "bunny_vertices.npy"), v.astype(np.float32))
    print("bunny_vertices.npy:", v.shape, v.dtype)
