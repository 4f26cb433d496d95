"""Generates point-cloud-utils_b200/csrc/mc_tables.h, the marching-cubes case tables (DESIGN.md §3).

    python tools/mc_tables.py            # rewrites the header
    python tools/mc_tables.py --check    # exits 1 when the committed header differs

The tables are derived from one rule, not transcribed:
  * corners are numbered as in marching_cubes_sparse_voxel_grid's docstring, edges (0,1) (1,2) (2,3) (3,0) (4,5) (5,6)
    (6,7) (7,4) (0,4) (1,5) (2,6) (3,7); corner k is "above" when bit k of the case is set;
  * on each cube face the crossing edges pair into segments; a face whose diagonal corners agree and whose two
    diagonals disagree is ambiguous, and there the corners above the isovalue are cut off separately.  The choice
    depends on the face's four signs alone, so two cubes sharing a face agree and a hex grid gives a watertight surface;
  * each segment is directed so that, with n the in-face direction towards the corners above and N the face's outward
    normal, it runs along n x N; the segments then chain into cycles whose right-hand normal points towards the corners
    above (an SDF that is negative inside gives outward faces);
  * the cycles are taken in order of their lowest-numbered edge, each starts at that edge, and each is fan-triangulated
    from it: a cycle of k edges gives k - 2 triangles.

A second table, kMcTrisManifold (make_mesh_watertight), has the same cases, cycles and triangle counts; only the fan's
apex differs.  It is the first edge in cycle order none of whose chords (its diagonals to the cycle's non-adjacent
edges) joins two edges on a common cube face.  A segment between two edges of one cube face is shared with the cube
across that face, so a chord there can give an edge four triangles (case 95's chord 4-6 on its top face meets case
245's on its bottom face); a chord between edges that share no face lies inside one cube, and on a grid of such cubes
every surface edge has exactly two triangles.
"""
import os
import sys

CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
# the six faces: four corners in cyclic order, and the outward normal
FACES = [((0, 3, 2, 1), (0, 0, -1)), ((4, 5, 6, 7), (0, 0, 1)), ((0, 1, 5, 4), (0, -1, 0)),
         ((3, 7, 6, 2), (0, 1, 0)), ((0, 4, 7, 3), (-1, 0, 0)), ((1, 2, 6, 5), (1, 0, 0))]
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "point-cloud-utils_b200", "csrc", "mc_tables.h")


def _edge(a, b):
    return EDGES.index((a, b)) if (a, b) in EDGES else EDGES.index((b, a))


def _mid(e):
    a, b = EDGES[e]
    return [(CORNERS[a][k] + CORNERS[b][k]) / 2 for k in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _face_segments(case, corners, normal):
    """Directed segments (edge from, edge to) of one face."""
    above = [(case >> c) & 1 for c in corners]
    ring = [_edge(corners[i], corners[(i + 1) % 4]) for i in range(4)]     # ring[i] joins corners i and i + 1
    crossing = [i for i in range(4) if above[i] != above[(i + 1) % 4]]
    if not crossing:
        return []
    if len(crossing) == 2:
        pairs = [([ring[crossing[0]], ring[crossing[1]]], [corners[i] for i in range(4) if above[i]])]
    else:                                   # ambiguous: cut off each corner above on its own
        pairs = [([ring[(i + 3) % 4], ring[i]], [corners[i]]) for i in range(4) if above[i]]
    out = []
    for (ea, eb), up in pairs:
        pa, pb = _mid(ea), _mid(eb)
        mid = [(pa[k] + pb[k]) / 2 for k in range(3)]
        centre = [sum(CORNERS[c][k] for c in up) / len(up) for k in range(3)]
        n_in = [centre[k] - mid[k] for k in range(3)]
        want = _cross(n_in, normal)
        d = [pb[k] - pa[k] for k in range(3)]
        dot = sum(d[k] * want[k] for k in range(3))
        assert dot != 0
        out.append((ea, eb) if dot > 0 else (eb, ea))
    return out


def case_cycles(case):
    """The cycles of a case, each a list of edges starting at its lowest edge, ordered by that edge."""
    nxt = {}
    for corners, normal in FACES:
        for a, b in _face_segments(case, corners, normal):
            assert a not in nxt, (case, a)
            nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values())            # every crossing edge has one way in and one way out
    cycles, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        cyc, e = [], start
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        assert e == start
        cycles.append(cyc)
    return cycles


def _edge_faces(e):
    """The two cube faces (indices into FACES) that edge e lies on."""
    a, b = EDGES[e]
    return {i for i, (corners, _) in enumerate(FACES) if a in corners and b in corners}


def _shares_face(e, g):
    return bool(_edge_faces(e) & _edge_faces(g))


def manifold_apex(cyc):
    """Position in `cyc` of the first edge whose chords join no two edges on a common cube face."""
    k = len(cyc)
    for j in range(k):
        if not any(_shares_face(cyc[j], cyc[(j + i) % k]) for i in range(2, k - 1)):
            return j
    raise AssertionError(cyc)


def _fan(cyc, j):
    """The fan of cycle `cyc` from position j, in cycle order (orientation kept)."""
    k = len(cyc)
    return [(cyc[j], cyc[(j + i) % k], cyc[(j + i + 1) % k]) for i in range(1, k - 1)]


def tables(manifold=False):
    """(edge masks, triangle lists) of the 256 cases; manifold: the triangles of kMcTrisManifold."""
    masks, tris = [], []
    for case in range(256):
        mask = 0
        for e, (a, b) in enumerate(EDGES):
            if ((case >> a) & 1) != ((case >> b) & 1):
                mask |= 1 << e
        cyc = case_cycles(case)
        assert sorted(e for c in cyc for e in c) == [e for e in range(12) if mask >> e & 1]
        masks.append(mask)
        tris.append([t for c in cyc for t in _fan(c, manifold_apex(c) if manifold else 0)])
    return masks, tris


def check_manifold_table():
    """The manifold table's asserted properties: the edge masks, cycles and triangle counts of kMcTris, every triangle's
    edges in one cycle of its case, and no chord between two edges that share a cube face.  Returns the number of
    cycles whose apex moved."""
    masks, tris = tables()
    masks_m, tris_m = tables(manifold=True)
    assert masks_m == masks and [len(t) for t in tris_m] == [len(t) for t in tris]
    moved = 0
    for case in range(256):
        cycles = case_cycles(case)
        got = list(tris_m[case])
        for c in cycles:
            fan, got = got[:len(c) - 2], got[len(c) - 2:]
            apex = fan[0][0] if fan else c[0]
            assert all(t[0] == apex and {t[1], t[2]} <= set(c) for t in fan)
            assert fan == _fan(c, c.index(apex))
            for t in fan:                       # chords: the apex's diagonals to non-adjacent cycle edges
                for e in (t[1], t[2]):
                    k, p, q = len(c), c.index(apex), c.index(e)
                    if (q - p) % k not in (1, k - 1):
                        assert not _shares_face(apex, e), (case, c, apex, e)
            moved += apex != c[0]
        assert not got
    return moved


MAX_TRIS = 5      # the most triangles any case has (asserted below); the kernels size per-cube work by it


def render():
    masks, tris = tables()
    _, tris_m = tables(manifold=True)
    check_manifold_table()
    most = max(len(t) for t in tris)
    assert most == MAX_TRIS, most
    lines = ["// mc_tables.h -- marching-cubes case tables, written by tools/mc_tables.py (do not edit; DESIGN.md §3).",
             "// Case bit k: corner k above the isovalue; edges are numbered as in the generator (mc_edge_corners, sparse_voxels.cuh).",
             "#pragma once", "", "namespace pcu {", "",
             "constexpr int kMcMaxTris = %d;   // the most triangles of any case" % most, "",
             "// crossing edges of each case (bit e: edge e)",
             "__device__ const unsigned short kMcEdgeMask[256] = {"]
    for r in range(0, 256, 16):
        lines.append("    " + ", ".join("0x%03x" % m for m in masks[r:r + 16]) + ",")
    lines += ["};", "", "// triangles of each case",
              "__device__ const unsigned char kMcTriCount[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in tris[r:r + 32]) + ",")
    lines += ["};", "", "// the triangles' edges, three per triangle, unused entries 255",
              "__device__ const unsigned char kMcTris[256][3 * kMcMaxTris] = {"]
    for case, t in enumerate(tris):
        flat = [e for tri in t for e in tri] + [255] * (3 * most - 3 * len(t))
        lines.append("    {%s},   // %d" % (", ".join(str(e) for e in flat), case))
    lines += ["};", "", "// make_mesh_watertight's triangles: kMcTris with each fan's apex moved to the first edge of its cycle none of",
              "// whose chords joins two edges on a common cube face (closed 2-manifolds on a grid of cubes); counts as kMcTriCount",
              "__device__ const unsigned char kMcTrisManifold[256][3 * kMcMaxTris] = {"]
    for case, t in enumerate(tris_m):
        flat = [e for tri in t for e in tri] + [255] * (3 * most - 3 * len(t))
        lines.append("    {%s},   // %d" % (", ".join(str(e) for e in flat), case))
    lines += ["};", "", "}  // namespace pcu", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    text = render()
    if "--check" in sys.argv:
        with open(HEADER) as fh:
            sys.exit(0 if fh.read() == text else 1)
    with open(HEADER, "w") as fh:
        fh.write(text)
    print(HEADER)
