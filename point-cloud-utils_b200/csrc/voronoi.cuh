// voronoi.cuh -- Voronoi cells of seeds in the unit cube / square, their centroids, and the Lloyd and L-BFGS
// relaxations on top of them (voronoi_centroids_unit_cube, lloyd_3d and lloyd_2d of the reference, src/lloyd.cpp).
//
// The cells are computed as in Ray, Sokolov, Lefebvre and Levy, "Meshless Voronoi on the GPU" (ACM TOG 37(6), 2018):
// one thread per cell clips the cube by the bisectors of the seed's nearest neighbours, in increasing distance, and
// stops once the security radius certifies the cell (DESIGN.md §3, Voronoi cell):
//   3-D  the cell is kept in the paper's dual form: planes are numbered (0..5 the cube's faces, then one per bisector
//        that cut the cell) and every vertex is an oriented triplet of plane numbers, so that the twin of the directed
//        edge (a, b) of one vertex is the edge (b, a) of its neighbour along that edge.  A clip removes the vertices
//        strictly outside the new plane and gives every boundary edge (x, y) of the removed set the vertex (x, y, new).
//        Vertex positions (relative to the seed) are cached when a vertex is made, by interpolation along its edge.
//   2-D  the cell is its counter-clockwise cycle of vertices, clipped by each bisector line.
//   certificate  4 R^2 (1 + kVorMargin) < d^2_next, R the largest seed-to-vertex distance, d_next the distance of the
//        first unused neighbour (or of the k-th when the list is used up): no seed at least 2R away can cut the cell.
// Volume, first moment and second moment about the seed are integrated in the same thread with a tetrahedron
// (triangle) fan from the seed.  Every sum is sequential in one thread: no atomics, results are bit-reproducible.
// The same passes clip the (face, seed) pairs of cells restricted to a triangle mesh (rvd.cuh), each as a convex
// polygon (Poly3) with the same certificate, duplicate rule and cut tolerance.
#pragma once
#include <cooperative_groups.h>
#include <type_traits>
#include "common.cuh"
#include "compact.cuh"

namespace pcu {

constexpr int kVorThreads = 128;
constexpr double kVorMassMin = 1e-30;     // the reference's threshold for a non-empty cell (src/lloyd.cpp:136)
constexpr double kVorMargin = 1e-10;      // relative margin that keeps the certificate conservative under fp64 rounding
constexpr int kVorMoments = 5;            // per cell: volume, first moment about the seed (x, y, z), second moment
// A vertex is cut off only when it lies beyond the plane by more than kVorClipTol * d (d = |c_j - c_i|^2 / 2): a plane
// through vertices made by an equal plane (a duplicate seed's bisector) or passing within rounding of them cuts nothing,
// where cutting a sliver of rounding noise would make vertices without a twin.
constexpr double kVorClipTol = 1e-13;

// One clipping pass over `count` cells.  Entry t of the pass is the cell rows[sub[t]] (a null array is the identity),
// and its neighbour list is row sub[t] of the lists.  Restricted cells (rvd.cuh) clip (face, seed) pairs instead: the
// row is a pair, whose seed and face the pair arrays give, and in the first pass the lists are the seeds' own.
struct VorPass {
    const double* x;          // (n, D) seeds
    const double* x3;         // (n, 3) seeds (the 2-D seeds with z = 0)
    long long n;
    const int* rows;
    const int* sub;
    long long count;
    const long long* nn_idx;  // (entries, k), ascending distance, -1 past the end of a short list
    const double* nn_d2;      // squared distances of the list, as the k-NN search rounds them
    int k;
    int list_is_all;          // every seed is in every list: a cell is exact once its list is used up
    int scan_all;             // the last resort: after the list, every seed with d^2 >= d^2_k is tried too
    double* mom;              // (n, kVorMoments)
    unsigned char* uncert;    // (count): 1 = the cell is left to the next pass
    void* cells;              // last resort: one cell record per entry
    const int* pair_seed;     // restricted cells: the seed of each pair (null: the row is the seed)
    const int* pair_face;     // the face of each pair
    const double* tri;        // (faces, 9): every face's corners
    int list_of_seed;         // the neighbour list of an entry is its seed's row of the lists
};

// the k-NN search's rounding of d^2, so that "in the list" is decided exactly
__host__ __device__ __forceinline__ double vor_d2(const double* a, const double* b) {
#ifdef __CUDA_ARCH__
    return dist2<double>(a[0], a[1], a[2], b[0], b[1], b[2]);
#else
    const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return (dx * dx + dy * dy) + dz * dz;
#endif
}

// ---- 3-D cells --------------------------------------------------------------------------------------------------
// A cell over storage it does not own: V vertex slots (plane triplets and positions), P plane numbers (a work array of
// P entries) and a V-bit mask.  The passes keep that storage on the thread's stack (VorStack) or, for the last resort,
// in device memory at a capacity chosen at run time (vor_cell_bytes).
template <class I>
struct Cell3 {
    I (*tri)[3];
    double (*pos)[3];
    I* work;            // P: plane renumbering while clipping, face anchors while integrating
    unsigned* out;      // (V + 31) / 32 words
    int V, P;
    int nv, np;

    __host__ __device__ void init(const double* c) {
        np = 6;
        nv = 8;
        for (int v = 0; v < 8; ++v) {
            const int sx = v & 1, sy = (v >> 1) & 1, sz = (v >> 2) & 1;
            // planes 2a (low side of axis a, normal -e_a) and 2a + 1 (high side, +e_a); the triplet is ordered so that
            // det(n_a, n_b, n_c) > 0, which orients every vertex alike
            I a = (I)sx, b = (I)(2 + sy), cc = (I)(4 + sz);
            const int sign = (sx ? 1 : -1) * (sy ? 1 : -1) * (sz ? 1 : -1);
            if (sign < 0) { const I t = a; a = b; b = t; }
            tri[v][0] = a; tri[v][1] = b; tri[v][2] = cc;
            pos[v][0] = (sx ? 1.0 : 0.0) - c[0];
            pos[v][1] = (sy ? 1.0 : 0.0) - c[1];
            pos[v][2] = (sz ? 1.0 : 0.0) - c[2];
        }
    }

    __host__ __device__ int twin(int y, int x) const {   // the vertex holding the directed edge (y, x), or -1
        for (int u = 0; u < nv; ++u) {
            const int t0 = tri[u][0], t1 = tri[u][1], t2 = tri[u][2];
            if ((t0 == y && t1 == x) || (t1 == y && t2 == x) || (t2 == y && t0 == x)) return u;
        }
        return -1;
    }

    __host__ __device__ double side(int v, const double* nrm, double d) const {
        return pos[v][0] * nrm[0] + pos[v][1] * nrm[1] + pos[v][2] * nrm[2] - d;
    }

    __host__ __device__ bool is_out(int v) const { return (out[v >> 5] >> (v & 31)) & 1u; }

    // Gives the planes that still bound a vertex the numbers 0, 1, ... in order of first use: a plane whose face a later
    // clip removed gives its number back.  The cell keeps at most V / 2 + 2 faces (its dual is a triangulated sphere
    // with nv triangles), so numbers run out only when the vertices do.
    __host__ __device__ void renumber() {
        const I none = (I)~(I)0;
        for (int p = 0; p < np; ++p) work[p] = none;
        int next = 0;
        for (int v = 0; v < nv; ++v)
            for (int e = 0; e < 3; ++e) {
                const int p = tri[v][e];
                if (work[p] == none) work[p] = (I)next++;
                tri[v][e] = work[p];
            }
        np = next;
    }

    // Clips by {x : nrm . x <= d}.  0: nothing cut, 1: clipped, 2: capacity exceeded (or a broken edge), 3: empty.
    __host__ __device__ int clip(const double* nrm, double d) {
        for (int w = 0; w < (V + 31) / 32; ++w) out[w] = 0u;
        int nout = 0;
        const double tol = kVorClipTol * d;
        for (int v = 0; v < nv; ++v)
            if (side(v, nrm, d) > tol) { out[v >> 5] |= 1u << (v & 31); ++nout; }
        if (nout == 0) return 0;
        if (nout == nv) { nv = 0; return 3; }
        if (np >= P) renumber();
        if (np >= P) return 2;
        const I pn = (I)np;
        int nb = 0;
        for (int v = 0; v < nv; ++v) {
            if (!is_out(v)) continue;
            for (int e = 0; e < 3; ++e) {
                const int x = tri[v][e], y = tri[v][(e + 1) % 3];
                const int u = twin(y, x);
                if (u < 0) return 2;
                if (is_out(u)) continue;
                const int s = nv + nb;
                if (s >= V) return 2;
                ++nb;
                const double hv = side(v, nrm, d), hu = side(u, nrm, d);   // hv > tol >= hu
                const double f = fmin(1.0, hv / (hv - hu));
                for (int a = 0; a < 3; ++a) pos[s][a] = pos[v][a] + (pos[u][a] - pos[v][a]) * f;
                tri[s][0] = (I)x; tri[s][1] = (I)y; tri[s][2] = pn;
            }
        }
        int w = 0;
        for (int v = 0; v < nv + nb; ++v) {
            if (v < nv && is_out(v)) continue;
            if (w != v) {
                for (int a = 0; a < 3; ++a) { tri[w][a] = tri[v][a]; pos[w][a] = pos[v][a]; }
            }
            ++w;
        }
        nv = w;
        np = pn + 1;
        return 1;
    }

    __host__ __device__ double radius2() const {
        double r = 0.0;
        for (int v = 0; v < nv; ++v) r = fmax(r, pos[v][0] * pos[v][0] + pos[v][1] * pos[v][1] + pos[v][2] * pos[v][2]);
        return r;
    }

    // Volume, first moment and second moment about the seed: every face is fanned from its first vertex, and every
    // fan triangle with the seed spans a tetrahedron.  The seed lies in its (convex) cell, so every such tetrahedron
    // has the orientation of its face and |det| / 6 is its volume.
    __host__ __device__ void integrate(double* m) {
        I* anchor = work;
        for (int p = 0; p < np; ++p) anchor[p] = (I)0;
        for (int v = nv - 1; v >= 0; --v)
            for (int e = 0; e < 3; ++e) anchor[tri[v][e]] = (I)v;
        double vol = 0.0, mx = 0.0, my = 0.0, mz = 0.0, m2 = 0.0;
        for (int v = 0; v < nv; ++v) {
            for (int e = 0; e < 3; ++e) {
                const int x = tri[v][e], y = tri[v][(e + 1) % 3];
                const int u = twin(y, x);       // the edge from v to u lies on face x
                const int a = anchor[x];
                if (u < 0 || a == v || a == u) continue;
                const double* A = pos[a];
                const double* B = pos[v];
                const double* C = pos[u];
                const double det = A[0] * (B[1] * C[2] - B[2] * C[1]) - A[1] * (B[0] * C[2] - B[2] * C[0]) +
                                   A[2] * (B[0] * C[1] - B[1] * C[0]);
                const double t = fabs(det) / 6.0;
                vol += t;
                mx += t * (A[0] + B[0] + C[0]) * 0.25;
                my += t * (A[1] + B[1] + C[1]) * 0.25;
                mz += t * (A[2] + B[2] + C[2]) * 0.25;
                const double q = A[0] * A[0] + A[1] * A[1] + A[2] * A[2] + B[0] * B[0] + B[1] * B[1] + B[2] * B[2] +
                                 C[0] * C[0] + C[1] * C[1] + C[2] * C[2] + A[0] * B[0] + A[1] * B[1] + A[2] * B[2] +
                                 B[0] * C[0] + B[1] * C[1] + B[2] * C[2] + C[0] * A[0] + C[1] * A[1] + C[2] * A[2];
                m2 += t * q * 0.1;
            }
        }
        m[0] = vol; m[1] = mx; m[2] = my; m[3] = mz; m[4] = m2;
    }
};

// ---- 2-D cells --------------------------------------------------------------------------------------------------
// The counter-clockwise vertex cycle over V slots of storage it does not own, and V more for the clip's output.
struct Cell2 {
    double (*pos)[2];
    double (*tmp)[2];
    int V;
    int nv;

    __host__ __device__ void init(const double* c) {
        nv = 4;
        const double xs[4] = {0.0, 1.0, 1.0, 0.0}, ys[4] = {0.0, 0.0, 1.0, 1.0};
        for (int v = 0; v < 4; ++v) { pos[v][0] = xs[v] - c[0]; pos[v][1] = ys[v] - c[1]; }
    }

    __host__ __device__ double side(const double* p, const double* nrm, double d) const { return p[0] * nrm[0] + p[1] * nrm[1] - d; }

    __host__ __device__ int clip(const double* nrm, double d) {
        const double tol = kVorClipTol * d;
        int nout = 0;
        for (int v = 0; v < nv; ++v) nout += side(pos[v], nrm, d) > tol;
        if (nout == 0) return 0;
        if (nout == nv) { nv = 0; return 3; }
        int w = 0;
        for (int v = 0; v < nv; ++v) {
            const int u = v + 1 == nv ? 0 : v + 1;
            const double hv = side(pos[v], nrm, d), hu = side(pos[u], nrm, d);
            if (!(hv > tol)) {
                if (w >= V) return 2;
                tmp[w][0] = pos[v][0]; tmp[w][1] = pos[v][1]; ++w;
            }
            if ((hv > tol) != (hu > tol)) {
                if (w >= V) return 2;
                // interpolate from the outside end, as the 3-D clip does
                const double* o = hv > tol ? pos[v] : pos[u];
                const double* i = hv > tol ? pos[u] : pos[v];
                const double ho = hv > tol ? hv : hu, hi = hv > tol ? hu : hv;
                const double f = fmin(1.0, ho / (ho - hi));
                tmp[w][0] = o[0] + (i[0] - o[0]) * f;
                tmp[w][1] = o[1] + (i[1] - o[1]) * f;
                ++w;
            }
        }
        for (int v = 0; v < w; ++v) { pos[v][0] = tmp[v][0]; pos[v][1] = tmp[v][1]; }
        nv = w;
        return 1;
    }

    __host__ __device__ double radius2() const {
        double r = 0.0;
        for (int v = 0; v < nv; ++v) r = fmax(r, pos[v][0] * pos[v][0] + pos[v][1] * pos[v][1]);
        return r;
    }

    __host__ __device__ void integrate(double* m) const {
        double vol = 0.0, mx = 0.0, my = 0.0, m2 = 0.0;
        for (int v = 0; v < nv; ++v) {
            const double* A = pos[v];
            const double* B = pos[v + 1 == nv ? 0 : v + 1];
            const double t = fabs(A[0] * B[1] - A[1] * B[0]) * 0.5;
            vol += t;
            mx += t * (A[0] + B[0]) / 3.0;
            my += t * (A[1] + B[1]) / 3.0;
            m2 += t * (A[0] * A[0] + A[1] * A[1] + B[0] * B[0] + B[1] * B[1] + A[0] * B[0] + A[1] * B[1]) / 6.0;
        }
        m[0] = vol; m[1] = mx; m[2] = my; m[3] = 0.0; m[4] = m2;
    }
};

// ---- restricted cells ---------------------------------------------------------------------------------------------
// One face's share of a restricted cell (DESIGN.md §3, restricted cell): the triangle, relative to the seed, clipped
// as a convex 3-D polygon (its vertex cycle) by each bisector, over V slots of storage it does not own and V more for
// the clip's output.  A triangle clipped by k planes has at most 3 + k vertices.
struct Poly3 {
    double (*pos)[3];
    double (*tmp)[3];
    int V;
    int nv;

    __host__ __device__ void init(const double* c, const double* t) {   // t: the face's corners a, b, c
        nv = 3;
        for (int v = 0; v < 3; ++v)
            for (int a = 0; a < 3; ++a) pos[v][a] = t[3 * v + a] - c[a];
    }

    __host__ __device__ double side(const double* p, const double* nrm, double d) const {
        return p[0] * nrm[0] + p[1] * nrm[1] + p[2] * nrm[2] - d;
    }

    // Cell2::clip in 3-D: the same tolerance, interpolation from the outside end, and results.
    __host__ __device__ int clip(const double* nrm, double d) {
        const double tol = kVorClipTol * d;
        int nout = 0;
        for (int v = 0; v < nv; ++v) nout += side(pos[v], nrm, d) > tol;
        if (nout == 0) return 0;
        if (nout == nv) { nv = 0; return 3; }
        int w = 0;
        for (int v = 0; v < nv; ++v) {
            const int u = v + 1 == nv ? 0 : v + 1;
            const double hv = side(pos[v], nrm, d), hu = side(pos[u], nrm, d);
            if (!(hv > tol)) {
                if (w >= V) return 2;
                for (int a = 0; a < 3; ++a) tmp[w][a] = pos[v][a];
                ++w;
            }
            if ((hv > tol) != (hu > tol)) {
                if (w >= V) return 2;
                const double* o = hv > tol ? pos[v] : pos[u];
                const double* i = hv > tol ? pos[u] : pos[v];
                const double ho = hv > tol ? hv : hu, hi = hv > tol ? hu : hv;
                const double f = fmin(1.0, ho / (ho - hi));
                for (int a = 0; a < 3; ++a) tmp[w][a] = o[a] + (i[a] - o[a]) * f;
                ++w;
            }
        }
        for (int v = 0; v < w; ++v)
            for (int a = 0; a < 3; ++a) pos[v][a] = tmp[v][a];
        nv = w;
        return 1;
    }

    __host__ __device__ double radius2() const {
        double r = 0.0;
        for (int v = 0; v < nv; ++v) r = fmax(r, pos[v][0] * pos[v][0] + pos[v][1] * pos[v][1] + pos[v][2] * pos[v][2]);
        return r;
    }

    // Area, first moment and second moment about the seed by a fan from vertex 0: a fan triangle w0 w1 w2 of area A
    // adds A (w0 + w1 + w2) / 3 and A / 12 (sum |w_a|^2 + |sum w_a|^2).
    __host__ __device__ void integrate(double* m) const {
        double ar = 0.0, mx = 0.0, my = 0.0, mz = 0.0, m2 = 0.0;
        const double* A = pos[0];
        for (int v = 1; v + 1 < nv; ++v) {
            const double* B = pos[v];
            const double* C = pos[v + 1];
            const double e1[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]}, e2[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
            const double cx = e1[1] * e2[2] - e1[2] * e2[1], cy = e1[2] * e2[0] - e1[0] * e2[2], cz = e1[0] * e2[1] - e1[1] * e2[0];
            const double t = 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
            const double sx = A[0] + B[0] + C[0], sy = A[1] + B[1] + C[1], sz = A[2] + B[2] + C[2];
            ar += t;
            mx += t * sx / 3.0;
            my += t * sy / 3.0;
            mz += t * sz / 3.0;
            const double q = A[0] * A[0] + A[1] * A[1] + A[2] * A[2] + B[0] * B[0] + B[1] * B[1] + B[2] * B[2] +
                             C[0] * C[0] + C[1] * C[1] + C[2] * C[2] + sx * sx + sy * sy + sz * sz;
            m2 += t * q / 12.0;
        }
        m[0] = ar; m[1] = mx; m[2] = my; m[3] = mz; m[4] = m2;
    }
};

template <int V>
struct PolyStack {
    double pos[V][3];
    double tmp[V][3];
    __host__ __device__ Poly3 view() { return Poly3{pos, tmp, V, 0}; }
};
__host__ __device__ inline size_t poly_bytes(int V) { return (size_t)V * 48; }
__host__ __device__ inline Poly3 poly_at(unsigned char* base, int V) {
    return Poly3{reinterpret_cast<double (*)[3]>(base), reinterpret_cast<double (*)[3]>(base + (size_t)V * 24), V, 0};
}

// Storage of a cell with a fixed capacity of V vertices (and, in 3-D, P = V / 2 + 8 plane numbers), and its layout in
// a block of device memory for a capacity chosen at run time.
template <int D, int V, class I = unsigned char>
struct VorStack;
template <int V, class I>
struct VorStack<3, V, I> {
    static constexpr int P = V / 2 + 8;
    I tri[V][3];
    double pos[V][3];
    I work[P];
    unsigned out[(V + 31) / 32];
    __host__ __device__ Cell3<I> view() { return Cell3<I>{tri, pos, work, out, V, P, 0, 0}; }
};
template <int V, class I>
struct VorStack<2, V, I> {
    double pos[V][2];
    double tmp[V][2];
    __host__ __device__ Cell2 view() { return Cell2{pos, tmp, V, 0}; }
};

// Bytes of one last-resort cell of V vertices (a multiple of 8), and the cell laid out at `base`.
template <int D>
__host__ __device__ inline size_t vor_cell_bytes(int V) {
    if (D == 2) return (size_t)V * 32;
    const size_t P = (size_t)V / 2 + 8;
    return ((size_t)V * 24 + (size_t)V * 12 + P * 4 + (size_t)((V + 31) / 32) * 4 + 7) / 8 * 8;
}
__host__ __device__ inline Cell3<int> vor_cell_at3(unsigned char* base, int V) {
    double (*pos)[3] = reinterpret_cast<double (*)[3]>(base);
    int (*tri)[3] = reinterpret_cast<int (*)[3]>(base + (size_t)V * 24);
    int* work = reinterpret_cast<int*>(base + (size_t)V * 36);
    unsigned* out = reinterpret_cast<unsigned*>(base + (size_t)V * 36 + ((size_t)V / 2 + 8) * 4);
    return Cell3<int>{tri, pos, work, out, V, V / 2 + 8, 0, 0};
}
__host__ __device__ inline Cell2 vor_cell_at2(unsigned char* base, int V) {
    return Cell2{reinterpret_cast<double (*)[2]>(base), reinterpret_cast<double (*)[2]>(base + (size_t)V * 16), V, 0};
}

// Entry t of a pass, in `cell`'s storage.  C: Cell2 or Cell3 at the pass's capacity, or Poly3 for a (face, seed) pair.
template <int D, class C>
__host__ __device__ __forceinline__ void vor_cell(const VorPass& a, long long t, C& cell) {
    const long long e = a.sub ? (long long)a.sub[t] : t;
    const long long row = a.rows ? (long long)a.rows[e] : e;                    // the output row: a cell or a pair
    constexpr bool pair = std::is_same<C, Poly3>::value;
    const long long seed = pair ? (long long)a.pair_seed[row] : row;
    const long long list = pair && a.list_of_seed ? seed : e;
    const double* c = a.x + seed * D;
    const double* c3 = a.x3 + seed * 3;
    const long long* li = a.nn_idx + list * a.k;
    const double* ld = a.nn_d2 + list * a.k;
    if constexpr (pair) cell.init(c, a.tri + 9 * (long long)a.pair_face[row]);
    else cell.init(c);
    double r2 = cell.radius2();
    bool done = false, empty = false, over = false;
    // a clip by the bisector of seed s; false: stop here (empty or over capacity)
    auto cut = [&](long long s) {
        const double* cs = a.x + s * D;
        double nrm[3] = {0.0, 0.0, 0.0};
        double dd = 0.0;
        for (int q = 0; q < D; ++q) { nrm[q] = cs[q] - c[q]; dd += nrm[q] * nrm[q]; }
        const int r = cell.clip(nrm, 0.5 * dd);
        if (r == 3) { empty = true; return false; }
        if (r == 2) { over = true; return false; }
        if (r == 1) r2 = cell.radius2();
        return true;
    };
    for (int j = 0; j < a.k; ++j) {
        const long long s = li[j];
        if (s < 0) break;                 // a short list: every seed is in it
        const double d2 = ld[j];
        if (4.0 * r2 * (1.0 + kVorMargin) < d2) { done = true; break; }
        if (s == seed) continue;
        if (d2 == 0.0) {                  // a duplicate: the lowest index owns the position
            if (s < seed) { empty = true; break; }
            continue;
        }
        if (!cut(s)) break;
    }
    if (!done && !empty && !over) {
        if (a.list_is_all) {
            done = true;
        } else if (a.scan_all) {
            const double dk = ld[a.k - 1];
            for (long long s = 0; s < a.n && !empty && !over; ++s) {
                if (s == seed) continue;
                const double d2 = vor_d2(c3, a.x3 + s * 3);
                if (d2 < dk) continue;     // in the list, clipped above
                if (d2 == 0.0) {
                    if (s < seed) empty = true;
                    continue;
                }
                if (4.0 * r2 * (1.0 + kVorMargin) < d2) continue;
                cut(s);
            }
            done = !over;
        } else {
            done = 4.0 * r2 * (1.0 + kVorMargin) < ld[a.k - 1];
        }
    }
    double* m = a.mom + row * kVorMoments;
    if (empty) {
        for (int q = 0; q < kVorMoments; ++q) m[q] = 0.0;
    } else if (done) {
        cell.integrate(m);
    }
    a.uncert[t] = (unsigned char)(!(done || empty));   // the last resort: over capacity, redone at twice it
}

// One thread per entry of the pass, its cell on the thread's stack at a capacity of V vertices.
template <int D, int V>
__global__ void __launch_bounds__(kVorThreads, 4) vor_clip_kernel(VorPass a) {   // 4 CTAs: up to 128 registers
    grid_dependency_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.count) return;
    VorStack<D, V> s;
    auto cell = s.view();
    vor_cell<D>(a, t, cell);
}

// The last resort: one thread per entry, its cell in device memory (a.cells) at a capacity of V vertices.
template <int D>
__global__ void __launch_bounds__(kVorThreads) vor_clip_wide_kernel(VorPass a, int V) {
    grid_dependency_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.count) return;
    unsigned char* base = (unsigned char*)a.cells + (size_t)t * vor_cell_bytes<D>(V);
    if constexpr (D == 3) {
        Cell3<int> cell = vor_cell_at3(base, V);
        vor_cell<D>(a, t, cell);
    } else {
        Cell2 cell = vor_cell_at2(base, V);
        vor_cell<D>(a, t, cell);
    }
}

// The (face, seed) pairs of restricted cells: one thread per entry, its polygon on the stack at V vertices, or for the
// last resort in device memory (a.cells).
template <int V>
__global__ void __launch_bounds__(kVorThreads, 4) rv_clip_kernel(VorPass a) {
    grid_dependency_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.count) return;
    PolyStack<V> s;
    Poly3 cell = s.view();
    vor_cell<3>(a, t, cell);
}
__global__ void __launch_bounds__(kVorThreads) rv_clip_wide_kernel(VorPass a, int V) {
    grid_dependency_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.count) return;
    Poly3 cell = poly_at((unsigned char*)a.cells + (size_t)t * poly_bytes(V), V);
    vor_cell<3>(a, t, cell);
}

// The next round of the last resort: the entries of this round (sub) whose cells are still flagged, in order.
__global__ void __launch_bounds__(kThreads) vor_keep_sub_kernel(const unsigned char* __restrict__ keep, long long n,
                                                                const unsigned* __restrict__ block_offset,
                                                                const int* __restrict__ sub, int* __restrict__ next) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? keep[i] : 0u;
    const unsigned pos = keep_rank(mine, block_offset);
    if (mine) next[pos] = sub[i];
}

// (n, 2) seeds -> (n, 3) with z = 0, the k-NN search's input
__global__ void __launch_bounds__(kThreads) vor_lift_kernel(const double* __restrict__ x, long long n, double* __restrict__ x3) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    x3[i * 3] = x[i * 2];
    x3[i * 3 + 1] = x[i * 2 + 1];
    x3[i * 3 + 2] = 0.0;
}

// the (count, 3) seeds of the compacted rows (of seed[row] when seed is not null): the queries of the next k-NN search
__global__ void __launch_bounds__(kThreads) vor_gather_kernel(const double* __restrict__ x3, const int* __restrict__ rows,
                                                              long long count, double* __restrict__ q,
                                                              const int* __restrict__ seed) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const long long r = seed ? seed[rows[i]] : rows[i];
    for (int a = 0; a < 3; ++a) q[i * 3 + a] = x3[r * 3 + a];
}

// Centroid rows: c + m1 / m when m > 1e-30, else the seed itself.  out may be x.
template <int D>
__global__ void __launch_bounds__(kThreads) vor_centroid_kernel(const double* x, long long n, const double* __restrict__ mom,
                                                                double* out) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* m = mom + i * kVorMoments;
    const double vol = m[0];
    for (int a = 0; a < D; ++a) {
        const double c = x[i * D + a];
        out[i * D + a] = vol > kVorMassMin ? c + m[1 + a] / vol : c;
    }
}

// The initial sample: coordinate (row, axis) is a 53-bit uniform value in [0, 1) from two mix32 words keyed by the
// seed and the counter 2 (row * D + axis) (+ 1), numpy's genrand_res53 construction (27 high bits, 26 low bits).
__device__ __forceinline__ unsigned lloyd_word(unsigned seed, unsigned long long c) {
    return mix32(seed ^ mix32((unsigned)c ^ mix32((unsigned)(c >> 32))));
}
__global__ void __launch_bounds__(kThreads) lloyd_init_kernel(unsigned seed, long long count, double* __restrict__ x) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const unsigned long long c = 2ull * (unsigned long long)i;
    const unsigned hi = lloyd_word(seed, c) >> 5, lo = lloyd_word(seed, c + 1) >> 6;
    x[i] = ((double)hi * 67108864.0 + (double)lo) * (1.0 / 9007199254740992.0);
}

// ---- L-BFGS on the CVT energy ----------------------------------------------------------------------------------
constexpr int kLbMemory = 7;
constexpr int kLbSlots = kLbMemory + 1;   // the slot at `head` is scratch for the pair being formed
constexpr int kLbMaxHalvings = 20;
constexpr double kLbArmijo = 1e-4;

// What the host reads at the synchronisation that sizes a fallback pass: the rows left to it, and the state of the
// Newton phase (written by the last step).
struct VorSync {
    long long count;      // rows flagged by the last pass
    int done;             // the Newton phase is over
    int iter;             // accepted Newton steps
};

struct LbState {
    double F, gtp, t, gamma;
    double rho[kLbSlots];
    int iter, halvings, done, init, hist, head;
};

struct LbArgs {
    long long n;
    int D;
    double* x_acc;     // (n, D) last accepted point
    double* g;         // its gradient
    double* x_t;       // the trial point, whose cells `mom` holds
    const double* mom;
    double* p;         // search direction (the two-loop recursion runs in place here)
    double* S;         // kLbSlots x (n D)
    double* Y;
    double* partial;   // 2 x gridDim.x
    LbState* st;
    VorSync* sync;
    double* energy;    // num_newton + 1: F of the accepted points
    int num_newton;
    int cube;          // trial points must lie in the unit cube (square); restricted cells have no domain test
};

// Sum over the grid in a fixed order: the block's tree, then the blocks in index order, redundantly in every block.
// Every thread of the grid calls it, the same number of times; the partials alternate between two halves so that a
// block may write the next sum's partial while another still reads this one's.
__device__ double lb_grid_sum(double v, double* partial, int& parity) {
    namespace cg = cooperative_groups;
    __shared__ double warp_sum[kThreads / 32];
    __shared__ double total;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_sum[w] = v;
    __syncthreads();
    double* half = partial + parity * gridDim.x;
    parity ^= 1;
    if (threadIdx.x == 0) {
        double b = 0.0;
        for (int q = 0; q < kThreads / 32; ++q) b += warp_sum[q];
        half[blockIdx.x] = b;
    }
    cg::this_grid().sync();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (unsigned q = 0; q < gridDim.x; ++q) s += ((volatile double*)half)[q];
        total = s;
    }
    __syncthreads();
    const double r = total;
    __syncthreads();
    return r;
}

// One step of the Newton phase, after the cells of the trial point x_t have been computed (or of the starting point,
// st->init): the Armijo test of the trial, then either the L-BFGS update and the next direction, or a halved step;
// and the next trial point x_acc + t p inside the cube (a point outside fails the test without being evaluated; with
// a.cube unset, as for restricted cells, every trial point is evaluated).
// Cooperative: every decision is taken identically by every thread from grid-wide sums.
__global__ void __launch_bounds__(kThreads) lbfgs_step_kernel(LbArgs a) {
    grid_dependency_wait();
    LbState s = *a.st;
    if (s.done) return;
    const long long N = a.n * a.D;
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long gsize = (long long)gridDim.x * blockDim.x;
    int parity = 0;
    double acc = 0.0;
    for (long long i = gtid; i < a.n; i += gsize) acc += a.mom[i * kVorMoments + 4];
    const double Ft = lb_grid_sum(acc, a.partial, parity);
    const bool accept = s.init || Ft <= s.F + kLbArmijo * s.t * s.gtp;
    bool need_dir = false;
    if (accept) {
        const int slot = s.head;
        double* Sv = a.S + (long long)slot * N;
        double* Yv = a.Y + (long long)slot * N;
        double sy = 0.0, yy = 0.0;
        for (long long i = gtid; i < N; i += gsize) {
            const double gt = -2.0 * a.mom[(i / a.D) * kVorMoments + 1 + (i % a.D)];
            if (!s.init) {
                const double sv = a.x_t[i] - a.x_acc[i], yv = gt - a.g[i];
                Sv[i] = sv; Yv[i] = yv;
                sy += sv * yv; yy += yv * yv;
            }
            a.x_acc[i] = a.x_t[i];
            a.g[i] = gt;
        }
        if (!s.init) {
            sy = lb_grid_sum(sy, a.partial, parity);
            yy = lb_grid_sum(yy, a.partial, parity);
            if (sy > 0.0) {                 // a pair is kept only with positive curvature
                s.rho[slot] = 1.0 / sy;
                s.gamma = sy / yy;
                s.head = (slot + 1) % kLbSlots;
                s.hist = min(s.hist + 1, kLbMemory);
            }
            ++s.iter;
        }
        s.init = 0;
        s.F = Ft;
        if (gtid == 0) a.energy[s.iter] = Ft;
        if (s.iter >= a.num_newton) s.done = 1;
        else need_dir = true;
    } else {
        ++s.halvings;
        s.t *= 0.5;
        if (s.halvings > kLbMaxHalvings) s.done = 1;
    }
    if (need_dir) {
        double gg = 0.0;
        for (long long i = gtid; i < N; i += gsize) { a.p[i] = a.g[i]; gg += a.g[i] * a.g[i]; }
        gg = lb_grid_sum(gg, a.partial, parity);
        if (gg == 0.0) {
            s.done = 1;
        } else {
            double alpha[kLbMemory];
            for (int h = 0; h < s.hist; ++h) {       // newest to oldest
                const int j = (s.head - 1 - h + 2 * kLbSlots) % kLbSlots;
                const double* Sv = a.S + (long long)j * N;
                const double* Yv = a.Y + (long long)j * N;
                double d = 0.0;
                for (long long i = gtid; i < N; i += gsize) d += Sv[i] * a.p[i];
                alpha[h] = s.rho[j] * lb_grid_sum(d, a.partial, parity);
                for (long long i = gtid; i < N; i += gsize) a.p[i] -= alpha[h] * Yv[i];
            }
            for (long long i = gtid; i < N; i += gsize) a.p[i] *= s.gamma;
            for (int h = s.hist - 1; h >= 0; --h) {  // oldest to newest
                const int j = (s.head - 1 - h + 2 * kLbSlots) % kLbSlots;
                const double* Sv = a.S + (long long)j * N;
                const double* Yv = a.Y + (long long)j * N;
                double d = 0.0;
                for (long long i = gtid; i < N; i += gsize) d += Yv[i] * a.p[i];
                const double beta = s.rho[j] * lb_grid_sum(d, a.partial, parity);
                for (long long i = gtid; i < N; i += gsize) a.p[i] += (alpha[h] - beta) * Sv[i];
            }
            double gp = 0.0;
            for (long long i = gtid; i < N; i += gsize) { a.p[i] = -a.p[i]; gp += a.g[i] * a.p[i]; }
            s.gtp = lb_grid_sum(gp, a.partial, parity);
            s.t = 1.0;
            s.halvings = 0;
            if (!(s.gtp < 0.0)) s.done = 1;          // not a descent direction: the line search cannot succeed
        }
    }
    while (!s.done) {                                // the trial point, inside the cube when there is one
        double outside = 0.0;
        if (a.cube) {
            for (long long i = gtid; i < N; i += gsize) {
                const double v = a.x_acc[i] + s.t * a.p[i];
                outside += (v < 0.0 || v > 1.0) ? 1.0 : 0.0;
            }
            outside = lb_grid_sum(outside, a.partial, parity);
        }
        if (outside == 0.0) {
            for (long long i = gtid; i < N; i += gsize) a.x_t[i] = a.x_acc[i] + s.t * a.p[i];
            break;
        }
        ++s.halvings;
        s.t *= 0.5;
        if (s.halvings > kLbMaxHalvings) s.done = 1;
    }
    if (gtid == 0) {
        *a.st = s;
        a.sync->done = s.done;
        a.sync->iter = s.iter;
    }
}

}  // namespace pcu
