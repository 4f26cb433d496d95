// watertight.cuh -- watertight manifold remeshing of a triangle mesh (make_mesh_watertight; the reference's
// src/manifold.cpp, after Huang et al., "Robust Watertight Manifold Surface Generation", arXiv 1802.01698).  The result
// is defined in DESIGN.md §3.  Pipeline, on a cubic grid of 2^d voxels per side (voxel o = (i 2^d + j) 2^d + k):
//   wt_bounds_kernel    per-axis min / max of v in fp64 and the count of non-finite coordinates (one sync)
//   depth search        per depth d = 3 .. 10 the voxelizer's counting pass (vx_test_kernel<kVxCount>, an upper
//                       bound of the occupied voxels), then where that bound reaches the resolution its grid pass
//                       (kVxGrid): occupancy bytes and the exact occupied count (one sync each)
//   exterior            ff_tile_kernel / ff_cross_kernel of the flood fill on the byte grid from voxel 0, then
//                       wt_exterior_kernel marks the seed's component kWtExterior
//   wt_count_kernel     per voxel: crossing lattice edges towards +x, +y, +z, and the case of the cube whose lowest
//                       corner it is (corner above = exterior); vertex and face counts per CTA tile; mc_tiles_kernel
//                       scans the tiles (one sync for the totals)
//   wt_verts_kernel     vertex ids (tile offset + block scan) into the int32 grid P, the vertices' positions
//   wt_faces_kernel     faces of every cube from kMcTrisManifold, their corners' ids read back from P
//   projection rounds   mq_query_kernel on the input's fp64 tree, wt_propose_kernel, then wt_flip_kernel passes
//                       until no face is flipped (one sync per pass) and wt_commit_kernel
// Dense scratch: the byte grid and P, 5 bytes per voxel.
#pragma once
#include "common.cuh"
#include "mc_tables.h"
#include "meshquery.cuh"
#include "sparse_voxels.cuh"
#include "union_find.cuh"
#include "voxelize.cuh"

namespace pcu {

constexpr int kWtMinDepth = 3, kWtMaxDepth = 10;
constexpr unsigned char kWtExterior = 2;   // byte grid: 0 empty, 1 occupied, kWtExterior empty and reached from voxel 0

// What the host reads of the bounds pass: ordered-int images of the per-axis min and max, non-finite coordinates.
struct WtBounds { long long lo[3], hi[3]; unsigned long long bad; };

__device__ __forceinline__ long long wt_ord(double x) {
    const long long b = __double_as_longlong(x);
    return b >= 0 ? b : b ^ 0x7fffffffffffffffll;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) wt_bounds_kernel(const T* __restrict__ v, long long nv, WtBounds* __restrict__ out) {
    double lo[3], hi[3];
    unsigned bad = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) { lo[k] = __longlong_as_double(0x7ff0000000000000ll); hi[k] = -lo[k]; }
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nv; i += (long long)gridDim.x * kThreads) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double x = (double)v[3 * i + k];
            if (!isfinite(x)) { ++bad; continue; }
            lo[k] = fmin(lo[k], x);
            hi[k] = fmax(hi[k], x);
        }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, sh);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            lo[k] = fmin(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], sh));
            hi[k] = fmax(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], sh));
        }
    }
    if ((threadIdx.x & 31) != 0) return;
    if (bad) atomicAdd(&out->bad, (unsigned long long)bad);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        atomicMin(&out->lo[k], wt_ord(lo[k]));
        atomicMax(&out->hi[k], wt_ord(hi[k]));
    }
}

// The exterior: the empty voxels in voxel 0's component (its root is 0, the smallest index).
__global__ void __launch_bounds__(kThreads) wt_exterior_kernel(unsigned char* __restrict__ grid, long long n, int* __restrict__ P) {
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (o >= n || grid[o] != 0) return;
    if (uf_find(P, (int)o) == 0) grid[o] = kWtExterior;
}

__device__ __forceinline__ bool wt_ext(const unsigned char* __restrict__ g, long long o) { return __ldg(g + o) == kWtExterior; }
// Bit `a` of corner k of a cube (corners numbered as in tools/mc_tables.py: (0,0,0) (1,0,0) (1,1,0) (0,1,0) (0,0,1) ...).
__host__ __device__ constexpr int wt_corner_bit(int k, int a) { return a == 0 ? ((k + 1) >> 1) & 1 : a == 1 ? (k >> 1) & 1 : k >> 2; }

// Voxel o's crossing lattice edges (bit a: the edge to o + e_a joins an exterior and a non-exterior centre), and the
// case of the cube whose lowest corner is o (0 when o lies on the grid's last layer of some axis).
struct WtVoxel { unsigned vmask, cs; };
__device__ __forceinline__ WtVoxel wt_classify(const unsigned char* __restrict__ g, int lg, long long o) {
    const long long N = 1ll << lg, st[3] = {N * N, N, 1};
    const long long c[3] = {o >> (2 * lg), (o >> lg) & (N - 1), o & (N - 1)};
    const bool e0 = wt_ext(g, o);
    WtVoxel r = {0u, 0u};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (c[a] + 1 < N && wt_ext(g, o + st[a]) != e0) r.vmask |= 1u << a;
    if (c[0] + 1 < N && c[1] + 1 < N && c[2] + 1 < N) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            r.cs |= (unsigned)wt_ext(g, o + wt_corner_bit(k, 0) * st[0] + wt_corner_bit(k, 1) * st[1] + wt_corner_bit(k, 2) * st[2]) << k;
    }
    return r;
}
// vertices in bits 0-15, faces in bits 16-31 (a CTA holds at most 3 * 256 and 5 * 256)
__device__ __forceinline__ unsigned wt_packed(const WtVoxel& x) { return (unsigned)__popc(x.vmask) | (unsigned)__ldg(&kMcTriCount[x.cs]) << 16; }

__global__ void __launch_bounds__(kThreads) wt_count_kernel(const unsigned char* __restrict__ g, int lg, long long n, unsigned* __restrict__ tile_sum) {
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    const unsigned mine = o < n ? wt_packed(wt_classify(g, lg, o)) : 0u;
    unsigned total;
    block_exclusive_scan<kThreads>(mine, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// This thread's voxel, its first vertex and its first face (block-wide: every thread of the CTA calls it).
struct WtOffsets { WtVoxel x; unsigned long long v0, f0; };
__device__ __forceinline__ WtOffsets wt_offsets(const unsigned char* __restrict__ g, int lg, long long n, const unsigned long long* __restrict__ tile_v0,
                                                const unsigned long long* __restrict__ tile_f0) {
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    WtOffsets r;
    r.x = o < n ? wt_classify(g, lg, o) : WtVoxel{0u, 0u};
    unsigned total;
    const unsigned ex = block_exclusive_scan<kThreads>(wt_packed(r.x), &total);
    r.v0 = tile_v0[blockIdx.x] + (ex & 0xffffu);
    r.f0 = tile_f0[blockIdx.x] + (ex >> 16);
    return r;
}

// Placement of the lattice: voxel centre (i, j, k) is o + (i + 1/2) s per axis.
struct WtPlace { double o[3], s; };

// P[o] = the id of voxel o's first vertex; vertex (o, a) at o_k + (c_k + 1/2 + [k == a] / 2) s per axis, each operation
// rounded.  The host has checked that the ids fit int32.
__global__ void __launch_bounds__(kThreads) wt_verts_kernel(const unsigned char* __restrict__ g, int lg, long long n,
                                                            const unsigned long long* __restrict__ tile_v0,
                                                            const unsigned long long* __restrict__ tile_f0, const __grid_constant__ WtPlace pl,
                                                            int* __restrict__ P, double* __restrict__ x) {
    const WtOffsets w = wt_offsets(g, lg, n, tile_v0, tile_f0);
    if (w.x.vmask == 0u) return;
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x, N = 1ll << lg;
    const long long c[3] = {o >> (2 * lg), (o >> lg) & (N - 1), o & (N - 1)};
    P[o] = (int)w.v0;
    unsigned long long id = w.v0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!(w.x.vmask >> a & 1u)) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) x[3 * id + k] = __dadd_rn(pl.o[k], __dmul_rn((double)c[k] + (k == a ? 1.0 : 0.5), pl.s));
        ++id;
    }
}

// The id of the vertex on the lattice edge from voxel q along axis a (the edge crosses).
__device__ __forceinline__ int wt_vertex_id(const unsigned char* __restrict__ g, int lg, const int* __restrict__ P, long long q, int a) {
    const long long N = 1ll << lg, st[3] = {N * N, N, 1};
    const long long c[3] = {q >> (2 * lg), (q >> lg) & (N - 1), q & (N - 1)};
    const bool e0 = wt_ext(g, q);
    int id = __ldg(P + q);
    for (int b = 0; b < a; ++b) id += (c[b] + 1 < N && wt_ext(g, q + st[b]) != e0) ? 1 : 0;
    return id;
}

// The faces of every cube, cube by cube in voxel order, each case's triangles in kMcTrisManifold's order.
__global__ void __launch_bounds__(kThreads) wt_faces_kernel(const unsigned char* __restrict__ g, int lg, long long n,
                                                            const unsigned long long* __restrict__ tile_v0,
                                                            const unsigned long long* __restrict__ tile_f0, const int* __restrict__ P,
                                                            int* __restrict__ F) {
    const WtOffsets w = wt_offsets(g, lg, n, tile_v0, tile_f0);
    const int nt = __ldg(&kMcTriCount[w.x.cs]);
    if (nt == 0) return;
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x, N = 1ll << lg, st[3] = {N * N, N, 1};
    const unsigned char* tri = kMcTrisManifold[w.x.cs];
#pragma unroll 1
    for (int j = 0; j < 3 * nt; ++j) {
        const int e = __ldg(tri + j), ca = mc_edge_corner(e, 0), cb = mc_edge_corner(e, 1);
        int a = 0;
        while (wt_corner_bit(ca, a) == wt_corner_bit(cb, a)) ++a;
        const int lo = wt_corner_bit(ca, a) < wt_corner_bit(cb, a) ? ca : cb;
        const long long q = o + wt_corner_bit(lo, 0) * st[0] + wt_corner_bit(lo, 1) * st[1] + wt_corner_bit(lo, 2) * st[2];
        F[3 * w.f0 + j] = wt_vertex_id(g, lg, P, q, a);
    }
}

// ---- projection rounds -------------------------------------------------------------------------------------------
// f32 inputs: the fp64 copy of v the tree and the closest points are computed on.
template <typename T>
__global__ void __launch_bounds__(kThreads) wt_widen_kernel(const T* __restrict__ v, long long n3, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i < n3) out[i] = (double)v[i];
}

// The pre-projection positions x0 = x, and every step alpha = 1.
__global__ void __launch_bounds__(kThreads) wt_start_kernel(const double* __restrict__ x, long long n, double* __restrict__ x0,
                                                            double* __restrict__ alpha) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) x0[3 * i + k] = x[3 * i + k];
    alpha[i] = 1.0;
}

// t = (b0 a + b1 b) + b2 c per axis on the closest face, y = x + alpha (t - x); every operation rounded.
__global__ void __launch_bounds__(kThreads) wt_propose_kernel(const double* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                              const long long* __restrict__ fidx, const double* __restrict__ bc,
                                                              const double* __restrict__ x, const double* __restrict__ alpha, long long n,
                                                              double* __restrict__ y) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    double a[3], b[3], c[3];
    mq_corners<double>(v, nv, f, fkind, fidx[i], a, b, c);
    const double b0 = bc[3 * i], b1 = bc[3 * i + 1], b2 = bc[3 * i + 2], al = alpha[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double t = __dadd_rn(__dadd_rn(__dmul_rn(b0, a[k]), __dmul_rn(b1, b[k])), __dmul_rn(b2, c[k]));
        y[3 * i + k] = __dadd_rn(x[3 * i + k], __dmul_rn(al, __dsub_rn(t, x[3 * i + k])));
    }
}

// (b - a) x (c - a), every operation rounded
__device__ __forceinline__ void wt_normal(const double a[3], const double b[3], const double c[3], double n[3]) {
    const double u[3] = {__dsub_rn(b[0], a[0]), __dsub_rn(b[1], a[1]), __dsub_rn(b[2], a[2])};
    const double w[3] = {__dsub_rn(c[0], a[0]), __dsub_rn(c[1], a[1]), __dsub_rn(c[2], a[2])};
    n[0] = __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1]));
    n[1] = __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2]));
    n[2] = __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]));
}

// Pass `pass` (1, 2, ...) of a round: a vertex reverted by an earlier pass (0 < rev < pass) sits at x, every other at y.
// A face whose normal's dot product with its pre-projection normal, (n0x nx + n0y ny) + n0z nz, is <= 0 is flipped:
// its vertices not yet reverted get rev = pass, and *flipped counts it.  Within a pass every face sees the same set.
__global__ void __launch_bounds__(kThreads) wt_flip_kernel(const int* __restrict__ F, long long nf, const double* __restrict__ x0,
                                                           const double* __restrict__ x, const double* __restrict__ y, int* __restrict__ rev,
                                                           int pass, unsigned long long* __restrict__ flipped) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool flip = false;
    if (t < nf) {
        int id[3];
        double p[3][3], q[3][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            id[c] = F[3 * t + c];
            const volatile int* r = rev;
            const int rv = r[id[c]];
            const double* src = (rv != 0 && rv < pass) ? x : y;
#pragma unroll
            for (int k = 0; k < 3; ++k) { p[c][k] = src[3ll * id[c] + k]; q[c][k] = __ldg(x0 + 3ll * id[c] + k); }
        }
        double n[3], n0[3];
        wt_normal(p[0], p[1], p[2], n);
        wt_normal(q[0], q[1], q[2], n0);
        flip = !(__dadd_rn(__dadd_rn(__dmul_rn(n0[0], n[0]), __dmul_rn(n0[1], n[1])), __dmul_rn(n0[2], n[2])) > 0.0);
        if (flip) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                volatile int* r = rev;
                if (r[id[c]] == 0) r[id[c]] = pass;
            }
        }
    }
    const unsigned count = __syncthreads_count(flip);
    if (threadIdx.x == 0 && count) atomicAdd(flipped, (unsigned long long)count);
}

// The round's positions: reverted vertices stay at x and halve their step, the others move to y.
__global__ void __launch_bounds__(kThreads) wt_commit_kernel(const double* __restrict__ y, const int* __restrict__ rev, long long n,
                                                             double* __restrict__ x, double* __restrict__ alpha) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    if (rev[i] != 0) { alpha[i] = __dmul_rn(alpha[i], 0.5); return; }
#pragma unroll
    for (int k = 0; k < 3; ++k) x[3 * i + k] = y[3 * i + k];
}

// vw = x in T, fw = F widened to the index kind's width.
template <typename T>
__global__ void __launch_bounds__(kThreads) wt_emit_kernel(const double* __restrict__ x, long long nv, const int* __restrict__ F, long long nf,
                                                           int wide, T* __restrict__ out_v, void* __restrict__ out_f) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t < 3 * nv) out_v[t] = (T)x[t];
    if (t < 3 * nf) {
        if (wide) reinterpret_cast<long long*>(out_f)[t] = F[t];
        else reinterpret_cast<int*>(out_f)[t] = F[t];
    }
}

}  // namespace pcu
