// rvd.cuh -- the Voronoi diagram of seeds restricted to a triangle mesh, and its cells' moments (sample_mesh_lloyd of
// the reference, src/lloyd.cpp:357-401, which uses geogram's restricted Voronoi diagram).
//
// The cell of seed i is R_i = {y on the faces : |y - x_i|^2 <= |y - x_j|^2 for every x_j != x_i} (DESIGN.md §3,
// restricted cell).  It is computed in (face, seed) pairs, so that a coarse mesh with many seeds and a fine mesh with
// few seeds both keep the device busy:
//   rv_face_kernel     per face: its corners, centroid c_T and radius r_T = max |corner - c_T|; a face of zero area or
//                      with a corner out of range gets no radius (it meets no cell)
//   (k = 1 search)     d_T, the distance from c_T to its nearest seed
//   rv_ball_kernel     the candidate ball (c_T, rho_T), rho_T = (d_T + 2 r_T)(1 + kRvMargin): a seed whose cell meets T
//                      lies in it, because the distance to the nearest seed is 1-Lipschitz
//   (tree build)       the shared builder of meshquery.cuh over the balls (RvBall leaves)
//   rv_count_kernel    one thread per seed counts the balls that hold it (exact fp64 test), block scan of the counts
//   rv_tiles_kernel    one CTA: exclusive scan of the block totals, the pair total for the host
//   rv_emit_kernel     one thread per seed walks again and writes its pairs at its offset: pairs are grouped by seed,
//                      in tree order, with no sort
//   (voronoi.cuh)      every pair clipped as a polygon by the passes of the cube's cells (vor_cell with Poly3)
//   rv_reduce_kernel   each seed's run of pair moments summed in order into its (n, 5) row
// Nothing is summed with atomics, so results are bit-reproducible.
#pragma once
#include "common.cuh"
#include "meshquery.cuh"
#include "voronoi.cuh"

namespace pcu {

// Relative widening of the candidate radius: d_T, r_T and the pair test are each a few roundings from exact.
constexpr double kRvMargin = 1e-9;

// Face t: tri (9 doubles: a, b, c), centroid ((a + b) + c) / 3 and radius r_T, or NaN for a face that meets no cell
// (zero area, or a corner out of range: counted in *bad).
__global__ void __launch_bounds__(kThreads) rv_face_kernel(const double* __restrict__ v, long long nv, const void* __restrict__ f,
                                                           int fkind, long long m, double* __restrict__ tri, double* __restrict__ cen,
                                                           double* __restrict__ rad, unsigned long long* __restrict__ bad) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    double p[3][3];
    const bool ok = mq_corners<double>(v, nv, f, fkind, t, p[0], p[1], p[2]);
    if (!ok) {
        atomicAdd(bad, 1ull);
        for (int k = 0; k < 3; ++k) p[0][k] = p[1][k] = p[2][k] = 0.0;
    }
    double c[3], r2 = 0.0;
    for (int k = 0; k < 3; ++k) c[k] = ((p[0][k] + p[1][k]) + p[2][k]) / 3.0;
    for (int q = 0; q < 3; ++q) {
        const double dx = p[q][0] - c[0], dy = p[q][1] - c[1], dz = p[q][2] - c[2];
        r2 = fmax(r2, dx * dx + dy * dy + dz * dz);
    }
    for (int q = 0; q < 3; ++q)
        for (int k = 0; k < 3; ++k) tri[9 * t + 3 * q + k] = p[q][k];
    for (int k = 0; k < 3; ++k) cen[3 * t + k] = c[k];
    rad[t] = ok && face_area(p[0], p[1], p[2]) > 0.0 ? sqrt(r2) : __longlong_as_double(0x7ff8000000000000LL);
}

// The candidate balls (m, 4): centre c_T, radius (d_T + 2 r_T)(1 + kRvMargin); +inf when the search found no seed.
__global__ void __launch_bounds__(kThreads) rv_ball_kernel(const double* __restrict__ cen, const double* __restrict__ rad,
                                                           const double* __restrict__ d2, const long long* __restrict__ idx,
                                                           long long m, double* __restrict__ balls) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    const double r = rad[t];
    const double rho = idx[t] < 0 ? __longlong_as_double(0x7ff0000000000000LL) : (sqrt(d2[t]) + 2.0 * r) * (1.0 + kRvMargin);
    for (int k = 0; k < 3; ++k) balls[4 * t + k] = cen[3 * t + k];
    balls[4 * t + 3] = r >= 0.0 ? rho : r;   // NaN stays NaN
}

// Every face whose ball holds x (|x - c|^2 <= rho^2 in fp64), in tree order: visit(face).  The walk enters a node's
// child when x's fp32 enclosure meets the child's box (boxes are rounded outward, so no ball holding x is skipped).
template <typename F>
__device__ __forceinline__ void rv_walk(const double* x, long long valid, const MqNode* __restrict__ nodes,
                                        const RvBall* __restrict__ leaves, const int* __restrict__ ids, F&& visit) {
    if (valid < 1) return;
    float pl[3], ph[3];
    for (int k = 0; k < 3; ++k) { pl[k] = __double2float_rd(x[k]); ph[k] = __double2float_ru(x[k]); }
    auto test = [&](int leaf) {
        const RvBall b = leaves[leaf];
        const double dx = x[0] - b.c[0], dy = x[1] - b.c[1], dz = x[2] - b.c[2];
        if ((dx * dx + dy * dy) + dz * dz <= b.r * b.r) visit(ids[leaf]);
    };
    if (valid == 1) { test(0); return; }
    auto meets = [&](const float* lo, const float* hi) {
        return pl[0] <= hi[0] && ph[0] >= lo[0] && pl[1] <= hi[1] && ph[1] >= lo[1] && pl[2] <= hi[2] && ph[2] >= lo[2];
    };
    int stack[kMqStack];
    int sp = 0, node = 0;
    while (true) {
        const float4* np_ = reinterpret_cast<const float4*>(nodes + node);
        const float4 q0 = __ldg(np_), q1 = __ldg(np_ + 1), q2 = __ldg(np_ + 2), q3 = __ldg(np_ + 3);
        const float lo0[3] = {q0.x, q0.y, q0.z}, hi0[3] = {q0.w, q1.x, q1.y};
        const float lo1[3] = {q1.z, q1.w, q2.x}, hi1[3] = {q2.y, q2.z, q2.w};
        const int c0 = __float_as_int(q3.x), c1 = __float_as_int(q3.y);
        bool k0 = meets(lo0, hi0), k1 = meets(lo1, hi1);
        if (k0 && c0 < 0) { test(~c0); k0 = false; }
        if (k1 && c1 < 0) { test(~c1); k1 = false; }
        if (k0 && k1) { stack[sp++] = c1; node = c0; continue; }
        if (k0) { node = c0; continue; }
        if (k1) { node = c1; continue; }
        if (sp == 0) break;
        node = stack[--sp];
    }
}

// Seed i's pair count; local[i] = its exclusive prefix within the block, tile_sum[block] = the block's total.
__global__ void __launch_bounds__(kThreads) rv_count_kernel(const double* __restrict__ x, long long n, long long m,
                                                            const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                            const RvBall* __restrict__ leaves, const int* __restrict__ ids,
                                                            unsigned long long* __restrict__ local,
                                                            unsigned long long* __restrict__ tile_sum) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long cnt = 0;
    if (i < n) rv_walk(x + 3 * i, m - (long long)sc->bad, nodes, leaves, ids, [&](int) { ++cnt; });
    unsigned long long total;
    const unsigned long long ex = block_exclusive_scan<kThreads, unsigned long long>(cnt, &total);
    if (i < n) local[i] = ex;
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// One CTA: the block totals scanned in place into the blocks' first pairs; the pair total into sync->count.
__global__ void __launch_bounds__(1024) rv_tiles_kernel(unsigned long long* __restrict__ tile_sum, long long tiles,
                                                        VorSync* __restrict__ sync) {
    const unsigned long long total = block_scan_rounds<1024, unsigned long long>(
        (unsigned)tiles, [&](unsigned b) { return tile_sum[b]; },
        [&](unsigned b, unsigned long long ex, unsigned long long) { tile_sum[b] = ex; });
    if (threadIdx.x == 0) sync->count = (long long)total;
}

// Seed i's pairs (seed, face) from its first pair on, in the order of rv_count_kernel's walk; start[i] = its first.
__global__ void __launch_bounds__(kThreads) rv_emit_kernel(const double* __restrict__ x, long long n, long long m,
                                                           const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                           const RvBall* __restrict__ leaves, const int* __restrict__ ids,
                                                           const unsigned long long* __restrict__ local,
                                                           const unsigned long long* __restrict__ tile_off,
                                                           long long* __restrict__ start, int* __restrict__ pair_seed,
                                                           int* __restrict__ pair_face) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    long long at = (long long)(tile_off[blockIdx.x] + local[i]);
    start[i] = at;
    rv_walk(x + 3 * i, m - (long long)sc->bad, nodes, leaves, ids, [&](int face) {
        pair_seed[at] = (int)i;
        pair_face[at] = face;
        ++at;
    });
}

// Row i of the cells' moments: the sum, in pair order, of seed i's pairs [start[i], start[i + 1]) (the last ends at
// `pairs`).
__global__ void __launch_bounds__(kThreads) rv_reduce_kernel(const long long* __restrict__ start, long long n, long long pairs,
                                                             const double* __restrict__ pair_mom, double* __restrict__ mom) {
    grid_dependency_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long a = start[i], b = i + 1 < n ? start[i + 1] : pairs;
    double s[kVorMoments] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (long long p = a; p < b; ++p)
        for (int q = 0; q < kVorMoments; ++q) s[q] += pair_mom[p * kVorMoments + q];
    for (int q = 0; q < kVorMoments; ++q) mom[i * kVorMoments + q] = s[q];
}

}  // namespace pcu
