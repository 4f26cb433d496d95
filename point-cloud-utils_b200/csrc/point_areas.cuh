// point_areas.cuh -- areas of the points of an oriented cloud from their neighbour rows (estimate_point_cloud_areas;
// the reference's src/point_areas.cpp, libigl's igl::copyleft::cgal::point_areas).  The result is defined in
// DESIGN.md §3: for row r of the (n, k) index array, the neighbours whose normals face the centre's (a strictly positive
// dot product), projected onto their PCA plane (PlaneFit of plane_fit.h); the star of the centre c = q_0 in the 2-D
// Delaunay triangulation of the projected points, walked one triangle at a time from the nearest neighbour; and Meyer et
// al.'s mixed Voronoi area of c summed over that star.  Everything is fp64 and rounded once to T.
//
// One warp per row.  The kept points are staged in shared memory in column order (a ballot per 32 columns), so rows
// up to kAreaMaxK columns run the same code: lane l owns the kept positions l, l + 32, ...  Every sum is a per-lane
// sum in position order followed by an xor butterfly, so each lane ends with the same bits and the result does not
// depend on scheduling.  Each walk step is a warp arg-min over (circumcentre parameter, position).
#pragma once
#include "common.cuh"
#include "plane_fit.h"

namespace pcu {

constexpr int kAreaWarps = 4;     // rows per CTA
constexpr int kAreaMaxK = 256;    // the widest index row

// Dynamic shared memory of one CTA for rows of up to `cap` columns (a multiple of 32): per warp, the 2-D offsets from
// the centre (cap x 2 doubles), then the kept points in T (cap x 3).
template <typename T>
constexpr size_t point_area_smem(int cap) { return (size_t)kAreaWarps * cap * (2 * sizeof(double) + 3 * sizeof(T)); }

__device__ __forceinline__ double area_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// (key, position) lexicographic minimum over the warp; every lane returns the same pair.
__device__ __forceinline__ void area_warp_argmin(double& key, int& pos) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double k2 = __shfl_xor_sync(0xffffffffu, key, o);
        const int p2 = __shfl_xor_sync(0xffffffffu, pos, o);
        if (k2 < key || (k2 == key && p2 < pos)) { key = k2; pos = p2; }
    }
}

__device__ __forceinline__ double area_cross(double ax, double ay, double bx, double by) {
    return __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));   // no FMA: a x a is exactly 0
}
__device__ __forceinline__ double area_dot(double ax, double ay, double bx, double by) {
    return __dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by));
}

// Meyer et al.'s mixed area at X of the counter-clockwise triangle (X, Y, Z), from y = Y - X and z = Z - X.
__device__ __forceinline__ double mixed_area(double yx, double yy, double zx, double zy) {
    const double cr = area_cross(yx, yy, zx, zy);
    const double dX = area_dot(yx, yy, zx, zy);
    const double dY = area_dot(-yx, -yy, __dsub_rn(zx, yx), __dsub_rn(zy, yy));
    const double dZ = area_dot(-zx, -zy, __dsub_rn(yx, zx), __dsub_rn(yy, zy));
    if (dX >= 0.0 && dY >= 0.0 && dZ >= 0.0)
        return __ddiv_rn(__dadd_rn(__dmul_rn(area_dot(yx, yy, yx, yy), dZ), __dmul_rn(area_dot(zx, zy, zx, zy), dY)), __dmul_rn(8.0, cr));
    return dX < 0.0 ? __ddiv_rn(cr, 4.0) : __ddiv_rn(cr, 8.0);
}

// grid: ceil(n / kAreaWarps) CTAs of kAreaWarps warps, point_area_smem<T>(cap) bytes of dynamic shared memory,
// cap = k rounded up to 32.  idx: (n, k) of index kind `kind`.  *bad (zeroed by the caller) counts the entries outside
// [0, n); they are left out of their row.
template <typename T>
__global__ void __launch_bounds__(kAreaWarps * 32) point_areas_kernel(const T* __restrict__ p, const T* __restrict__ nrm, long long n,
                                                                      const void* __restrict__ idx, int k, int kind, int cap,
                                                                      T* __restrict__ out, unsigned long long* __restrict__ bad) {
    grid_dependency_wait();
    extern __shared__ double area_smem[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long row = (long long)blockIdx.x * kAreaWarps + w;
    if (row >= n) return;   // the whole warp
    double* dq = area_smem + (size_t)w * cap * 2;
    T* xs = reinterpret_cast<T*>(area_smem + (size_t)kAreaWarps * cap * 2) + (size_t)w * cap * 3;

    // 1. neighbours: column j is kept when n0 . n_j > 0 (fp64, left to right); K in column order
    const long long i0 = k > 0 ? load_index(idx, row * k, kind, n, false) : -1;
    double n0x = 0.0, n0y = 0.0, n0z = 0.0;
    if (i0 >= 0) { n0x = (double)nrm[3 * i0]; n0y = (double)nrm[3 * i0 + 1]; n0z = (double)nrm[3 * i0 + 2]; }
    int m = 0;
    bool centre_kept = false;
    unsigned nbad = 0;
    for (int base = 0; base < k; base += 32) {
        const int j = base + lane;
        long long pj = -1;
        bool keep = false;
        if (j < k) {
            pj = load_index(idx, row * k + j, kind, n, false);
            if (pj < 0) {
                ++nbad;
            } else {
                const double d = __dadd_rn(__dadd_rn(__dmul_rn(n0x, (double)nrm[3 * pj]), __dmul_rn(n0y, (double)nrm[3 * pj + 1])),
                                           __dmul_rn(n0z, (double)nrm[3 * pj + 2]));
                keep = d > 0.0;
            }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (base == 0) centre_kept = mask & 1u;
        if (keep) {
            const int s = m + __popc(mask & ((1u << lane) - 1u));
            xs[3 * s] = p[3 * pj]; xs[3 * s + 1] = p[3 * pj + 1]; xs[3 * s + 2] = p[3 * pj + 2];
        }
        m += __popc(mask);
    }
    nbad = __reduce_add_sync(0xffffffffu, nbad);
    if (lane == 0 && nbad) atomicAdd(bad, (unsigned long long)nbad);
    if (!centre_kept || m <= 2) {
        if (lane == 0) out[row] = (T)0;
        return;
    }
    __syncwarp();

    // 2. plane: mean, then PlaneFit over the offsets; q = the offsets on the basis columns other than the normal's
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int s = lane; s < m; s += 32) {
        sx = __dadd_rn(sx, (double)xs[3 * s]); sy = __dadd_rn(sy, (double)xs[3 * s + 1]); sz = __dadd_rn(sz, (double)xs[3 * s + 2]);
    }
    const double mx = __ddiv_rn(area_warp_sum(sx), (double)m), my = __ddiv_rn(area_warp_sum(sy), (double)m),
                 mz = __ddiv_rn(area_warp_sum(sz), (double)m);
    auto offset = [&](int s, double& ox, double& oy, double& oz) {
        ox = __dsub_rn((double)xs[3 * s], mx); oy = __dsub_rn((double)xs[3 * s + 1], my); oz = __dsub_rn((double)xs[3 * s + 2], mz);
    };
    double big = 0.0;
    for (int s = lane; s < m; s += 32) {
        double ox, oy, oz;
        offset(s, ox, oy, oz);
        big = fmax(big, fmax(fabs(ox), fmax(fabs(oy), fabs(oz))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) big = fmax(big, __shfl_xor_sync(0xffffffffu, big, o));
    PlaneFit fit(pow2_scale(big));
    do {
        for (int s = lane; s < m; s += 32) {
            double ox, oy, oz;
            offset(s, ox, oy, oz);
            fit.add(ox, oy, oz);
        }
        fit.s00 = area_warp_sum(fit.s00); fit.s01 = area_warp_sum(fit.s01); fit.s02 = area_warp_sum(fit.s02);
        fit.s11 = area_warp_sum(fit.s11); fit.s12 = area_warp_sum(fit.s12); fit.s22 = area_warp_sum(fit.s22);
    } while (fit.solve());
    // the two columns in index order (selects rather than a run-time index keep the basis in registers)
    const int ax = fit.normal_axis();
    const double ux = ax == 0 ? fit.v[0][1] : fit.v[0][0], uy = ax == 0 ? fit.v[1][1] : fit.v[1][0], uz = ax == 0 ? fit.v[2][1] : fit.v[2][0];
    const double wx = ax == 2 ? fit.v[0][1] : fit.v[0][2], wy = ax == 2 ? fit.v[1][1] : fit.v[1][2], wz = ax == 2 ? fit.v[2][1] : fit.v[2][2];
    auto project = [&](int s, double& qx, double& qy) {
        double ox, oy, oz;
        offset(s, ox, oy, oz);
        qx = __dadd_rn(__dadd_rn(__dmul_rn(ox, ux), __dmul_rn(oy, uy)), __dmul_rn(oz, uz));
        qy = __dadd_rn(__dadd_rn(__dmul_rn(ox, wx), __dmul_rn(oy, wy)), __dmul_rn(oz, wz));
    };
    double cx, cy;
    project(0, cx, cy);
    // 3. the star: candidates are the positions whose offset from c is not (0, 0) (position 0 is c); the walk starts at
    // the nearest
    double dkey = Real<double>::inf();
    int j0 = INT_MAX;
    for (int s = lane; s < m; s += 32) {
        double qx, qy;
        project(s, qx, qy);
        const double dx = __dsub_rn(qx, cx), dy = __dsub_rn(qy, cy);
        dq[2 * s] = dx; dq[2 * s + 1] = dy;
        const double d2 = area_dot(dx, dy, dx, dy);
        if (!(dx == 0.0 && dy == 0.0) && (d2 < dkey || (d2 == dkey && s < j0))) { dkey = d2; j0 = s; }
    }
    area_warp_argmin(dkey, j0);
    double sum = 0.0;
    if (j0 != INT_MAX) {
        __syncwarp();
        bool closed = false;
        for (int side = 1; side >= -1 && !closed; side -= 2) {   // left walk, then (when it did not close) right walk
            int cur = j0;
            for (int step = 0; step < m; ++step) {
                const double ax_ = dq[2 * cur], ay_ = dq[2 * cur + 1];
                double key = Real<double>::inf();
                int r = INT_MAX;
                for (int s = lane; s < m; s += 32) {
                    const double bx = dq[2 * s], by = dq[2 * s + 1];
                    if (bx == 0.0 && by == 0.0) continue;
                    const double o = side > 0 ? area_cross(ax_, ay_, bx, by) : -area_cross(ax_, ay_, bx, by);
                    if (!(o > 0.0)) continue;
                    // the circumcentre of (c, q_cur, q_s) is c + a / 2 + t perp(a) with t = (|b|^2 - a . b) / (2 a x b)
                    const double t = __ddiv_rn(__dsub_rn(area_dot(bx, by, bx, by), area_dot(ax_, ay_, bx, by)), __dmul_rn(2.0, o));
                    if (t < key || (t == key && s < r)) { key = t; r = s; }
                }
                area_warp_argmin(key, r);
                if (r == INT_MAX) break;
                const int y = side > 0 ? cur : r, z = side > 0 ? r : cur;
                sum = __dadd_rn(sum, mixed_area(dq[2 * y], dq[2 * y + 1], dq[2 * z], dq[2 * z + 1]));
                cur = r;
                if (r == j0) { closed = true; break; }
            }
        }
    }
    if (lane == 0) out[row] = (T)sum;
}

}  // namespace pcu
