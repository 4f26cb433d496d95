// normals.cuh -- point-cloud normals from k nearest neighbours (SURVEY.md 8f, row N1).
//
// Replaces estimate_local_normal_knn + estimate_normals of the reference
// (src/point_cloud_normals.cpp:115-173, :175-300; binding :375-411): for every point, the k nearest points of
// the SAME cloud (the point itself included, as nanoflann's knnSearch returns it), the plane fitted to them
// and, optionally, orientation towards / filtering by a per-point view direction.
//
// The neighbour search is the exact top-k path of this library (topk.cuh + tie replay), so the neighbour SETS
// are the reference's, bit for bit.  The plane fit is where parity is a tolerance: the reference takes the
// right singular vector of the smallest singular value of the (k, 3) matrix of neighbour offsets from Eigen's
// JacobiSVD in double precision (Eigen is fetched at build time and is not in the reference tree); here it is
// PlaneFit of plane_fit.h: the offsets scaled by a power of two, the scatter matrix diagonalised by Jacobi
// rotations and refined on the offsets rotated into its eigenbasis, to the SVD's accuracy u s1 / (s2 - s3) --
// the same vector up to rounding (and up to sign: without view directions the reference's sign is whatever its SVD
// happens to return).  Fewer than 3 neighbours give the zero vector, all-zero offsets give (0, 0, 1).
//
// The ball walk below also serves the ball mode of mesh_principal_curvatures (curv_ball_kernel, with the rules of
// curvature.cuh).
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "plane_fit.h"
#include "curvature.cuh"

namespace pcu {

// Orientation towards / filtering by the view direction (:160-171 and :103-112, the same code in both estimators).
__device__ __forceinline__ bool orient_by_view(double (&nrm)[3], double vx, double vy, double vz, double drop_angle_threshold) {
    const double d = nrm[0] * vx + nrm[1] * vy + nrm[2] * vz;
    const double sgn = (double)((0.0 < d) - (d < 0.0));       // sign(): 0 when the dot product is 0 (:21-23)
    nrm[0] *= sgn; nrm[1] *= sgn; nrm[2] *= sgn;
    const double angle = acos(nrm[0] * vx + nrm[1] * vy + nrm[2] * vz);
    if (angle > drop_angle_threshold) { nrm[0] = nrm[1] = nrm[2] = 0.0; return false; }
    return true;
}

// One thread per point.  idx: (n, k) neighbour rows from the k-NN call (-1 padded when the cloud has fewer than k
// points: such points are dropped, src/point_cloud_normals.cpp:139-142).  view_dirs: (n, 3) or null.
// normals: (n, 3) dense, written for every point; keep: (n) 1 = the reference would return this point.
template <typename T>
__global__ void __launch_bounds__(kThreads) normals_knn_kernel(const T* __restrict__ points, long long n,
                                                               const long long* __restrict__ idx, int k,
                                                               const T* __restrict__ view_dirs, double drop_angle_threshold,
                                                               T* __restrict__ normals, unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long* row = idx + i * k;
    bool ok = row[k - 1] >= 0;
    double nrm[3] = {0.0, 0.0, 0.0};
    if (ok) {
        using R = Real<T>;
        const T qx = points[3 * i], qy = points[3 * i + 1], qz = points[3 * i + 2];
        // the reference subtracts in the cloud's precision and widens the difference (:150-154)
        auto offsets = [&](auto&& f) {
            for (int j = 0; j < k; ++j) {
                const long long p = row[j];
                f((double)R::sub(points[3 * p], qx), (double)R::sub(points[3 * p + 1], qy), (double)R::sub(points[3 * p + 2], qz));
            }
        };
        double big = 0.0;
        offsets([&](double x, double y, double z) { big = fmax(big, fmax(fabs(x), fmax(fabs(y), fabs(z)))); });
        PlaneFit fit(pow2_scale(big));
        do offsets([&](double x, double y, double z) { fit.add(x, y, z); }); while (fit.solve());
        fit.normal(k, nrm);
        if (view_dirs != nullptr) {
            const double vx = (double)view_dirs[3 * i], vy = (double)view_dirs[3 * i + 1], vz = (double)view_dirs[3 * i + 2];
            ok = orient_by_view(nrm, vx, vy, vz, drop_angle_threshold);   // :160-171
        }
    }
    normals[3 * i] = (T)nrm[0]; normals[3 * i + 1] = (T)nrm[1]; normals[3 * i + 2] = (T)nrm[2];
    keep[i] = ok ? 1 : 0;
}

// ---- normals from all points in a ball (estimate_local_normal_rbf, src/point_cloud_normals.cpp:48-113; binding
// :303-370) ------------------------------------------------------------------------------------------------------
// The reference hands `ball_radius` to nanoflann's radiusSearch, whose radius is in the metric's units -- SQUARED
// distance for L2_Simple (nanoflann.hpp RadiusResultSet::addPoint: `if (dist < radius)`) -- so the neighbourhood is
//     { j : d2(p_i, p_j) < (T)ball_radius }        (the point itself included),
// while the weight function receives the true distance: w = wendland(sqrt(d2), ball_radius).  Both are reproduced as
// they are.  The neighbourhood test uses the reference-rounded d2 of common.cuh, so neighbour SETS are exact.
//
// max_pts_per_ball > 0: the reference shuffles the neighbours with std::shuffle(default_random_engine(rand())) and
// keeps the first max_pts_per_ball -- a uniformly random subset that depends on the C library's rand() state and on
// the thread that happens to process the point.  Here: a uniformly random subset of the same size by selection
// sampling (Knuth 3.4.2 S) over the neighbours in cell order, driven by a counter-based hash of (seed, row, position):
// deterministic for a given seed, the same distribution, not the same subset.
struct BallParams {
    double radius;
    double drop_angle_threshold;
    int min_pts, max_pts;
    int weight_kind;        // 0 constant, 1 Wendland ("rbf")
    unsigned seed;
};

template <typename T> __device__ __forceinline__ T sub_down(T a, T b);
template <> __device__ __forceinline__ float sub_down<float>(float a, float b) { return __fsub_rd(a, b); }
template <> __device__ __forceinline__ double sub_down<double>(double a, double b) { return __dsub_rd(a, b); }
template <typename T> __device__ __forceinline__ T add_up(T a, T b);
template <> __device__ __forceinline__ float add_up<float>(float a, float b) { return __fadd_ru(a, b); }
template <> __device__ __forceinline__ double add_up<double>(double a, double b) { return __dadd_ru(a, b); }

// Calls visit(pos, point, d2) for every point of the binned cloud with d2(q, point) < r2, in cell order, until visit
// returns true (the walk then ends and returns true); pos is the point's position in cl.sorted.
// Coverage: d2 >= fl(fl(q-p)^2) per axis and every rounding is monotone, so |q_a - p_a| <= sqrt(r2) (1 + 2 ulp) for
// every qualifying point; the box below is that interval, widened and rounded outwards, mapped through the monotone
// cell_of.  Rows (fixed y, z) whose wall gap already reaches r2 are skipped with the bound of search.cuh.
template <typename T, typename Visit>
__device__ __forceinline__ bool walk_ball_until(const Cloud<T>& cl, const GridHeader<T>& g, const Pt<T>& q, T r2, Visit&& visit) {
    using R = Real<T>;
    const T eps = sizeof(T) == 4 ? (T)1.1920929e-7 : (T)2.220446049250313e-16;
    const T reach = R::root(r2) * ((T)1 + (T)8 * eps) + (sizeof(T) == 4 ? (T)1.1754944e-38 : (T)2.2250738585072014e-308);
    int lo[3], hi[3], c[3];
    const T qv[3] = {q.x, q.y, q.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = cell_of<T>(sub_down<T>(qv[a], reach), g.origin[a], g.inv_h, g.dim[a]);
        hi[a] = cell_of<T>(add_up<T>(qv[a], reach), g.origin[a], g.inv_h, g.dim[a]);
        c[a] = cell_of<T>(qv[a], g.origin[a], g.inv_h, g.dim[a]);
    }
    const int st = g.stride;
    const T* lo_y = cl.wall_lo + st;      const T* hi_y = cl.wall_hi + st;
    const T* lo_z = cl.wall_lo + 2 * st;  const T* hi_z = cl.wall_hi + 2 * st;
    for (int z = lo[2]; z <= hi[2]; ++z) {
        const T bz = z < c[2] ? sq_gap<T>(q.z, lo_z[z + 1]) : (z > c[2] ? sq_gap<T>(q.z, hi_z[z]) : (T)0);
        if (!(bz < r2)) continue;
        for (int y = lo[1]; y <= hi[1]; ++y) {
            const T by = y < c[1] ? sq_gap<T>(q.y, lo_y[y + 1]) : (y > c[1] ? sq_gap<T>(q.y, hi_y[y]) : (T)0);
            if (!(R::add(by, bz) < r2)) continue;
            const unsigned row = (unsigned)((z * g.dim[1] + y) * g.dim[0]);
            const unsigned a = cl.cell_start[row + lo[0]], b = cl.cell_start[row + hi[0] + 1];
            for (unsigned j = a; j < b; ++j) {
                const Pt<T> p = load_pt<T>(cl.sorted + j);
                const T d2 = dist2<T>(q.x, q.y, q.z, p.x, p.y, p.z);
                if (d2 < r2 && visit(j, p, d2)) return true;
            }
        }
    }
    return false;
}

// Calls visit(point, d2) for every point of the binned cloud with d2(q, point) < r2, in cell order.
template <typename T, typename Visit>
__device__ __forceinline__ void walk_ball(const Cloud<T>& cl, const GridHeader<T>& g, const Pt<T>& q, T r2, Visit&& visit) {
    walk_ball_until<T>(cl, g, q, r2, [&](unsigned, const Pt<T>& p, T d2) { visit(p, d2); return false; });
}

// The binning kernels place the points of a cell in arrival order (an atomic counter), which changes from run to run.
// The ball walk adds its neighbours up in cell order, so for reproducible sums -- and a reproducible random subset --
// the points of every cell are put in ascending row order first.  One thread per cell; cells hold a few points
// (insertion sort), the odd crowded cell is heap-sorted in place.
template <typename T>
__device__ __forceinline__ void sift_down(Pt<T>* p, unsigned root, unsigned m) {
    for (;;) {
        unsigned child = 2 * root + 1;
        if (child >= m) return;
        if (child + 1 < m && p[child].i < p[child + 1].i) ++child;
        if (!(p[root].i < p[child].i)) return;
        const Pt<T> t = p[root]; p[root] = p[child]; p[child] = t;
        root = child;
    }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) cell_order_kernel(Cloud<T> cl) {
    grid_dependency_wait();
    const int ncells = cl.grid->ncells;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < ncells; c += (long long)gridDim.x * blockDim.x) {
        const unsigned a = cl.cell_start[c], b = cl.cell_start[c + 1];
        const unsigned m = b - a;
        if (m < 2) continue;
        Pt<T>* p = cl.sorted + a;
        if (m <= 24) {
            for (unsigned j = 1; j < m; ++j) {
                const Pt<T> key = p[j];
                unsigned t = j;
                while (t > 0 && p[t - 1].i > key.i) { p[t] = p[t - 1]; --t; }
                p[t] = key;
            }
        } else {
            for (unsigned r = m / 2; r-- > 0;) sift_down<T>(p, r, m);
            for (unsigned end = m - 1; end > 0; --end) {
                const Pt<T> t = p[0]; p[0] = p[end]; p[end] = t;
                sift_down<T>(p, 0, end);
            }
        }
    }
}

// The scale of every ball's fit (PlaneFit): one power of two for the call, bounding every weighted offset a ball holds.
// A member has d2 < r2, so |offset| <= sqrt(r2) (1 + 2 ulp); Wendland's weight falls from 1 on [0, 1] and rises
// beyond, so it is at most max(1, w(r_max)).  The bound scales with the cloud (r2 by 4^e for constant weights), and
// an infinite fp32 r2 admits offsets below 2^129 only.
template <typename T>
__device__ __forceinline__ double ball_scale(T r2, const BallParams& bp) {
    double bound = fmin(sqrt((double)r2), sizeof(T) == 4 ? 0x1p128 : 0x1.fffffffffffffp1023) * (1.0 + 0x1p-20);
    const double r = bound / bp.radius;
    if (bp.weight_kind == 1 && r > 1.0) {
        const double v1 = r - 1.0, v2 = 4 * r + 1.0;
        bound *= fmax(1.0, v1 * v1 * v1 * v1 * v2 * (1.0 + 0x1p-20));
    }
    return pow2_scale(fmin(bound, 0x1.fffffffffffffp1023));
}

// One thread per point, in CELL order (neighbouring lanes walk overlapping boxes).  normals / keep are indexed by the
// caller's row.  The fit's first pass rides on the walk that counts the ball; each further pass walks it again.
template <typename T>
__global__ void __launch_bounds__(kThreads) normals_ball_kernel(Cloud<T> cl, const T* __restrict__ view_dirs, BallParams bp,
                                                                T* __restrict__ normals, unsigned char* __restrict__ keep) {
    grid_dependency_wait();
    using R = Real<T>;
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *cl.grid;
    __syncthreads();
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= cl.n) return;
    const Pt<T> q = load_pt<T>(cl.sorted + pos);
    const long long row = (long long)q.i;
    const T r2 = (T)bp.radius;                       // radiusSearch takes a DistanceType: the double is narrowed (:74)
    auto wendland = [&](double r) { const double v1 = 1.0 - r, v2 = 4 * r + 1.0; return v1 * v1 * v1 * v1 * v2; };
    PlaneFit fit(ball_scale<T>(r2, bp));
    auto fold = [&](const Pt<T>& p, T d2) {
        // wendland_rbf (:334-339), in double like the reference
        const double w = bp.weight_kind == 1 ? wendland(sqrt((double)d2) / bp.radius) : 1.0;
        // (points(nbr, j) - query[j]) * weight: the difference in the cloud's precision, the product in double (:89)
        fit.add((double)R::sub(p.x, q.x) * w, (double)R::sub(p.y, q.y) * w, (double)R::sub(p.z, q.z) * w);
    };
    long long found = 0;
    walk_ball<T>(cl, g, q, r2, [&](const Pt<T>& p, T d2) { ++found; fold(p, d2); });   // also the fit's first pass
    bool ok = found >= (long long)bp.min_pts;        // :75-77 (before the cap)
    const bool capped = bp.max_pts > 0 && found > (long long)bp.max_pts;
    // The capped fit's passes replay one selection sequence: the same subset every time.
    const unsigned salt = mix32(bp.seed ^ mix32((unsigned)row * 0x9e3779b9u + 0x85ebca6bu));
    auto fold_subset = [&]() {
        unsigned long long remaining = (unsigned long long)found, needed = (unsigned long long)bp.max_pts;
        unsigned t = 0;
        walk_ball<T>(cl, g, q, r2, [&](const Pt<T>& p, T d2) {
            const unsigned long long u = ((unsigned long long)mix32(salt + t * 0x9e3779b9u) * remaining) >> 32;   // uniform in [0, remaining)
            ++t;
            if (u < needed) { fold(p, d2); --needed; }
            --remaining;
        });
    };
    double nrm[3] = {0.0, 0.0, 0.0};
    if (ok) {
        if (capped) { fit.reset(); fold_subset(); }
        while (fit.solve()) {
            if (capped) fold_subset();
            else walk_ball<T>(cl, g, q, r2, fold);
        }
        fit.normal(capped ? (long long)bp.max_pts : found, nrm);
        if (view_dirs != nullptr)
            ok = orient_by_view(nrm, (double)view_dirs[3 * row], (double)view_dirs[3 * row + 1], (double)view_dirs[3 * row + 2],
                                bp.drop_angle_threshold);
    }
    normals[3 * row] = (T)nrm[0]; normals[3 * row + 1] = (T)nrm[1]; normals[3 * row + 2] = (T)nrm[2];
    keep[row] = ok ? 1 : 0;
}

// ---- principal curvatures from a quadric fit over a ball (mesh_principal_curvatures with r > 0, curvature.cuh) -----
// One thread per vertex, in CELL order, over the binned vertices.  The ball is { j != i : d2(p_i, p_j) < (T)(r r) }.
// With n = the vertex's fp64 normal and (t1, t2) its frame, each neighbour's offset o = p_j - p_i (fp64) gives
// (x, y, z) = (o . t1, o . t2, o . n) / r, and z = a x^2 + b x y + c y^2 + d x + e y is fitted by least squares: the
// 5 x 5 normal equations, folded in cell order, solved by Cholesky.  Undetermined: fewer than 5 neighbours, a zero
// normal, or a pivot <= 1e-12 times the largest diagonal entry of the system.
template <typename T>
__global__ void __launch_bounds__(kThreads) curv_ball_kernel(Cloud<T> cl, const double* __restrict__ normal, double r, T* __restrict__ out_k1,
                                                             T* __restrict__ out_k2, T* __restrict__ out_d1, T* __restrict__ out_d2) {
    grid_dependency_wait();
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *cl.grid;
    __syncthreads();
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= cl.n) return;
    const Pt<T> q = load_pt<T>(cl.sorted + pos);
    const long long row = (long long)q.i;
    double n[3], t1[3], t2[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) n[a] = normal[3 * row + a];
    const bool has_normal = n[0] != 0.0 || n[1] != 0.0 || n[2] != 0.0;
    curv_frame(n, t1, t2);
    double M[15], y[5];   // M: the lower triangle by rows, M[i (i + 1) / 2 + j] for j <= i
#pragma unroll
    for (int k = 0; k < 15; ++k) M[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 5; ++k) y[k] = 0.0;
    long long found = 0;
    if (has_normal)
        walk_ball<T>(cl, g, q, (T)(r * r), [&](const Pt<T>& p, T) {
            if (p.i == q.i) return;
            ++found;
            const double o[3] = {(double)p.x - (double)q.x, (double)p.y - (double)q.y, (double)p.z - (double)q.z};
            const double x = curv_dot(o, t1) / r, yy = curv_dot(o, t2) / r, z = curv_dot(o, n) / r;
            const double phi[5] = {x * x, x * yy, yy * yy, x, yy};
#pragma unroll
            for (int i = 0; i < 5; ++i) {
#pragma unroll
                for (int j = 0; j <= i; ++j) M[i * (i + 1) / 2 + j] += phi[i] * phi[j];
                y[i] += phi[i] * z;
            }
        });
    bool ok = has_normal && found >= 5;
    double big = 0.0;
#pragma unroll
    for (int i = 0; i < 5; ++i) big = fmax(big, M[i * (i + 1) / 2 + i]);
    // M = L L^T in place: pivot_k = M_kk - sum_{j<k} L_kj^2 must exceed 1e-12 big; L_ik = (M_ik - sum_{j<k} L_ij L_kj) / L_kk
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        double piv = M[k * (k + 1) / 2 + k];
#pragma unroll
        for (int j = 0; j < k; ++j) piv -= M[k * (k + 1) / 2 + j] * M[k * (k + 1) / 2 + j];
        ok = ok && piv > 1e-12 * big;
        const double lkk = sqrt(fmax(piv, 0.0));
        M[k * (k + 1) / 2 + k] = lkk;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) {
            double s = M[i * (i + 1) / 2 + k];
#pragma unroll
            for (int j = 0; j < k; ++j) s -= M[i * (i + 1) / 2 + j] * M[k * (k + 1) / 2 + j];
            M[i * (i + 1) / 2 + k] = s / lkk;
        }
    }
    // L z = y, then L^T x = z
#pragma unroll
    for (int i = 0; i < 5; ++i) {
#pragma unroll
        for (int j = 0; j < i; ++j) y[i] -= M[i * (i + 1) / 2 + j] * y[j];
        y[i] /= M[i * (i + 1) / 2 + i];
    }
#pragma unroll
    for (int i = 4; i >= 0; --i) {
#pragma unroll
        for (int j = i + 1; j < 5; ++j) y[i] -= M[j * (j + 1) / 2 + i] * y[j];
        y[i] /= M[i * (i + 1) / 2 + i];
    }
    double k1 = 0.0, k2 = 0.0, d1[3] = {t1[0], t1[1], t1[2]}, d2[3] = {0.0, 0.0, 0.0};
    if (ok) curv_monge(y, r, n, t1, t2, k1, k2, d1, d2);
    curv_store<T>(row, ok, k1, k2, d1, d2, out_k1, out_k2, out_d1, out_d2);
}

// The kept points and their normals in index order (the reference's single-thread loop appends in that order,
// :267-279), after keep_count / keep_offsets of compact.cuh.
template <typename T>
__global__ void __launch_bounds__(kThreads) keep_scatter_kernel(const unsigned char* __restrict__ keep, long long n,
                                                                const unsigned* __restrict__ block_offset,
                                                                const T* __restrict__ normals, long long* __restrict__ out_idx,
                                                                T* __restrict__ out_normals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? keep[i] : 0u;
    const unsigned pos = keep_rank(mine, block_offset);
    if (mine) {
        out_idx[pos] = i;
        out_normals[3ll * pos] = normals[3 * i];
        out_normals[3ll * pos + 1] = normals[3 * i + 1];
        out_normals[3ll * pos + 2] = normals[3 * i + 2];
    }
}

}  // namespace pcu
