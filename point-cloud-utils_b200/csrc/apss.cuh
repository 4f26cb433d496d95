// apss.cuh -- algebraic point set surfaces of oriented point clouds (Guennebaud & Gross 2007, the spherical fit with
// beta = 1): pointcloud_apss_curvature and project_points_onto_apss.  The rules are DESIGN.md §3's; in brief, from an
// iterate x (fp64) the ball N(x) = { j : d2(fl_T(x), p_j) < (T)(r r), n_j != 0 } is walked in cell order, each member
// adds w = max(0, 1 - |o|^2 / r^2)^4 (o = p_j - x) to nine fp64 sums, the algebraic sphere
// s(y) = u0 + u . y + u4 |y|^2 is fitted in closed form, and x moves to the sphere along u.  The last fit gives the
// normal u / |u| and the mean curvature 2 u4 / sqrt(D).
//
// nearest.cu bins the cloud (single_cloud_plan with cells no finer than r / 2, enqueue_binning, cell_order_kernel),
// then apss_normals_kernel writes every point's unit normal in cell order, so the walk reads a member's normal at the
// member's own position, and apss_kernel runs one thread per query.  No synchronisation: the call is stream-ordered,
// as the plan and the binning are.
#pragma once
#include "normals.cuh"

namespace pcu {

constexpr int kApssMaxSteps = 20;         // MeshLab's default iteration cap
constexpr double kApssStepTol = 1e-10;    // a step of at most this times r ends the iteration

// nrm[pos] = n[row] / |n[row]| in fp64 for the point at cell position pos (row its index); 0 for a zero normal.
template <typename T>
__global__ void __launch_bounds__(kThreads) apss_normals_kernel(Cloud<T> cl, const T* __restrict__ n, double* __restrict__ nrm) {
    grid_dependency_wait();
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= cl.n) return;
    const long long row = (long long)load_pt<T>(cl.sorted + pos).i;
    const double a = (double)n[3 * row], b = (double)n[3 * row + 1], c = (double)n[3 * row + 2];
    const double len = sqrt((a * a + b * b) + c * c);
    const bool ok = len > 0.0;
    nrm[3 * pos] = ok ? a / len : 0.0;
    nrm[3 * pos + 1] = ok ? b / len : 0.0;
    nrm[3 * pos + 2] = ok ? c / len : 0.0;
}

// One thread per query.  q == nullptr: the queries are the binned points themselves, in cell order, and each result
// goes to the point's row; otherwise query i is q[i] and its result goes to row i.  out_x and out_n may be null.
template <typename T>
__global__ void __launch_bounds__(kThreads) apss_kernel(Cloud<T> cl, const double* __restrict__ nrm, const T* __restrict__ q, long long nq,
                                                        double r, T* __restrict__ out_x, T* __restrict__ out_n, T* __restrict__ out_kh) {
    grid_dependency_wait();
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *cl.grid;
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    long long row = i;
    double x[3];
    if (q != nullptr) {
        x[0] = (double)q[3 * i]; x[1] = (double)q[3 * i + 1]; x[2] = (double)q[3 * i + 2];
    } else {
        const Pt<T> p = load_pt<T>(cl.sorted + i);
        row = (long long)p.i;
        x[0] = (double)p.x; x[1] = (double)p.y; x[2] = (double)p.z;
    }
    const double rr = r * r;
    const T r2 = (T)rr;
    double u[3] = {0.0, 0.0, 0.0}, u4 = 0.0, gu = 0.0, D = 0.0;
    bool ok = true;
    for (int step = 0; step < kApssMaxSteps; ++step) {
        Pt<T> c;
        c.x = (T)x[0]; c.y = (T)x[1]; c.z = (T)x[2];
        double W = 0.0, P[3] = {0.0, 0.0, 0.0}, N[3] = {0.0, 0.0, 0.0}, PN = 0.0, PP = 0.0;
        int members = 0;
        walk_ball_until<T>(cl, g, c, r2, [&](unsigned j, const Pt<T>& p, T) {
            const double n0 = nrm[3ull * j], n1 = nrm[3ull * j + 1], n2 = nrm[3ull * j + 2];
            if (n0 == 0.0 && n1 == 0.0 && n2 == 0.0) return false;
            ++members;
            const double o0 = (double)p.x - x[0], o1 = (double)p.y - x[1], o2 = (double)p.z - x[2];
            const double oo = (o0 * o0 + o1 * o1) + o2 * o2;
            const double t = fmax(0.0, 1.0 - oo / rr), t2 = t * t, w = t2 * t2;
            W += w;
            P[0] += w * o0; P[1] += w * o1; P[2] += w * o2;
            N[0] += w * n0; N[1] += w * n1; N[2] += w * n2;
            PN += w * ((o0 * n0 + o1 * n1) + o2 * n2);
            PP += w * oo;
            return false;
        });
        if (members < 4 || !(W > 0.0)) { ok = false; break; }
        // the fit in coordinates centred at x
        const double den = PP - ((P[0] * P[0] + P[1] * P[1]) + P[2] * P[2]) / W;
        u4 = den > 1e-12 * PP ? 0.5 * (PN - ((P[0] * N[0] + P[1] * N[1]) + P[2] * N[2]) / W) / den : 0.0;
#pragma unroll
        for (int a = 0; a < 3; ++a) u[a] = (N[a] - 2.0 * u4 * P[a]) / W;
        const double u0 = -(((u[0] * P[0] + u[1] * P[1]) + u[2] * P[2]) + u4 * PP) / W;
        // the step: the stable root of s(t u / |u|) = 0
        gu = sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]);
        D = gu * gu - 4.0 * u0 * u4;
        if (!(gu > 0.0) || D < 0.0) { ok = false; break; }
        const double t = -2.0 * u0 / (gu + sqrt(D));
        double y[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            y[a] = t * (u[a] / gu);
            x[a] += y[a];
        }
        if (sqrt((y[0] * y[0] + y[1] * y[1]) + y[2] * y[2]) <= kApssStepTol * r) break;
    }
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    if (out_x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) out_x[3 * row + a] = (T)(ok ? x[a] : nan);
    }
    if (out_n) {
#pragma unroll
        for (int a = 0; a < 3; ++a) out_n[3 * row + a] = (T)(ok ? u[a] / gu : 0.0);
    }
    out_kh[row] = (T)(ok ? 2.0 * u4 / sqrt(D) : nan);
}

// The result of every query against an empty cloud: undetermined.
template <typename T>
__global__ void __launch_bounds__(kThreads) apss_undetermined_kernel(long long nq, T* __restrict__ out_x, T* __restrict__ out_n,
                                                                     T* __restrict__ out_kh) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const T nan = (T)__longlong_as_double(0x7ff8000000000000LL);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (out_x) out_x[3 * i + a] = nan;
        if (out_n) out_n[3 * i + a] = (T)0;
    }
    out_kh[i] = nan;
}

}  // namespace pcu
