// curvature.cuh -- principal curvatures and directions of a triangle mesh (mesh_principal_curvatures; the reference
// declares it in src/curvature.cpp but ships no body).  Results defined in DESIGN.md §3.
//
//   curv_frame / curv_eigen / curv_directions / curv_monge   the device rules both modes share: the tangent frame of a
//                         unit normal, the 2 x 2 eigen rule, the sign rule of the directions and the shape operator of
//                         a fitted height field
//   curv_face_kernel      one thread per face (one-ring mode): the face's second fundamental form (E, F, G) in its own
//                         frame (u, w x u), by least squares over its three edges, and its corners' mixed Voronoi areas
//   curv_vertex_kernel    one thread per vertex over the corner CSR of mesh_geometry.cuh: the area-weighted mean of its
//                         faces' forms, each rotated into the vertex's frame, then the eigen rule
// The ball mode's kernel (curv_ball_kernel) sits with the other ball walk in normals.cuh.  Every kernel here is a
// template launched from mesh_topology.cu alone, so each compiles once although nearest.cu sees this header too.
#pragma once
#include "common.cuh"
#include "meshsample.cuh"

namespace pcu {

__device__ __forceinline__ double curv_dot(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ __forceinline__ void curv_cross(const double a[3], const double b[3], double out[3]) {
    out[0] = a[1] * b[2] - a[2] * b[1];
    out[1] = a[2] * b[0] - a[0] * b[2];
    out[2] = a[0] * b[1] - a[1] * b[0];
}

// The branchless orthonormal basis (t1, t2) of the unit normal n, with t1 x t2 = n (Duff et al. 2017).
__device__ __forceinline__ void curv_frame(const double n[3], double t1[3], double t2[3]) {
    const double s = copysign(1.0, n[2]);
    const double a = -1.0 / (s + n[2]);
    const double b = n[0] * n[1] * a;
    t1[0] = 1.0 + s * n[0] * n[0] * a; t1[1] = s * b; t1[2] = -s * n[0];
    t2[0] = b; t2[1] = s + n[1] * n[1] * a; t2[2] = -n[1];
}

// Eigenvalues k1 >= k2 of [[a, b], [b, c]], (a + c) / 2 +- hypot((a - c) / 2, b), and the unit eigenvector (x, y) of
// k1: (h + p, b) when p = (a - c) / 2 >= 0, else (b, h - p), normalised; (1, 0) at an umbilic (h = 0).
__device__ __forceinline__ void curv_eigen(double a, double b, double c, double& k1, double& k2, double& x, double& y) {
    const double m = 0.5 * (a + c), p = 0.5 * (a - c);
    const double h = hypot(p, b);
    k1 = m + h;
    k2 = m - h;
    if (h == 0.0) { x = 1.0; y = 0.0; return; }
    x = p >= 0.0 ? h + p : b;
    y = p >= 0.0 ? b : h - p;
    const double len = hypot(x, y);
    x /= len;
    y /= len;
}

// d normalised, its component of largest magnitude made positive (the lowest axis wins a tie); e = n x d.
__device__ __forceinline__ void curv_directions(double d[3], const double n[3], double e[3]) {
    const double len = sqrt(curv_dot(d, d));
    int j = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        d[a] /= len;
        if (fabs(d[a]) > fabs(d[j])) j = a;
    }
    if (d[j] < 0.0)
#pragma unroll
        for (int a = 0; a < 3; ++a) d[a] = -d[a];
    curv_cross(n, d, e);
}

// Writes vertex i's result rounded once to T: k = NaN and zero directions when ok is false.
template <typename T>
__device__ __forceinline__ void curv_store(long long i, bool ok, double k1, double k2, const double d1[3], const double d2[3], T* out_k1,
                                           T* out_k2, T* out_d1, T* out_d2) {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    out_k1[i] = (T)(ok ? k1 : nan);
    out_k2[i] = (T)(ok ? k2 : nan);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        out_d1[3 * i + a] = (T)(ok ? d1[a] : 0.0);
        out_d2[3 * i + a] = (T)(ok ? d2[a] : 0.0);
    }
}

// The shape operator of the height field z = a x^2 + b x y + c y^2 + d x + e y over the frame (t1, t2, n), in
// coordinates scaled by 1 / r: the eigenvalues of -I^-1 II rescaled by 1 / r, with I = [[1 + d^2, d e], [d e, 1 + e^2]]
// and II = [[2a, b], [b, 2c]] / sqrt(1 + d^2 + e^2).  I = L L^T (Cholesky), S = -L^-1 II L^-T / r is symmetric and
// takes the eigen rule; the eigenvector w of k1 maps back to v = L^-T w and to 3-D as v0 (t1 + d n) + v1 (t2 + e n).
// d1 follows the sign rule and d2 = nf x d1, nf the unit normal of the fitted surface, n - d t1 - e t2 normalised.
__device__ __forceinline__ void curv_monge(const double q[5], double r, const double n[3], const double t1[3], const double t2[3],
                                           double& k1, double& k2, double d1[3], double d2[3]) {
    const double a = q[0], b = q[1], c = q[2], d = q[3], e = q[4];
    const double g = sqrt(1.0 + d * d + e * e);
    const double l11 = sqrt(1.0 + d * d), l21 = d * e / l11, l22 = sqrt((1.0 + e * e) - l21 * l21);
    const double p = 1.0 / l11, s = 1.0 / l22, t = -l21 * p * s;   // L^-1 = [[p, 0], [t, s]]
    const double B00 = 2.0 * a, B01 = b, B11 = 2.0 * c;
    const double scale = -1.0 / (r * g);
    const double S00 = p * p * B00 * scale;
    const double S01 = p * (t * B00 + s * B01) * scale;
    const double S11 = (t * t * B00 + 2.0 * t * s * B01 + s * s * B11) * scale;
    double w0, w1;
    curv_eigen(S00, S01, S11, k1, k2, w0, w1);
    const double v0 = p * w0 + t * w1, v1 = s * w1;
    double nf[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        d1[k] = v0 * (t1[k] + d * n[k]) + v1 * (t2[k] + e * n[k]);
        nf[k] = n[k] - d * t1[k] - e * t2[k];
    }
    const double len = sqrt(curv_dot(nf, nf));
#pragma unroll
    for (int k = 0; k < 3; ++k) nf[k] /= len;
    curv_directions(d1, nf, d2);
}

// One thread per face, one-ring mode.  Corners p0, p1, p2, vertex normals n0, n1, n2 (fp64, unit), edges e0 = p2 - p1,
// e1 = p0 - p2, e2 = p1 - p0 with normal differences dn0 = n2 - n1, dn1 = n0 - n2, dn2 = n1 - n0.  Frame u = e0 / |e0|,
// w = the face's unit normal, v = w x u.  (E, F, G) solves the normal equations M x = y of the six rows
// [e.u, e.v, 0] x = dn.u and [0, e.u, e.v] x = dn.v (M[0][2] = 0) by Cholesky: every pivot must be positive.  A face
// with dblA = 0 or a pivot that is not contributes nothing: E = NaN.  cw: each corner's mixed Voronoi area, from
// halfcot (cot / 2) and dblA -- (|e_j|^2 cot_j + |e_k|^2 cot_k) / 8 over the corner's other two corners j, k, or dblA / 4
// at the obtuse corner and dblA / 8 at the others of an obtuse face.
template <typename T>
__global__ void __launch_bounds__(kThreads) curv_face_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                             long long m, const double* __restrict__ normal, const double* __restrict__ unit,
                                                             const double* __restrict__ dbla, const double* __restrict__ halfcot,
                                                             double* __restrict__ frame_u, double* __restrict__ efg, double* __restrict__ cw) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    long long c[3];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c[k] = load_index(f, 3 * t + k, fkind, nv, false);
        bad = bad || c[k] < 0;
    }
    const double A = bad ? 0.0 : dbla[t];
    double p[3][3], n[3][3], e[3][3], dn[3][3], len2[3], hc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        load_vertex<T>(v, bad ? 0 : c[k], p[k]);
#pragma unroll
        for (int a = 0; a < 3; ++a) n[k][a] = __ldg(normal + 3 * (bad ? 0 : c[k]) + a);
        hc[k] = halfcot[3 * t + k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            e[k][a] = p[(k + 2) % 3][a] - p[(k + 1) % 3][a];
            dn[k][a] = n[(k + 2) % 3][a] - n[(k + 1) % 3][a];
        }
        len2[k] = curv_dot(e[k], e[k]);
    }
    const bool obtuse = hc[0] < 0.0 || hc[1] < 0.0 || hc[2] < 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int j = (k + 1) % 3, l = (k + 2) % 3;
        cw[3 * t + k] = A == 0.0 ? 0.0 : obtuse ? (hc[k] < 0.0 ? 0.25 * A : 0.125 * A) : 0.25 * (len2[j] * hc[j] + len2[l] * hc[l]);
    }
    double u[3], w[3], vv[3];
    const double el = sqrt(len2[0]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        u[a] = e[0][a] / el;
        w[a] = unit[3 * t + a];
    }
    curv_cross(w, u, vv);
    double M00 = 0.0, M01 = 0.0, M11 = 0.0, M12 = 0.0, M22 = 0.0, y0 = 0.0, y1 = 0.0, y2 = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double eu = curv_dot(e[k], u), ev = curv_dot(e[k], vv), nu = curv_dot(dn[k], u), nw = curv_dot(dn[k], vv);
        M00 += eu * eu;
        M01 += eu * ev;
        M11 += eu * eu + ev * ev;
        M12 += eu * ev;
        M22 += ev * ev;
        y0 += eu * nu;
        y1 += ev * nu + eu * nw;
        y2 += ev * nw;
    }
    // M = L L^T: L00 = sqrt(M00), L10 = M01 / L00, L11 = sqrt(M11 - L10^2), L21 = M12 / L11, L22 = sqrt(M22 - L21^2)
    const double q0 = M00;
    const double L00 = sqrt(q0), L10 = M01 / L00;
    const double q1 = M11 - L10 * L10;
    const double L11 = sqrt(q1), L21 = M12 / L11;
    const double q2 = M22 - L21 * L21;
    const double L22 = sqrt(q2);
    const bool ok = A != 0.0 && q0 > 0.0 && q1 > 0.0 && q2 > 0.0;
    const double z0 = y0 / L00, z1 = (y1 - L10 * z0) / L11, z2 = (y2 - L21 * z1) / L22;
    const double G = z2 / L22, F = (z1 - L21 * G) / L11, E = (z0 - L10 * F) / L00;
    efg[3 * t] = ok ? E : __longlong_as_double(0x7ff8000000000000LL);
    efg[3 * t + 1] = ok ? F : 0.0;
    efg[3 * t + 2] = ok ? G : 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) frame_u[3 * t + a] = ok ? u[a] : 0.0;
}

// One thread per vertex, one-ring mode.  Over its corners in ascending (face, corner) order, every contributing face's
// (E, F, G) is carried into the vertex frame: the face frame (u, v) is rotated about w x n so that w lands on n,
// rt = t - (t . p) (w + n) / (1 + w . n) with p = n - (w . n) w (rt = -t when w . n <= -1), and with u1 = t1 . ru,
// v1 = t1 . rv, u2 = t2 . ru, v2 = t2 . rv the form becomes a = E u1^2 + 2 F u1 v1 + G v1^2, b = E u1 u2 +
// F (u1 v2 + u2 v1) + G v1 v2, c = E u2^2 + 2 F u2 v2 + G v2^2.  The cw-weighted sum over the sum of the weights takes
// the eigen rule; d1 = x t1 + y t2.  No contributing face or a zero normal: undetermined.
template <typename T>
__global__ void __launch_bounds__(kThreads) curv_vertex_kernel(const int* __restrict__ first, const int* __restrict__ corner, long long nv,
                                                               const double* __restrict__ normal, const double* __restrict__ unit,
                                                               const double* __restrict__ frame_u, const double* __restrict__ efg,
                                                               const double* __restrict__ cw, T* __restrict__ out_k1, T* __restrict__ out_k2,
                                                               T* __restrict__ out_d1, T* __restrict__ out_d2) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= nv) return;
    double n[3], t1[3], t2[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) n[a] = normal[3 * i + a];
    const bool has_normal = n[0] != 0.0 || n[1] != 0.0 || n[2] != 0.0;
    curv_frame(n, t1, t2);
    double sa = 0.0, sb = 0.0, sc = 0.0, sw = 0.0;
    for (int j = first[i], end = first[i + 1]; has_normal && j < end; ++j) {
        const int c = __ldg(corner + j);
        const long long t = c / 3;
        const double E = __ldg(efg + 3 * t);
        if (E != E) continue;
        const double F = __ldg(efg + 3 * t + 1), G = __ldg(efg + 3 * t + 2), wt = __ldg(cw + c);
        double u[3], w[3], vv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            u[a] = __ldg(frame_u + 3 * t + a);
            w[a] = __ldg(unit + 3 * t + a);
        }
        curv_cross(w, u, vv);
        const double nd = curv_dot(w, n);
        if (nd <= -1.0) {
#pragma unroll
            for (int a = 0; a < 3; ++a) { u[a] = -u[a]; vv[a] = -vv[a]; }
        } else {
            double perp[3], dperp[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                perp[a] = n[a] - nd * w[a];
                dperp[a] = (w[a] + n[a]) / (1.0 + nd);
            }
            const double up = curv_dot(u, perp), vp = curv_dot(vv, perp);
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                u[a] -= dperp[a] * up;
                vv[a] -= dperp[a] * vp;
            }
        }
        const double u1 = curv_dot(t1, u), v1 = curv_dot(t1, vv), u2 = curv_dot(t2, u), v2 = curv_dot(t2, vv);
        sa += wt * (E * u1 * u1 + 2.0 * F * u1 * v1 + G * v1 * v1);
        sb += wt * (E * u1 * u2 + F * (u1 * v2 + u2 * v1) + G * v1 * v2);
        sc += wt * (E * u2 * u2 + 2.0 * F * u2 * v2 + G * v2 * v2);
        sw += wt;
    }
    const bool ok = has_normal && sw > 0.0;
    double k1 = 0.0, k2 = 0.0, x = 1.0, y = 0.0, d1[3], d2[3];
    if (ok) curv_eigen(sa / sw, sb / sw, sc / sw, k1, k2, x, y);
#pragma unroll
    for (int a = 0; a < 3; ++a) d1[a] = x * t1[a] + y * t2[a];
    curv_directions(d1, n, d2);
    curv_store<T>(i, ok, k1, k2, d1, d2, out_k1, out_k2, out_d1, out_d2);
}

}  // namespace pcu
