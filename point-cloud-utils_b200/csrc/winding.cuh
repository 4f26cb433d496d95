// winding.cuh -- winding numbers and signed distances on the tree of meshquery.cuh (triangle_soup_fast_winding_number
// and signed_distance_to_mesh of the reference, src/fast_winding_numbers.cpp and src/signed_distance.cpp, which call
// libigl's fast_winding_number and signed_distance).
//
// The field is defined in DESIGN.md §3 (winding number), after Barill et al. 2018, "Fast Winding Numbers for Soups and
// Clouds", evaluated in fp32 as libigl does.  The tree's leaves are faces (Pt<T>) or, for point_cloud_fast_winding_number
// (the same section of DESIGN.md), points (WnPoint, filled by wn_point_leaves_kernel); every pass below serves both
// leaf kinds, which differ only where noted:
//   leaf           always exact: a face's signed solid angle or a point's dipole term, in fp32 (wn_leaf_omega)
//   internal node  when |q - P| > beta r, the order-2 far-field expansion about its area-weighted centre P (wn_far),
//                  and its subtree is not entered; otherwise child 0's subtree, then child 1's.  A point tree's node of
//                  radius 0 is always entered.
//   query          the terms summed in fp64 in that fixed order, w = fp32(sum / 4 pi): a function of the leaves and q
//
//   wn_centres_kernel   bottom-up over the existing topology (as mq_refit_kernel): each node's area and centre P
//   wn_radius_kernel    every leaf climbs to the root and raises each ancestor's r to the farthest of its points
//   wn_moments_kernel   bottom-up again: the second child to arrive at a node shifts both children's moments to the
//                       node's P, child 0 then child 1, and writes them in units of the node's r
//   wn_query_kernel     one thread per query
//   sd_sign_kernel      signed distance after mq_query_kernel: the band on d^2, then sigma = 1 - 2|w| and s = sigma d
#pragma once
#include "meshquery.cuh"

namespace pcu {

// Far-field data of an internal node, about P (fp32).  The first and second moments of the area-weighted normal field,
// M_ij = int (x - P)_j n_i dA and Q_ijk = int (x - P)_j (x - P)_k n_i dA, enter the expansion only through their
// fully symmetric parts, which are what is stored.  The moments are stored in units of the node's radius (N / r^2,
// M / r^3, Q / r^4; 0 when r = 0), so neither they nor the expansion (wn_far) depend on the mesh's scale.
struct __align__(16) WnNode {
    float P[3], r;   // area-weighted centre; largest distance from P to a corner in the subtree (rounded up)
    float N[3], A;   // sum of the area-weighted normals (order 0) / r^2; area
    float M[6];      // symmetric part of M / r^3: xx yy zz xy xz yz
    float S[10];     // fully symmetric part of Q / r^4: xxx yyy zzz xxy xxz xyy yyz xzz yzz xyz
};
static_assert(sizeof(WnNode) == 96, "six float4 per node");

// The same data in fp64 while a node is combined.
struct WnRec { double P[3], A, N[3], M[6], S[10]; };

// Slots of the symmetric storage: M_ij at wn_m(i, j); Q_ijk, i <= j <= k, at t with (i, j, k) = wn_s(t, 0..2).  Called
// with unrolled constant arguments only, so every index folds away.
__device__ __forceinline__ int wn_m(int i, int j) { return i == j ? i : i + j + 2; }   // (0,1) 3, (0,2) 4, (1,2) 5
__device__ __forceinline__ int wn_s(int t, int s) {
    const int code[10] = {0x000, 0x111, 0x222, 0x001, 0x002, 0x011, 0x112, 0x022, 0x122, 0x012};
    return (code[t] >> (4 * (2 - s))) & 15;
}

template <typename T>
__device__ __forceinline__ void wn_leaf_corners(const Pt<T>* __restrict__ leaves, int j, float a[3], float b[3], float c[3]) {
    const Pt<T> A = leaves[3 * j], B = leaves[3 * j + 1], C = leaves[3 * j + 2];
    a[0] = (float)A.x; a[1] = (float)A.y; a[2] = (float)A.z;
    b[0] = (float)B.x; b[1] = (float)B.y; b[2] = (float)B.z;
    c[0] = (float)C.x; c[1] = (float)C.y; c[2] = (float)C.z;
}

// One face's exact moments (fp64 from its fp32 corners) about its centroid g: N = (b - a) x (c - a) / 2, A = |N|,
// M = 0, Q_ijk = N_i C_jk with C = (1/12) sum over the corners of (x - g)(x - g)^T (the triangle's exact second moment
// about g, divided by its area).
template <typename T>
__device__ __forceinline__ WnRec wn_leaf_rec(const Pt<T>* __restrict__ leaves, int j) {
    float fa[3], fb[3], fc[3];
    wn_leaf_corners<T>(leaves, j, fa, fb, fc);
    double a[3], b[3], c[3], e1[3], e2[3];
    WnRec r;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        a[k] = fa[k]; b[k] = fb[k]; c[k] = fc[k];
        e1[k] = b[k] - a[k]; e2[k] = c[k] - a[k];
        r.P[k] = (a[k] + b[k] + c[k]) / 3.0;
        a[k] -= r.P[k]; b[k] -= r.P[k]; c[k] -= r.P[k];
    }
    r.N[0] = 0.5 * (e1[1] * e2[2] - e1[2] * e2[1]);
    r.N[1] = 0.5 * (e1[2] * e2[0] - e1[0] * e2[2]);
    r.N[2] = 0.5 * (e1[0] * e2[1] - e1[1] * e2[0]);
    r.A = sqrt(r.N[0] * r.N[0] + r.N[1] * r.N[1] + r.N[2] * r.N[2]);
    double C[6];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = i; k < 3; ++k) C[wn_m(i, k)] = (a[i] * a[k] + b[i] * b[k] + c[i] * c[k]) / 12.0;
#pragma unroll
    for (int t = 0; t < 6; ++t) r.M[t] = 0.0;
#pragma unroll
    for (int t = 0; t < 10; ++t) {
        const int i = wn_s(t, 0), j2 = wn_s(t, 1), k = wn_s(t, 2);
        r.S[t] = (r.N[i] * C[wn_m(j2, k)] + r.N[j2] * C[wn_m(i, k)] + r.N[k] * C[wn_m(i, j2)]) / 3.0;
    }
    return r;
}

// One point's moments about the point itself: N = an, A = |a|, M = 0, Q = 0.
__device__ __forceinline__ WnRec wn_leaf_rec(const WnPoint* __restrict__ leaves, int j) {
    const float4* s = reinterpret_cast<const float4*>(leaves + j);
    const float4 x = s[0], y = s[1];
    WnRec r;
    r.P[0] = x.x; r.P[1] = x.y; r.P[2] = x.z; r.A = x.w;
    r.N[0] = y.x; r.N[1] = y.y; r.N[2] = y.z;
#pragma unroll
    for (int t = 0; t < 6; ++t) r.M[t] = 0.0;
#pragma unroll
    for (int t = 0; t < 10; ++t) r.S[t] = 0.0;
    return r;
}

// The fp32 points of leaf j that bound its ancestors' radii: a face's three corners, or the point.
template <typename T>
__device__ __forceinline__ void wn_leaf_points(const Pt<T>* __restrict__ leaves, int j, float (&c)[3][3]) {
    wn_leaf_corners<T>(leaves, j, c[0], c[1], c[2]);
}
__device__ __forceinline__ void wn_leaf_points(const WnPoint* __restrict__ leaves, int j, float (&c)[1][3]) {
    const float4 x = *reinterpret_cast<const float4*>(leaves + j);
    c[0][0] = x.x; c[0][1] = x.y; c[0][2] = x.z;
}

// The build passes below read a leaf only through wn_leaf_rec and wn_leaf_points.
// Child c of a node, its area and centre: a leaf's own, or an internal node's as stored (written by other threads of
// this launch).
template <typename L>
__device__ __forceinline__ void wn_child_centre(const WnNode* wn, const L* __restrict__ leaves, int c, double P[3], double& A) {
    if (c < 0) {
        const WnRec r = wn_leaf_rec(leaves, ~c);
        P[0] = r.P[0]; P[1] = r.P[1]; P[2] = r.P[2]; A = r.A;
        return;
    }
    const float4* p = reinterpret_cast<const float4*>(wn + c);
    const float4 q0 = __ldcg(p), q1 = __ldcg(p + 1);
    P[0] = q0.x; P[1] = q0.y; P[2] = q0.z; A = q1.w;
}

// Child c of a node, its moments: a leaf's exact ones, or an internal node's as stored, back in absolute units (fp64).
template <typename L>
__device__ __forceinline__ WnRec wn_child_rec(const WnNode* wn, const L* __restrict__ leaves, int c) {
    if (c < 0) return wn_leaf_rec(leaves, ~c);
    const float4* p = reinterpret_cast<const float4*>(wn + c);
    float x[24];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const float4 q = __ldcg(p + k);
        x[4 * k] = q.x; x[4 * k + 1] = q.y; x[4 * k + 2] = q.z; x[4 * k + 3] = q.w;
    }
    const double r1 = x[3], r2 = r1 * r1, r3 = r2 * r1, r4 = r2 * r2;
    WnRec r;
#pragma unroll
    for (int k = 0; k < 3; ++k) { r.P[k] = x[k]; r.N[k] = x[4 + k] * r2; }
    r.A = x[7];
#pragma unroll
    for (int k = 0; k < 6; ++k) r.M[k] = x[8 + k] * r3;
#pragma unroll
    for (int k = 0; k < 10; ++k) r.S[k] = x[14 + k] * r4;
    return r;
}

// Adds child r's moments, shifted from r.P to P (d = r.P - P): N += N_r; M_ij += M_r,ij + (N_i d_j + d_i N_j) / 2;
// Q_ijk += Q_r,ijk + (2/3)(d_i M_jk + d_j M_ik + d_k M_ij) + (1/3)(N_i d_j d_k + N_j d_i d_k + N_k d_i d_j), N and M the
// child's.
__device__ __forceinline__ void wn_shift_add(const WnRec& r, const double P[3], double N[3], double M[6], double S[10]) {
    const double d[3] = {r.P[0] - P[0], r.P[1] - P[1], r.P[2] - P[2]};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        N[i] += r.N[i];
#pragma unroll
        for (int j = i; j < 3; ++j) M[wn_m(i, j)] += r.M[wn_m(i, j)] + 0.5 * (r.N[i] * d[j] + d[i] * r.N[j]);
    }
#pragma unroll
    for (int t = 0; t < 10; ++t) {
        const int i = wn_s(t, 0), j = wn_s(t, 1), k = wn_s(t, 2);
        S[t] += r.S[t] + (2.0 / 3.0) * (d[i] * r.M[wn_m(j, k)] + d[j] * r.M[wn_m(i, k)] + d[k] * r.M[wn_m(i, j)]) +
                (1.0 / 3.0) * (r.N[i] * d[j] * d[k] + r.N[j] * d[i] * d[k] + r.N[k] * d[i] * d[j]);
    }
}

// One thread per leaf climbs towards the root; at each node the first arrival stops and the second, which finds both
// children complete, writes the node's area A (in fp32) and centre P: the area-weighted mean of the children's centres
// (their midpoint when both have zero area; a leaf's centre is its centroid, or its point), in fp64 rounded to fp32.
// r is left 0 for wn_radius_kernel.  `arrivals` starts at 0.
template <typename L>
__global__ void __launch_bounds__(kThreads) wn_centres_kernel(long long m, const MqScratch* __restrict__ sc,
                                                              const MqNode* __restrict__ nodes, const int* __restrict__ node_parent,
                                                              const int* __restrict__ leaf_parent, const L* __restrict__ leaves,
                                                              WnNode* wn, int* __restrict__ arrivals) {
    const long long n = m - (long long)sc->bad;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n < 2 || i >= n) return;
    int node = leaf_parent[i];
    while (true) {
        __threadfence();
        if (atomicAdd(&arrivals[node], 1) == 0) return;
        double P0[3], P1[3], A0, A1;
        wn_child_centre(wn, leaves, nodes[node].c0, P0, A0);
        wn_child_centre(wn, leaves, nodes[node].c1, P1, A1);
        const double A = A0 + A1;
        float P[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) P[k] = (float)(A > 0.0 ? (A0 * P0[k] + A1 * P1[k]) / A : 0.5 * (P0[k] + P1[k]));
        float4* p = reinterpret_cast<float4*>(wn + node);
        p[0] = make_float4(P[0], P[1], P[2], 0.f);
        p[1] = make_float4(0.f, 0.f, 0.f, (float)A);
        if (node == 0) return;
        node = node_parent[node];
    }
}

// r of every ancestor of leaf i, from the leaf's K fp32 points c (wn_leaf_points): the largest distance from the
// ancestor's P to one of them, in fp64 rounded up, then up to fp32; the maximum over the subtree's leaves is the same
// whatever order the atomics land in.
template <typename L>
__global__ void __launch_bounds__(kThreads) wn_radius_kernel(long long m, const MqScratch* __restrict__ sc,
                                                             const int* __restrict__ node_parent, const int* __restrict__ leaf_parent,
                                                             const L* __restrict__ leaves, WnNode* wn) {
    constexpr int K = kPointLeaf<L> ? 1 : 3;
    const long long n = mq_tree_size<L>(m, sc);
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n < 2 || i >= n) return;
    float c[K][3];
    wn_leaf_points(leaves, (int)i, c);
    int node = leaf_parent[i];
    while (true) {
        float* rec = reinterpret_cast<float*>(wn + node);
        double d2 = 0.0;
#pragma unroll
        for (int v = 0; v < K; ++v) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double d = fabs((double)c[v][k] - (double)rec[k]);   // exact: both are fp32 values
                s = __dadd_ru(s, __dmul_ru(d, d));
            }
            d2 = fmax(d2, s);
        }
        const int r = __float_as_int(__double2float_ru(__dsqrt_ru(d2)));   // >= 0: its bits order as the values
        if (r > *reinterpret_cast<volatile int*>(rec + 3)) atomicMax(reinterpret_cast<int*>(rec + 3), r);
        if (node == 0) return;
        node = node_parent[node];
    }
}

// The same climb after wn_radius_kernel (`arrivals` cleared again): the second arrival shifts both children's moments,
// child 0 then child 1, to the node's P in fp64 (an internal child's taken back from units of its own r), so what a
// node stores does not depend on which child arrived last, and writes them in units of the node's r.
template <typename L>
__global__ void __launch_bounds__(kThreads) wn_moments_kernel(long long m, const MqScratch* __restrict__ sc,
                                                              const MqNode* __restrict__ nodes, const int* __restrict__ node_parent,
                                                              const int* __restrict__ leaf_parent, const L* __restrict__ leaves,
                                                              WnNode* wn, int* __restrict__ arrivals) {
    const long long n = m - (long long)sc->bad;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n < 2 || i >= n) return;
    int node = leaf_parent[i];
    while (true) {
        __threadfence();
        if (atomicAdd(&arrivals[node], 1) == 0) return;
        const WnRec r0 = wn_child_rec(wn, leaves, nodes[node].c0), r1 = wn_child_rec(wn, leaves, nodes[node].c1);
        float4* p = reinterpret_cast<float4*>(wn + node);
        const float4 head = p[0];                         // P and r, from the earlier passes
        const double P[3] = {head.x, head.y, head.z};
        double N[3] = {0.0, 0.0, 0.0}, M[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, S[10];
#pragma unroll
        for (int t = 0; t < 10; ++t) S[t] = 0.0;
        wn_shift_add(r0, P, N, M, S);
        wn_shift_add(r1, P, N, M, S);
        // a node of radius 0 has every corner at P, so its moments are 0; a node of coincident points has N != 0, which
        // these units cannot hold: the point walk never takes its far field (wn_walk)
        const double i1 = head.w > 0.f ? 1.0 / (double)head.w : 0.0, i2 = i1 * i1, i3 = i2 * i1, i4 = i2 * i2;
        p[1] = make_float4((float)(N[0] * i2), (float)(N[1] * i2), (float)(N[2] * i2), (float)(r0.A + r1.A));
        p[2] = make_float4((float)(M[0] * i3), (float)(M[1] * i3), (float)(M[2] * i3), (float)(M[3] * i3));
        p[3] = make_float4((float)(M[4] * i3), (float)(M[5] * i3), (float)(S[0] * i4), (float)(S[1] * i4));
        p[4] = make_float4((float)(S[2] * i4), (float)(S[3] * i4), (float)(S[4] * i4), (float)(S[5] * i4));
        p[5] = make_float4((float)(S[6] * i4), (float)(S[7] * i4), (float)(S[8] * i4), (float)(S[9] * i4));
        if (node == 0) return;
        node = node_parent[node];
    }
}

// The signed solid angle of leaf j seen from q, in fp32 with every operation rounded on its own (van Oosterom and
// Strackee, with a, b, c the corners minus q, e1 = B - A, e2 = C - A):
//   Omega = 2 atan2(a.(e1 x e2), |a||b||c| + (a.b)|c| + (a.c)|b| + (b.c)|a|),
// and 0 when a corner's squared distance to q is 0 or the triple product is exactly 0.
template <typename T>
__device__ __forceinline__ float wn_leaf_omega(const Pt<T>* __restrict__ leaves, int j, const float q[3]) {
    using R = Real<float>;
    float A[3], B[3], C[3];
    wn_leaf_corners<T>(leaves, j, A, B, C);
    const float a[3] = {R::sub(A[0], q[0]), R::sub(A[1], q[1]), R::sub(A[2], q[2])};
    const float b[3] = {R::sub(B[0], q[0]), R::sub(B[1], q[1]), R::sub(B[2], q[2])};
    const float c[3] = {R::sub(C[0], q[0]), R::sub(C[1], q[1]), R::sub(C[2], q[2])};
    const float e1[3] = {R::sub(B[0], A[0]), R::sub(B[1], A[1]), R::sub(B[2], A[2])};
    const float e2[3] = {R::sub(C[0], A[0]), R::sub(C[1], A[1]), R::sub(C[2], A[2])};
    const float aa = mq_dot<float>(a[0], a[1], a[2], a[0], a[1], a[2]), bb = mq_dot<float>(b[0], b[1], b[2], b[0], b[1], b[2]),
                cc = mq_dot<float>(c[0], c[1], c[2], c[0], c[1], c[2]);
    if (aa == 0.f || bb == 0.f || cc == 0.f) return 0.f;
    const float nx = R::sub(R::mul(e1[1], e2[2]), R::mul(e1[2], e2[1]));
    const float ny = R::sub(R::mul(e1[2], e2[0]), R::mul(e1[0], e2[2]));
    const float nz = R::sub(R::mul(e1[0], e2[1]), R::mul(e1[1], e2[0]));
    const float det = mq_dot<float>(a[0], a[1], a[2], nx, ny, nz);
    if (det == 0.f) return 0.f;
    const float la = R::root(aa), lb = R::root(bb), lc = R::root(cc);
    const float den = R::add(R::add(R::add(R::mul(R::mul(la, lb), lc), R::mul(mq_dot<float>(a[0], a[1], a[2], b[0], b[1], b[2]), lc)),
                                    R::mul(mq_dot<float>(a[0], a[1], a[2], c[0], c[1], c[2]), lb)),
                             R::mul(mq_dot<float>(b[0], b[1], b[2], c[0], c[1], c[2]), la));
    return R::mul(2.f, atan2f(det, den));
}

// The dipole term of point j seen from q, Omega = an.d / |d|^3 with d = p - q, in fp32 with every operation rounded on
// its own, in this order:
//   d_k = p_k - q_k,  d2 = (dx dx + dy dy) + dz dz,  l = sqrt(d2),  t = ((an_x dx + an_y dy) + an_z dz) / l,
//   Omega = t / d2,
// and 0 when d2 = 0 (a query on the point).  Scaling p and q by 2^k and a by 2^2k scales d and l by 2^k, t by 2^2k and
// d2 by 2^2k, each exactly where nothing over- or underflows, so Omega keeps its bits.  The intermediate t is of the
// size of an, so only Omega itself can leave the fp32 range.
__device__ __forceinline__ float wn_leaf_omega(const WnPoint* __restrict__ leaves, int j, const float q[3]) {
    using R = Real<float>;
    const float4* s = reinterpret_cast<const float4*>(leaves + j);
    const float4 x = __ldg(s), an = __ldg(s + 1);
    const float dx = R::sub(x.x, q[0]), dy = R::sub(x.y, q[1]), dz = R::sub(x.z, q[2]);
    const float d2 = mq_dot<float>(dx, dy, dz, dx, dy, dz);
    if (d2 == 0.f) return 0.f;
    const float t = __fdiv_rn(mq_dot<float>(an.x, an.y, an.z, dx, dy, dz), R::root(d2));
    return __fdiv_rn(t, d2);
}

// The order-2 expansion of a node's solid angle, d = P - q, |d|^2 = d2 (Taylor expansion of y / |y|^3 about d):
//   N.d / |d|^3 + tr(M) / |d|^3 - 3 d.M.d / |d|^5 - (9/2) c.d / |d|^5 + (15/2) Q[d, d, d] / |d|^7,  c_k = sum_i Q_iik,
// evaluated as (N'.u) k^2 + (tr M' - 3 u.M'.u) k^3 + ((15/2) Q'[u, u, u] - (9/2) c'.u) k^4 with the unit direction
// u = d / |d|, k = r / |d| (< 1 / beta) and the stored moments N', M', Q' in units of r: every factor is of order 1
// whatever the mesh's scale, so nothing overflows or underflows in fp32.
__device__ __forceinline__ float wn_far(const WnNode* __restrict__ node, float dx, float dy, float dz, float d2, float r) {
    const float4* p = reinterpret_cast<const float4*>(node);
    const float4 n = __ldg(p + 1), m0 = __ldg(p + 2), m1 = __ldg(p + 3), s0 = __ldg(p + 4), s1 = __ldg(p + 5);
    const float Mxx = m0.x, Myy = m0.y, Mzz = m0.z, Mxy = m0.w, Mxz = m1.x, Myz = m1.y;
    const float Sxxx = m1.z, Syyy = m1.w, Szzz = s0.x, Sxxy = s0.y, Sxxz = s0.z, Sxyy = s0.w;
    const float Syyz = s1.x, Sxzz = s1.y, Syzz = s1.z, Sxyz = s1.w;
    const float ir = __frsqrt_rn(d2), ux = dx * ir, uy = dy * ir, uz = dz * ir;
    const float k = r * ir, k2 = k * k, k3 = k2 * k, k4 = k2 * k2;
    const float t0 = (n.x * ux + n.y * uy + n.z * uz) * k2;
    const float uMu = ux * (Mxx * ux + Mxy * uy + Mxz * uz) + uy * (Mxy * ux + Myy * uy + Myz * uz) +
                      uz * (Mxz * ux + Myz * uy + Mzz * uz);
    const float t1 = ((Mxx + Myy + Mzz) - 3.f * uMu) * k3;
    const float cu = (Sxxx + Sxyy + Sxzz) * ux + (Sxxy + Syyy + Syzz) * uy + (Sxxz + Syyz + Szzz) * uz;
    const float xx = ux * ux, yy = uy * uy, zz = uz * uz;
    const float uuu = ux * (Sxxx * xx + 3.f * (Sxyy * yy + Sxzz * zz)) + uy * (Syyy * yy + 3.f * (Sxxy * xx + Syzz * zz)) +
                      uz * (Szzz * zz + 3.f * (Sxxz * xx + Syyz * yy)) + 6.f * Sxyz * ux * uy * uz;
    const float t2 = (7.5f * uuu - 4.5f * cu) * k4;
    return (t0 + t1) + t2;
}

// w at q (fp32) for a tree of n leaves: the walk of the header, child 0 first, at most one node pushed per level
// (kMqStack holds the deepest path).  In a point tree a node of radius 0 (every point of its subtree at P, its N not
// held by WnNode's units) is always opened.
template <typename L>
__device__ __forceinline__ float wn_walk(const float q[3], long long n, const MqNode* __restrict__ nodes, const WnNode* __restrict__ wn,
                                         const L* __restrict__ leaves, float beta) {
    double acc = 0.0;
    if (n == 1) {
        acc = (double)wn_leaf_omega(leaves, 0, q);
    } else {
        int stack[kMqStack];
        int sp = 0, x = 0;
        while (true) {
            if (x < 0) {
                acc += (double)wn_leaf_omega(leaves, ~x, q);
            } else {
                const float4 pr = __ldg(reinterpret_cast<const float4*>(wn + x));
                const float dx = pr.x - q[0], dy = pr.y - q[1], dz = pr.z - q[2];
                const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                const float br = beta * pr.w;   // beta = inf, r = 0: NaN, never far
                if ((!kPointLeaf<L> || pr.w > 0.f) && d2 > br * br) {
                    acc += (double)wn_far(wn + x, dx, dy, dz, d2, pr.w);
                } else {
                    const int2 c = __ldg(reinterpret_cast<const int2*>(&nodes[x].c0));
                    stack[sp++] = c.y;
                    x = c.x;
                    continue;
                }
            }
            if (sp == 0) break;
            x = stack[--sp];
        }
    }
    return __double2float_rn(__ddiv_rn(acc, 4.0 * 3.141592653589793));
}

// The face walk is not inlined, so the winding-number and the signed-distance kernels run the very same code and get the
// same bits; the point walk is inlined into wn_query_kernel.
template <typename T>
__device__ __noinline__ float wn_eval(const float q[3], long long n, const MqNode* __restrict__ nodes, const WnNode* __restrict__ wn,
                                      const Pt<T>* __restrict__ leaves, float beta) {
    return wn_walk(q, n, nodes, wn, leaves, beta);
}
__device__ __forceinline__ float wn_eval(const float q[3], long long n, const MqNode* __restrict__ nodes, const WnNode* __restrict__ wn,
                                         const WnPoint* __restrict__ leaves, float beta) {
    return wn_walk(q, n, nodes, wn, leaves, beta);
}

template <typename T>
__device__ __forceinline__ void wn_query_point(const T* q, long long i, float out[3]) {
    out[0] = (float)q[3 * i]; out[1] = (float)q[3 * i + 1]; out[2] = (float)q[3 * i + 2];
}

// Query i in input order; nothing is written when a face tree is empty (every face invalid: the caller raises).  A point
// tree is never empty (the caller handles m = 0 without one).
template <typename T, typename L>
__global__ void __launch_bounds__(kThreads) wn_query_kernel(const T* __restrict__ q, long long nq, long long m,
                                                            const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                            const WnNode* __restrict__ wn, const L* __restrict__ leaves,
                                                            float beta, T* __restrict__ out_w) {
    const long long n = mq_tree_size<L>(m, sc);
    if (!kPointLeaf<L> && n < 1) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += (long long)gridDim.x * blockDim.x) {
        float p[3];
        wn_query_point<T>(q, i, p);
        out_w[i] = (T)wn_eval(p, n, nodes, wn, leaves, beta);
    }
}

// Signed distance of query i, after mq_query_kernel left d in out_s, the face in out_fidx (int32) and bc.  d^2 is
// recomputed bit for bit from that face (closest_on_face is a pure function of the query and the corners; a query that
// matched no face has d^2 = inf).  Out of band (d^2 >= up or d^2 < low): s = NaN, fi = m + 1, bc = NaN, and no walk.
// Otherwise s = fl_T(sigma d), sigma = fl_T(1 - 2|w|) with the fp64 expression of libigl and w = (T) wn_eval.
template <typename T>
__global__ void __launch_bounds__(kThreads) sd_sign_kernel(const T* __restrict__ p, long long np, const T* __restrict__ v, long long nv,
                                                           const void* __restrict__ f, int fkind, long long m,
                                                           const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                           const WnNode* __restrict__ wn, const Pt<T>* __restrict__ leaves, float beta,
                                                           T up, T low,
                                                           T* __restrict__ out_s, int* __restrict__ out_fidx, T* __restrict__ out_bc) {
    const long long n = m - (long long)sc->bad;
    if (n < 1) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (long long)gridDim.x * blockDim.x) {
        const T q[3] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
        const int fi = out_fidx[i];
        T d2 = Real<T>::inf();
        double a[3], b[3], c[3];
        if (fi >= 0 && mq_corners<T>(v, nv, f, fkind, fi, a, b, c)) {
            const T ta[3] = {(T)a[0], (T)a[1], (T)a[2]}, tb[3] = {(T)b[0], (T)b[1], (T)b[2]}, tc[3] = {(T)c[0], (T)c[1], (T)c[2]};
            d2 = closest_on_face<T>(q, ta, tb, tc, mq_degenerate<T>(a, b, c)).d2;
        }
        if (d2 >= up || d2 < low) {
            const T nan = (T)__int_as_float(0x7fffffff);
            out_s[i] = nan;
            out_fidx[i] = (int)(m + 1);
            out_bc[3 * i] = nan; out_bc[3 * i + 1] = nan; out_bc[3 * i + 2] = nan;
            continue;
        }
        float qf[3];
        wn_query_point<T>(p, i, qf);
        const T w = (T)wn_eval<T>(qf, n, nodes, wn, leaves, beta);
        const T sigma = (T)(1.0 - 2.0 * fabs((double)w));
        out_s[i] = Real<T>::mul(sigma, out_s[i]);
    }
}

// ---- oriented point clouds (point_cloud_fast_winding_number, DESIGN.md §3) -------------------------------------------
// The leaves pass of a point tree, in place of mq_leaves_kernel.  Leaf i: the fp32 point, |a| and an_k = fl32(fl_T(a n_k)).
// a is read as a flat array of m values.
template <typename T>
__global__ void __launch_bounds__(kThreads) wn_point_leaves_kernel(const T* __restrict__ p, const T* __restrict__ nrm, const T* __restrict__ a,
                                                                   long long m, const MqRec* __restrict__ sorted, WnPoint* __restrict__ leaves) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const long long t = (long long)sorted[i].idx;
    float x[3];
    wn_query_point<T>(p, t, x);
    const T ai = a[t];
    const float an0 = (float)Real<T>::mul(ai, nrm[3 * t]), an1 = (float)Real<T>::mul(ai, nrm[3 * t + 1]),
                an2 = (float)Real<T>::mul(ai, nrm[3 * t + 2]);
    float4* s = reinterpret_cast<float4*>(leaves + i);
    s[0] = make_float4(x[0], x[1], x[2], fabsf((float)ai));
    s[1] = make_float4(an0, an1, an2, 0.f);
}

}  // namespace pcu
