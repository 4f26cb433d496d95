// raycast.cuh -- rays against a triangle mesh (ray_mesh_intersection / RayMeshIntersector of the reference,
// src/ray_mesh_intersection.cpp, one Embree ray at a time), and rays against surfels (ray_surfel_intersection /
// RaySurfelIntersector, src/ray_point_cloud_intersection.cpp: the same test on each point's fan, rs_query_kernel below).
//
// The result is defined exactly (DESIGN.md §3, ray casting) as a pure function of (v, f, o_i, d_i, near, far):
//   rounding          corners, origin, direction, near and far are rounded to fp32 whatever the input precision
//   per (ray, face)   the watertight test of Woop, Benthin and Wald (JCGT 2013) in fp32, every operation rounded on
//                     its own (rc_face below); both sides of a face count
//   per ray           the lexicographic minimum of (t, face index) over the faces with every corner in [0, #v) and
//                     near < t <= far; a zero or non-finite origin or direction hits nothing
// The walk runs on the tree of meshquery.cuh, one thread per ray; rc_box prunes with the margin of §3.
#pragma once
#include "meshquery.cuh"

namespace pcu {

// The per-ray constants: the fp32 origin, the permuted axes and shear of Woop et al., and for the box test the
// reciprocal direction, the per-axis margin m_k = 2^-19 R / |d_k| and the spatial margin delta = 2^-20 R (DESIGN.md §3),
// R bounding |x_k - o_k| over the scene box.  mode[k]: 0 d_k = 0, 1 |d_k| < 2^-100 (axis left unconstrained), 2 slab.
struct RcRay {
    float o[3];
    int kx, ky, kz;
    float sx, sy, sz;
    float inv[3], m[3];
    int mode[3];
    float delta;
};

__device__ __forceinline__ float rc_pick(const float a[3], int k) { return k == 0 ? a[0] : (k == 1 ? a[1] : a[2]); }

// Woop et al.'s test for corners a, b, c: true on a hit with near < t, t, b1 = V / det and b2 = W / det.
__device__ __forceinline__ bool rc_face(const RcRay& r, const float a[3], const float b[3], const float c[3], float near,
                                        float& t, float& b1, float& b2) {
    const float A[3] = {__fsub_rn(a[0], r.o[0]), __fsub_rn(a[1], r.o[1]), __fsub_rn(a[2], r.o[2])};
    const float B[3] = {__fsub_rn(b[0], r.o[0]), __fsub_rn(b[1], r.o[1]), __fsub_rn(b[2], r.o[2])};
    const float C[3] = {__fsub_rn(c[0], r.o[0]), __fsub_rn(c[1], r.o[1]), __fsub_rn(c[2], r.o[2])};
    const float Akz = rc_pick(A, r.kz), Bkz = rc_pick(B, r.kz), Ckz = rc_pick(C, r.kz);
    const float Ax = __fsub_rn(rc_pick(A, r.kx), __fmul_rn(r.sx, Akz)), Ay = __fsub_rn(rc_pick(A, r.ky), __fmul_rn(r.sy, Akz));
    const float Bx = __fsub_rn(rc_pick(B, r.kx), __fmul_rn(r.sx, Bkz)), By = __fsub_rn(rc_pick(B, r.ky), __fmul_rn(r.sy, Bkz));
    const float Cx = __fsub_rn(rc_pick(C, r.kx), __fmul_rn(r.sx, Ckz)), Cy = __fsub_rn(rc_pick(C, r.ky), __fmul_rn(r.sy, Ckz));
    float U = __fsub_rn(__fmul_rn(Cx, By), __fmul_rn(Cy, Bx));
    float V = __fsub_rn(__fmul_rn(Ax, Cy), __fmul_rn(Ay, Cx));
    float W = __fsub_rn(__fmul_rn(Bx, Ay), __fmul_rn(By, Ax));
    if (U == 0.f || V == 0.f || W == 0.f) {   // the paper's fallback: the fp32 products are exact in fp64
        U = __double2float_rn(__dsub_rn(__dmul_rn((double)Cx, (double)By), __dmul_rn((double)Cy, (double)Bx)));
        V = __double2float_rn(__dsub_rn(__dmul_rn((double)Ax, (double)Cy), __dmul_rn((double)Ay, (double)Cx)));
        W = __double2float_rn(__dsub_rn(__dmul_rn((double)Bx, (double)Ay), __dmul_rn((double)By, (double)Ax)));
    }
    if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) return false;
    const float det = __fadd_rn(__fadd_rn(U, V), W);
    if (det == 0.f) return false;
    const float Az = __fmul_rn(r.sz, Akz), Bz = __fmul_rn(r.sz, Bkz), Cz = __fmul_rn(r.sz, Ckz);
    const float T = __fadd_rn(__fadd_rn(__fmul_rn(U, Az), __fmul_rn(V, Bz)), __fmul_rn(W, Cz));
    t = __fdiv_rn(T, det);
    if (!(near < t)) return false;
    b1 = __fdiv_rn(V, det);
    b2 = __fdiv_rn(W, det);
    return true;
}

// Whether the box can hold a face whose computed t lies in (near, best] (DESIGN.md §3): the slabs widened by m_k
// must overlap, and the kz slab's interval, in which every computed t of a face inside lies, must reach past near.
// `lb` gets the kz slab's lower end, a lower bound of every such t.
__device__ __forceinline__ bool rc_box(const RcRay& r, const float lo[3], const float hi[3], float near, float& lb) {
    const float inf = __int_as_float(0x7f800000);
    float enter = -inf, exit = inf, zlo = -inf, zhi = inf;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float a = -inf, b = inf;
        if (r.mode[k] == 0) {
            const bool in = __fsub_rd(lo[k], r.delta) <= r.o[k] && r.o[k] <= __fadd_ru(hi[k], r.delta);
            a = in ? -inf : inf;
            b = in ? inf : -inf;
        } else if (r.mode[k] == 2) {
            const float ta = __fmul_rn(__fsub_rn(lo[k], r.o[k]), r.inv[k]), tb = __fmul_rn(__fsub_rn(hi[k], r.o[k]), r.inv[k]);
            a = __fsub_rd(fminf(ta, tb), r.m[k]);
            b = __fadd_ru(fmaxf(ta, tb), r.m[k]);
        }
        enter = fmaxf(enter, a);
        exit = fminf(exit, b);
        if (k == r.kz) { zlo = a; zhi = b; }
    }
    lb = zlo;
    return enter <= exit && zhi > near;
}

// Largest |coordinate| of the scene box, which covers every leaf's box.
__device__ __forceinline__ float rc_scene(const MqScratch* __restrict__ sc) {
    float scene = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) scene = fmaxf(scene, fabsf(mq_unord(sc->scene[k])));
    return scene;
}

// Ray (oi, di) rounded to fp32 into o and dir; false for a zero or non-finite origin or direction.
template <typename TR>
__device__ __forceinline__ bool rc_round(const TR* oi, const TR* di, float o[3], float dir[3]) {
    bool valid = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        o[k] = (float)oi[k];
        dir[k] = (float)di[k];
        valid = valid && isfinite(o[k]) && isfinite(dir[k]);
    }
    return valid && (dir[0] != 0.f || dir[1] != 0.f || dir[2] != 0.f);
}

// The constants of a valid ray (r.o, dir).  Where a kernel calls it decides its register allocation (nvcc 12.9,
// sm_90a): rc_query_kernel calls it inside the branch that walks, since set up ahead of that branch it spills;
// rs_query_kernel sets up ahead, which is how it reaches 64 registers and its measured speed (DESIGN.md §4).
__device__ __forceinline__ void rc_ray(const float dir[3], float scene, RcRay& r) {
    r.kz = 0;
    if (fabsf(dir[1]) > fabsf(dir[r.kz])) r.kz = 1;
    if (fabsf(dir[2]) > fabsf(dir[r.kz])) r.kz = 2;
    r.kx = r.kz == 2 ? 0 : r.kz + 1;
    r.ky = r.kx == 2 ? 0 : r.kx + 1;
    const float dz = rc_pick(dir, r.kz);
    if (dz < 0.f) { const int s = r.kx; r.kx = r.ky; r.ky = s; }
    r.sx = __fdiv_rn(rc_pick(dir, r.kx), dz);
    r.sy = __fdiv_rn(rc_pick(dir, r.ky), dz);
    r.sz = __fdiv_rn(1.f, dz);
    const float R = __fadd_ru(fmaxf(fabsf(r.o[0]), fmaxf(fabsf(r.o[1]), fabsf(r.o[2]))), scene);
    r.delta = __fmul_ru(R, 0x1p-20f);
    const float R19 = __fmul_ru(R, 0x1p-19f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float ad = fabsf(dir[k]);
        r.mode[k] = ad == 0.f ? 0 : (ad < 0x1p-100f ? 1 : 2);
        r.inv[k] = __fdiv_rn(1.f, dir[k]);
        r.m[k] = __fdiv_ru(R19, ad);
    }
}

// The walk over a tree of n >= 1 leaves: leaf(l) for every leaf whose box rc_box keeps with its lower bound not past
// best, which leaf() may lower; nearer child first, the other pushed with its bound.
template <typename F>
__device__ __forceinline__ void rc_walk(const RcRay& r, const MqNode* __restrict__ nodes, long long n, float near, const float& best,
                                        F&& leaf) {
    if (n == 1) {
        leaf(0);
        return;
    }
    int stack[kMqStack];
    float stack_lb[kMqStack];
    int sp = 0, node = 0;
    while (true) {
        const float4* np_ = reinterpret_cast<const float4*>(nodes + node);
        const float4 q0 = __ldg(np_), q1 = __ldg(np_ + 1), q2 = __ldg(np_ + 2), q3 = __ldg(np_ + 3);
        const float lo0[3] = {q0.x, q0.y, q0.z}, hi0[3] = {q0.w, q1.x, q1.y};
        const float lo1[3] = {q1.z, q1.w, q2.x}, hi1[3] = {q2.y, q2.z, q2.w};
        const int c0 = __float_as_int(q3.x), c1 = __float_as_int(q3.y);
        float l0, l1;
        bool k0 = rc_box(r, lo0, hi0, near, l0) && !(l0 > best);
        bool k1 = rc_box(r, lo1, hi1, near, l1) && !(l1 > best);
        if (k0 && c0 < 0) { leaf(~c0); k0 = false; }
        if (k1 && c1 < 0) { leaf(~c1); k1 = false; }
        k0 = k0 && !(l0 > best);
        k1 = k1 && !(l1 > best);
        if (k0 && k1) {
            const bool first0 = l0 <= l1;
            stack[sp] = first0 ? c1 : c0;
            stack_lb[sp] = first0 ? l1 : l0;
            ++sp;
            node = first0 ? c0 : c1;
            continue;
        }
        if (k0) { node = c0; continue; }
        if (k1) { node = c1; continue; }
        node = -1;
        while (sp > 0) {
            --sp;
            if (!(stack_lb[sp] > best)) { node = stack[sp]; break; }
        }
        if (node < 0) break;
    }
}

// Ray i: origin o + i * o_stride (o_stride 0: one origin for every ray), direction d + 3 i.  fidx_wide: 8-byte face
// indices (f's width), else 4-byte.  Misses get fidx = -1, t = +inf, bc = 0.  Nothing is written when the tree is
// empty (every face invalid: the caller raises).  Per visit one 64-byte node; per face tested three Pt<TM>.
template <typename TR, typename TM>
__global__ void __launch_bounds__(kThreads) rc_query_kernel(const TR* __restrict__ o, int o_stride, const TR* __restrict__ d,
                                                            long long nr, float near, float far, long long m,
                                                            const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                            const Pt<TM>* __restrict__ leaves, void* __restrict__ out_fidx,
                                                            int fidx_wide, TR* __restrict__ out_bc, TR* __restrict__ out_t) {
    const long long n = m - (long long)sc->bad;
    if (n < 1) return;
    const float scene = rc_scene(sc);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += (long long)gridDim.x * blockDim.x) {
        RcRay r;
        float dir[3];
        float best = far, bb1 = 0.f, bb2 = 0.f;
        long long best_face = LLONG_MAX;
        if (rc_round<TR>(o + (long long)o_stride * i, d + 3 * i, r.o, dir)) {
            rc_ray(dir, scene, r);
            rc_walk(r, nodes, n, near, best, [&](int l) {
                const Pt<TM> A = leaves[3 * l], B = leaves[3 * l + 1], C = leaves[3 * l + 2];
                const float a[3] = {(float)A.x, (float)A.y, (float)A.z}, b[3] = {(float)B.x, (float)B.y, (float)B.z},
                            c[3] = {(float)C.x, (float)C.y, (float)C.z};
                float t, b1, b2;
                if (!rc_face(r, a, b, c, near, t, b1, b2)) return;
                const long long face = (long long)A.i;
                if (t < best || (t == best && face < best_face)) { best = t; best_face = face; bb1 = b1; bb2 = b2; }
            });
        }
        const bool hit = best_face != LLONG_MAX;
        if (fidx_wide) ((long long*)out_fidx)[i] = hit ? best_face : -1ll;
        else ((int*)out_fidx)[i] = hit ? (int)best_face : -1;
        out_t[i] = hit ? (TR)best : (TR)__int_as_float(0x7f800000);
        out_bc[3 * i] = hit ? (TR)__dsub_rn(__dsub_rn(1.0, (double)bb1), (double)bb2) : (TR)0;
        out_bc[3 * i + 1] = hit ? (TR)bb1 : (TR)0;
        out_bc[3 * i + 2] = hit ? (TR)bb2 : (TR)0;
    }
}

// Rays against surfels (ray_surfel_intersection, DESIGN.md §3): the walk of rc_query_kernel over a surfel tree of
// m points (meshquery.cuh, leaves SfWord of s-triangle fans).  At a leaf the s triangles (centre, rim j, rim
// (j + 1) mod s) are tested with rc_face, each triangle loading its three corners (L1 hits after the first), so no
// corner stays live across triangles.  The first hit by (t, point id) wins.  Misses, an empty tree (m = 0, or every fan non-finite) and invalid rays give pid = -1, t = +inf.  Per visit
// one 64-byte node; per surfel tested sf_words(s) 16-byte words and one id.
template <typename TR>
__global__ void __launch_bounds__(kThreads) rs_query_kernel(const TR* __restrict__ o, int o_stride, const TR* __restrict__ d,
                                                            long long nr, float near, float far, long long m, int s,
                                                              const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                              const SfWord* __restrict__ leaves, const int* __restrict__ ids,
                                                            int* __restrict__ out_pid, TR* __restrict__ out_t) {
    const long long n = m > 0 ? m - (long long)sc->bad : 0;
    const float scene = n > 0 ? rc_scene(sc) : 0.f;
    const long long words = sf_words(s);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += (long long)gridDim.x * blockDim.x) {
        RcRay r;
        float best = far;
        int best_pid = INT_MAX;
        const auto ahead = [&]() {   // the setup ahead of the walk's branch, dir scoped to it (see rc_ray)
            float dir[3];
            if (!rc_round<TR>(o + (long long)o_stride * i, d + 3 * i, r.o, dir)) return false;
            rc_ray(dir, scene, r);
            return true;
        };
        if (n > 0 && ahead()) {
            rc_walk(r, nodes, n, near, best, [&](int l) {
                const float* q = reinterpret_cast<const float*>(leaves + (long long)l * words);
                const int pid = __ldg(ids + l);
                for (int j = 0; j < s; ++j) {   // every corner reloaded (L1 hits): nothing held across triangles
                    const float* u = q + 3 * (j + 1);
                    const float* w = q + (j + 1 < s ? 3 * (j + 2) : 3);
                    const float centre[3] = {__ldg(q), __ldg(q + 1), __ldg(q + 2)};
                    const float a[3] = {__ldg(u), __ldg(u + 1), __ldg(u + 2)}, b[3] = {__ldg(w), __ldg(w + 1), __ldg(w + 2)};
                    float t, b1, b2;
                    if (rc_face(r, centre, a, b, near, t, b1, b2) && (t < best || (t == best && pid < best_pid))) {
                        best = t;
                        best_pid = pid;
                    }
                }
            });
        }
        const bool hit = best_pid != INT_MAX;
        out_pid[i] = hit ? best_pid : -1;
        out_t[i] = hit ? (TR)best : (TR)__int_as_float(0x7f800000);
    }
}

}  // namespace pcu
