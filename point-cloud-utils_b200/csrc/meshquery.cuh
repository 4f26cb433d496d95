// meshquery.cuh -- closest points on a triangle mesh (closest_points_on_mesh of the reference,
// src/closest_point_on_mesh.cpp, which walks libigl's AABB tree).
//
// The result is defined exactly (DESIGN.md §3, point-to-mesh distance) as a pure function of (p, v, f):
//   per (query, face)  the Voronoi-region closest point of Ericson, Real-Time Collision Detection §5.1.5, in the input
//                      precision T with every operation rounded on its own (closest_on_face below); faces whose
//                      interior denominator D = (e1.e1)(e2.e2) - (e1.e2)^2 is not positive are the union of their edges.
//   per query          the lexicographic minimum of (d^2, face index) over the faces with every corner in [0, #v);
//                      d = sqrt(d^2) rounded once, bc the chosen face's coordinates.
// So neither the tree's shape, nor the sort, nor thread scheduling can change a result.
//
// The tree is a linear BVH (Karras 2012), built per call by one sequence over either leaf kind L:
//   faces   L = Pt<T>, three per leaf (corners, face id, degeneracy); a face with a corner out of range is invalid: it is
//           counted in MqScratch::bad and sorts last, out of the tree; leaves have boxes and the nodes are refit
//   points  L = WnPoint (point_cloud_fast_winding_number, winding.cuh), one per leaf, always valid; no boxes, no refit
//   surfels L = SfWord (ray_surfel_intersection, raycast.cuh), a whole fp32 fan per leaf (sf_fan); a fan with a
//           non-finite coordinate is invalid, counted and left out as a face is; leaves have boxes and the nodes are refit
//   balls   L = RvBall (sample_mesh_lloyd, rvd.cuh), one face's candidate ball per leaf; a ball without a radius is
//           invalid, counted and left out as a face is; leaves have boxes and the nodes are refit
// The passes:
//   mq_bounds_kernel    scene box of the leaves' boxes (a point's box is the point), count of invalid faces
//   mq_codes_kernel     63-bit Morton code of each face's box centre or each fp32 point over the scene box (invalid
//                       faces: ~0, last)
//   (sort.cuh)          stable radix sort of (code, leaf): equal codes stay in input order
//   mq_leaves_kernel    corners packed in leaf order (face id and degeneracy in the spare lanes), leaf boxes; points:
//                       wn_point_leaves_kernel
//   mq_nodes_kernel     Karras's internal nodes; equal codes are split by position (delta = 64 + clz(i ^ j))
//   mq_refit_kernel     faces: bottom-up boxes with per-node arrival counters: the second child to arrive writes both
//                       children's boxes into the parent (one 64-byte record per visit)
//   mq_query_kernel     one thread per query: nearer child first, the other pushed; pruning with the margin of §3.
// mesh_query.cu builds and queries every tree; the passes that are not templates (mq_nodes_kernel, mq_refit_kernel,
// rv_ball_leaves_kernel, sf_upload_kernel) are defined there, and the other families include this header for its types.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "meshsample.cuh"
#include "morton.cuh"
#include "sort.cuh"

namespace pcu {

using MqRec = SortRec<unsigned long long, 1>;

// Tree depth bound: along a root-to-leaf path the nodes' common-prefix lengths strictly increase.  They lie in
// [1, 63] for distinct codes (codes are < 2^63, so two of them share at least the top bit) and in [65, 95] for equal
// codes (64 + clz(i ^ j) with 0 < i ^ j < 2^31), so a path has at most 63 + 31 = 94 internal nodes.  Traversal pushes
// at most one node per internal node of the current path, so this stack cannot overflow.
constexpr int kMqStack = 96;

// Both children of an internal node: their boxes (fp32, rounded outward and widened, §3) and their ids (>= 0: internal
// node, < 0: ~leaf position).
struct __align__(16) MqNode {
    float lo0[3], hi0[3], lo1[3], hi1[3];
    int c0, c1, pad0, pad1;
};
struct MqBox { float lo[3], hi[3]; };

// A point leaf of point_cloud_fast_winding_number, one per input point in tree order: the point, its weight |a| and
// an = a n (fp32, an rounded once from T), 32 bytes whatever the input precision.
struct __align__(16) WnPoint {
    float p[3], w;
    float an[3], pad;
};
static_assert(sizeof(WnPoint) == 32, "two float4 per point");

template <typename L>
constexpr bool kPointLeaf = std::is_same<L, WnPoint>::value;

// 16 bytes of a surfel leaf of ray_surfel_intersection (raycast.cuh).  Leaf l is sf_words(s) words from word
// l sf_words(s): its fan's s + 1 fp32 vertices (the centre, then rim 0 .. s - 1), x y z each, zero-padded to whole
// words (96 B at s = 7); its point id lives in MeshTree::ids.  A surfel whose fan has a non-finite coordinate is
// counted in MqScratch::bad and sorts last, out of the tree, as an invalid face does.
struct __align__(16) SfWord { float x[4]; };

template <typename L>
constexpr bool kSurfelLeaf = std::is_same<L, SfWord>::value;

__host__ __device__ __forceinline__ long long sf_words(int s) { return (3ll * (s + 1) + 3) / 4; }

// A ball leaf of the restricted Voronoi pairs (rvd.cuh): a face's candidate ball, centre and radius in fp64.  The
// build's input v is the (m, 4) array of balls; a ball whose radius is not >= 0 (NaN: a face that meets no cell) is
// invalid, counted in MqScratch::bad and left out of the tree as an invalid face is.  The leaf's face id lives in
// MeshTree::ids; its box is the ball's, rounded outward to fp32.
struct __align__(16) RvBall { double c[3], r; };

template <typename L>
constexpr bool kBallLeaf = std::is_same<L, RvBall>::value;

// What a surfel fan is computed from: normals and radii (T, as the points), s and the table cs[2 j] = fl32(cos
// theta_j), cs[2 j + 1] = fl32(sin theta_j), computed on the host (DESIGN.md §3, ray-surfel casting).  During a tree
// build `boxes` holds each surfel's box in input order: mq_bounds_kernel writes it (lo[0] = NaN for a non-finite
// fan) and mq_codes_kernel reads it, so the fan is not computed again there.
struct SfSrc {
    const void* n;
    const void* r;
    const float* cs;
    MqBox* boxes;
    int s;
};

// Moves the host-computed table (and the SfSrc record, for the bounds and codes passes) to the device through kernel
// parameters, so no host buffer is copied: each launch writes `count` <= kSfChunk values of the table at `dst` and,
// when `dst_src` is set, the record there.
constexpr int kSfChunk = 960;
struct SfUpload {
    SfSrc* dst_src;
    SfSrc src;
    float* dst;
    int count;
    float v[kSfChunk];
};
static_assert(sizeof(SfUpload) <= 4096, "within the kernel parameter limit");

template <typename C> __device__ __forceinline__ C sf_div(C a, C b);
template <> __device__ __forceinline__ float sf_div<float>(float a, float b) { return __fdiv_rn(a, b); }
template <> __device__ __forceinline__ double sf_div<double>(double a, double b) { return __ddiv_rn(a, b); }

// a x b, each product and difference rounded on its own.
template <typename C>
__device__ __forceinline__ void sf_cross(const C a[3], const C b[3], C out[3]) {
    using R = Real<C>;
    out[0] = R::sub(R::mul(a[1], b[2]), R::mul(a[2], b[1]));
    out[1] = R::sub(R::mul(a[2], b[0]), R::mul(a[0], b[2]));
    out[2] = R::sub(R::mul(a[0], b[1]), R::mul(a[1], b[0]));
}

// a / |a|, |a| = sqrt((a0^2 + a1^2) + a2^2).
template <typename C>
__device__ __forceinline__ void sf_unit(C a[3]) {
    using R = Real<C>;
    const C l = R::root(R::add(R::add(R::mul(a[0], a[0]), R::mul(a[1], a[1])), R::mul(a[2], a[2])));
    for (int k = 0; k < 3; ++k) a[k] = sf_div<C>(a[k], l);
}

// Surfel i's fan in the compute precision C (float for rays, T for pointcloud_surfel_geometry): emit(j, x, y, z) for
// rim vertex j = 0 .. s - 1, then emit(s, p_i) for the centre.  The reference's local_basis and generate_splat_geometry
// op by op (DESIGN.md §3): n^ = n / |n|; right = n^ x e_x when | |(0 n^_x + 1 n^_y) + 0 n^_z| - 1 | < 1e-5 (in fp64),
// else n^ x e_y; right and up = n^ x right normalised; x0 = fl32(r_i c_j), y0 = fl32(r_i s_j) with the products in T;
// row k = ((right_k x0 + up_k y0) + n^_k 0) + p_k.
template <typename T, typename C, typename F>
__device__ __forceinline__ void sf_fan(const T* __restrict__ p, const SfSrc& src, long long i, F&& emit) {
    using R = Real<C>;
    const T* n = (const T*)src.n;
    C nh[3] = {(C)n[3 * i], (C)n[3 * i + 1], (C)n[3 * i + 2]};
    const C c[3] = {(C)p[3 * i], (C)p[3 * i + 1], (C)p[3 * i + 2]};
    sf_unit<C>(nh);
    const C dot = R::add(R::add(R::mul((C)0, nh[0]), R::mul((C)1, nh[1])), R::mul((C)0, nh[2]));
    const bool near_y = fabs((double)fabs(dot) - 1.0) < 1e-5;
    const C axis[3] = {near_y ? (C)1 : (C)0, near_y ? (C)0 : (C)1, (C)0};
    C right[3], up[3];
    sf_cross<C>(nh, axis, right);
    sf_unit<C>(right);
    sf_cross<C>(nh, right, up);
    sf_unit<C>(up);
    const T ri = ((const T*)src.r)[i];
    for (int j = 0; j < src.s; ++j) {
        const float x0 = (float)Real<T>::mul(ri, (T)src.cs[2 * j]), y0 = (float)Real<T>::mul(ri, (T)src.cs[2 * j + 1]);
        C v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            v[k] = R::add(R::add(R::add(R::mul(right[k], (C)x0), R::mul(up[k], (C)y0)), R::mul(nh[k], (C)0)), c[k]);
        emit(j, v[0], v[1], v[2]);
    }
    emit(src.s, c[0], c[1], c[2]);
}

// The surfel's fp32 box (the min / max of its fan's vertices); false when a fan coordinate is not finite.
template <typename T>
__device__ __forceinline__ bool sf_box(const T* __restrict__ p, const SfSrc& src, long long i, MqBox& bx) {
    const float inf = __int_as_float(0x7f800000);
    bool finite = true;
    for (int k = 0; k < 3; ++k) { bx.lo[k] = inf; bx.hi[k] = -inf; }
    sf_fan<T, float>(p, src, i, [&](int, float x, float y, float z) {
        finite = finite && isfinite(x) && isfinite(y) && isfinite(z);
        bx.lo[0] = fminf(bx.lo[0], x); bx.lo[1] = fminf(bx.lo[1], y); bx.lo[2] = fminf(bx.lo[2], z);
        bx.hi[0] = fmaxf(bx.hi[0], x); bx.hi[1] = fmaxf(bx.hi[1], y); bx.hi[2] = fmaxf(bx.hi[2], z);
    });
    return finite;
}

struct MqScratch {
    int scene[6];                 // ordered-int images of the scene box (min x y z, max x y z)
    unsigned long long bad;       // faces with a corner out of range: left out of the tree, counted for the caller
};

struct WnNode;   // winding.cuh

// A tree as mesh_query.cu's builder leaves it, in device memory.
template <typename L>
struct MeshTree {
    MqScratch* sc;
    MqNode* nodes;
    L* leaves;
    WnNode* wn;   // far-field data per node (with `moments` only)
    int* ids;     // surfel leaves: the point id of each leaf
};

// Leaves in the tree: m less the invalid faces, counted by mq_bounds_kernel (a point tree has none).
template <typename L>
__device__ __forceinline__ long long mq_tree_size(long long m, const MqScratch* sc) {
    return kPointLeaf<L> ? m : m - (long long)sc->bad;
}

__device__ __forceinline__ int mq_ord(float x) { const int b = __float_as_int(x); return b >= 0 ? b : b ^ 0x7fffffff; }
__device__ __forceinline__ float mq_unord(int b) { return __int_as_float(b >= 0 ? b : b ^ 0x7fffffff); }

// The face's corners when all three are in range.
template <typename T>
__device__ __forceinline__ bool mq_corners(const T* v, long long nv, const void* f, int fkind, long long t, double a[3],
                                           double b[3], double c[3]) {
    const long long i0 = load_index(f, 3 * t, fkind, nv, false), i1 = load_index(f, 3 * t + 1, fkind, nv, false),
                    i2 = load_index(f, 3 * t + 2, fkind, nv, false);
    if (i0 < 0 || i1 < 0 || i2 < 0) return false;
    load_vertex<T>(v, i0, a); load_vertex<T>(v, i1, b); load_vertex<T>(v, i2, c);
    return true;
}

// The face's box, widened by mu = 16 u M per side (u: unit roundoff of T, M: largest corner magnitude) and rounded
// outward to fp32.  DESIGN.md §3 shows that every closest point closest_on_face computes lies inside it.
template <typename T>
__device__ __forceinline__ MqBox mq_face_box(const double a[3], const double b[3], const double c[3]) {
    const double u = sizeof(T) == 4 ? 0x1p-24 : 0x1p-53;
    double M = 0.0;
    for (int k = 0; k < 3; ++k) M = fmax(M, fmax(fabs(a[k]), fmax(fabs(b[k]), fabs(c[k]))));
    const double mu = M * (16.0 * u);
    MqBox bx;
    for (int k = 0; k < 3; ++k) {
        bx.lo[k] = __double2float_rd(__dsub_rd(fmin(a[k], fmin(b[k], c[k])), mu));
        bx.hi[k] = __double2float_ru(__dadd_ru(fmax(a[k], fmax(b[k], c[k])), mu));
    }
    return bx;
}

// Leaf t of the input in fp64: a face's three corners (false when one is out of range), or the point in a (v holds the
// points; nv, f and fkind are unused).
template <typename L, typename T>
__device__ __forceinline__ bool mq_leaf_corners(const T* v, long long nv, const void* f, int fkind, long long t, double a[3],
                                                double b[3], double c[3]) {
    if constexpr (kPointLeaf<L>) {
        load_vertex<T>(v, t, a);
        return true;
    } else if constexpr (kBallLeaf<L>) {   // a: the centre, b[0]: the radius
        const double* ball = (const double*)v + 4 * t;
        a[0] = ball[0]; a[1] = ball[1]; a[2] = ball[2]; b[0] = ball[3];
        return ball[3] >= 0.0;
    } else {
        return mq_corners<T>(v, nv, f, fkind, t, a, b, c);
    }
}

// The leaf's fp32 box: a face's widened box, or the point's fp32 image as both corners.
template <typename L, typename T>
__device__ __forceinline__ MqBox mq_leaf_box(const double a[3], const double b[3], const double c[3]) {
    if constexpr (kPointLeaf<L>) {
        MqBox bx;
        for (int k = 0; k < 3; ++k) bx.lo[k] = bx.hi[k] = (float)a[k];
        return bx;
    } else if constexpr (kBallLeaf<L>) {
        MqBox bx;
        for (int k = 0; k < 3; ++k) {
            bx.lo[k] = __double2float_rd(__dsub_rd(a[k], b[0]));
            bx.hi[k] = __double2float_ru(__dadd_ru(a[k], b[0]));
        }
        return bx;
    } else {
        return mq_face_box<T>(a, b, c);
    }
}

// Coordinate k of the point a leaf's Morton code is taken at: a face's box centre, or the point itself (not
// 0.5 lo + 0.5 hi, which rounds a subnormal point and so could reorder the leaves).
template <typename L>
__device__ __forceinline__ float mq_code_point(const MqBox& bx, int k) {
    return kPointLeaf<L> ? bx.lo[k] : 0.5f * bx.lo[k] + 0.5f * bx.hi[k];
}

template <typename L, typename T>
__global__ void __launch_bounds__(kThreads) mq_bounds_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f,
                                                             int fkind, long long m, MqScratch* __restrict__ sc) {
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    unsigned long long bad = 0;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (long long)gridDim.x * blockDim.x) {
        if constexpr (kSurfelLeaf<L>) {   // v: the points, f: their SfSrc in device memory
            const SfSrc& src = *(const SfSrc*)f;
            MqBox bx;
            const bool finite = sf_box<T>(v, src, t, bx);
            if (!finite) bx.lo[0] = __int_as_float(0x7fffffff);
            src.boxes[t] = bx;
            if (!finite) { ++bad; continue; }
            for (int k = 0; k < 3; ++k) { lo[k] = min(lo[k], mq_ord(bx.lo[k])); hi[k] = max(hi[k], mq_ord(bx.hi[k])); }
            continue;
        }
        double a[3], b[3], c[3];
        if (!mq_leaf_corners<L, T>(v, nv, f, fkind, t, a, b, c)) { ++bad; continue; }
        const MqBox bx = mq_leaf_box<L, T>(a, b, c);
        for (int k = 0; k < 3; ++k) { lo[k] = min(lo[k], mq_ord(bx.lo[k])); hi[k] = max(hi[k], mq_ord(bx.hi[k])); }
    }
    for (int o = 16; o > 0; o >>= 1) {
        for (int k = 0; k < 3; ++k) {
            lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
        if constexpr (!kPointLeaf<L>) bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 3; ++k) { atomicMin(&sc->scene[k], lo[k]); atomicMax(&sc->scene[3 + k], hi[k]); }
        if (bad) atomicAdd(&sc->bad, bad);
    }
}

// Record t = (code of leaf t, t): its code point (mq_code_point) quantised to 21 bits per axis over the scene box.
template <typename L, typename T>
__global__ void __launch_bounds__(kThreads) mq_codes_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f,
                                                            int fkind, long long m, const MqScratch* __restrict__ sc,
                                                            MqRec* __restrict__ recs) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    unsigned long long code = ~0ull;
    double a[3], b[3], c[3];
    MqBox sb;
    bool surfel = false;
    if constexpr (kSurfelLeaf<L>) {   // v: the points, f: their SfSrc; the box mq_bounds_kernel stored
        sb = ((const SfSrc*)f)->boxes[t];
        surfel = !isnan(sb.lo[0]);
    }
    if (kSurfelLeaf<L> ? surfel : mq_leaf_corners<L, T>(v, nv, f, fkind, t, a, b, c)) {
        const MqBox bx = kSurfelLeaf<L> ? sb : mq_leaf_box<L, T>(a, b, c);
        code = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float slo = mq_unord(sc->scene[k]), shi = mq_unord(sc->scene[3 + k]);
            const float ext = shi - slo;
            const float centre = mq_code_point<L>(bx, k);
            const float s = ext > 0.f ? __fdividef(centre - slo, ext) * 2097152.f : 0.f;   // only orders the leaves
            code |= morton_split21((int)fminf(fmaxf(s, 0.f), 2097151.f)) << k;   // NaN -> 0
        }
    }
    *reinterpret_cast<ulonglong2*>(recs + t) = make_ulonglong2(code, (unsigned long long)t);   // {key[0], idx}
}

// A face is degenerate when D = (e1.e1)(e2.e2) - (e1.e2)^2 is not positive (DESIGN.md §3), in T from the corners.
template <typename T>
__device__ __forceinline__ bool mq_degenerate(const double a[3], const double b[3], const double c[3]) {
    using R = Real<T>;
    const T ax = (T)a[0], ay = (T)a[1], az = (T)a[2];
    const T e1x = R::sub((T)b[0], ax), e1y = R::sub((T)b[1], ay), e1z = R::sub((T)b[2], az);
    const T e2x = R::sub((T)c[0], ax), e2y = R::sub((T)c[1], ay), e2z = R::sub((T)c[2], az);
    const T d00 = R::add(R::add(R::mul(e1x, e1x), R::mul(e1y, e1y)), R::mul(e1z, e1z));
    const T d11 = R::add(R::add(R::mul(e2x, e2x), R::mul(e2y, e2y)), R::mul(e2z, e2z));
    const T d01 = R::add(R::add(R::mul(e1x, e2x), R::mul(e1y, e2y)), R::mul(e1z, e2z));
    const T D = R::sub(R::mul(d00, d11), R::mul(d01, d01));
    return !(D > (T)0);
}

// Leaf i (i < valid = m - bad): its face's corners as three Pt<T> (lane i: face id in the first, 1 for a degenerate
// face in the second) and its box.
template <typename T>
__global__ void __launch_bounds__(kThreads) mq_leaves_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f,
                                                             int fkind, long long m, const MqScratch* __restrict__ sc,
                                                             const MqRec* __restrict__ sorted, Pt<T>* __restrict__ leaves,
                                                             MqBox* __restrict__ boxes) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m - (long long)sc->bad) return;
    const long long t = (long long)sorted[i].idx;
    double a[3], b[3], c[3];
    mq_corners<T>(v, nv, f, fkind, t, a, b, c);
    boxes[i] = mq_face_box<T>(a, b, c);
    Pt<T> pa, pb, pc;
    pa.x = (T)a[0]; pa.y = (T)a[1]; pa.z = (T)a[2]; pa.i = (typename Real<T>::index_t)t;
    pb.x = (T)b[0]; pb.y = (T)b[1]; pb.z = (T)b[2]; pb.i = mq_degenerate<T>(a, b, c) ? 1 : 0;
    pc.x = (T)c[0]; pc.y = (T)c[1]; pc.z = (T)c[2]; pc.i = 0;
    leaves[3 * i] = pa; leaves[3 * i + 1] = pb; leaves[3 * i + 2] = pc;
}

// Surfel leaf i (i < m - bad): its fan in fp32 (layout at SfWord), its point id and its box.
template <typename T>
__global__ void __launch_bounds__(kThreads) sf_leaves_kernel(const T* __restrict__ p, const SfSrc src, long long m,
                                                             const MqScratch* __restrict__ sc, const MqRec* __restrict__ sorted,
                                                             SfWord* __restrict__ leaves, int* __restrict__ ids,
                                                             MqBox* __restrict__ boxes) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m - (long long)sc->bad) return;
    const long long t = (long long)sorted[i].idx;
    const long long words = sf_words(src.s);
    float* out = reinterpret_cast<float*>(leaves + i * words);
    MqBox bx;
    for (int k = 0; k < 3; ++k) { bx.lo[k] = __int_as_float(0x7f800000); bx.hi[k] = -bx.lo[k]; }
    sf_fan<T, float>(p, src, t, [&](int j, float x, float y, float z) {   // the fan once: the leaf and its box (sf_box's)
        const int at = j == src.s ? 0 : 3 * (j + 1);
        out[at] = x; out[at + 1] = y; out[at + 2] = z;
        bx.lo[0] = fminf(bx.lo[0], x); bx.lo[1] = fminf(bx.lo[1], y); bx.lo[2] = fminf(bx.lo[2], z);
        bx.hi[0] = fmaxf(bx.hi[0], x); bx.hi[1] = fmaxf(bx.hi[1], y); bx.hi[2] = fmaxf(bx.hi[2], z);
    });
    for (long long k = 3ll * (src.s + 1); k < 4 * words; ++k) out[k] = 0.f;
    ids[i] = (int)t;
    boxes[i] = bx;
}

// pointcloud_surfel_geometry: surfel i's s + 1 vertices at rows i (s + 1) .. (rim j at + j, the centre at + s), in T
// (the reference's mixed precision: basis and vertices in T, x0 and y0 in fp32), and its s faces (centre, rim j,
// rim (j + 1) mod s) at rows i s + j.  One thread per point.
template <typename T>
__global__ void __launch_bounds__(kThreads) sf_geometry_kernel(const T* __restrict__ p, const SfSrc src, long long m,
                                                               T* __restrict__ out_v, int* __restrict__ out_f) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int s = src.s;
    const long long base = i * (s + 1);
    sf_fan<T, T>(p, src, i, [&](int j, T x, T y, T z) {
        T* o = out_v + 3 * (base + j);
        o[0] = x; o[1] = y; o[2] = z;
    });
    for (int j = 0; j < s; ++j) {
        int* o = out_f + 3 * (i * s + j);
        o[0] = (int)(base + s); o[1] = (int)(base + j); o[2] = (int)(base + (j + 1) % s);
    }
}

// pointcloud_sphere_geometry: the reference's make_sphere_geometry for every point (DESIGN.md §3).  Point i has
// V = (stacks + 1)(slices + 1) vertices and F = 2 (stacks - 1) slices faces.  Threads [0, nv) write vertex rows,
// threads [nv, nv + nf) write faces, so a point's rows are written by consecutive threads (nv = m V < 2^31 - 1 and
// nf = m F < 2 nv: both fit 32 bits).  tab holds cos and sin of the stack angles a = 0 .. stacks, then cos and sin of
// the sector angles b = 0 .. slices, from the host's C library.  Vertex (a, b): xy = r_i cos_a, z = r_i sin_a,
// x = xy cos_b, y = xy sin_b, each product rounded on its own, and row k = (T)(p_ik + (x, y, z)_k) with the sum in fp64.
// Faces of stack a, sector j, k1 = a (slices + 1) + j, k2 = k1 + slices + 1: (k1, k2, k1 + 1) unless a = 0, then
// (k1 + 1, k2, k2 + 1) unless a = stacks - 1, offset by i V.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_geometry_kernel(const T* __restrict__ p, const T* __restrict__ r, const double* __restrict__ tab,
                                                               unsigned stacks, unsigned slices, unsigned nv, unsigned nf,
                                                               T* __restrict__ out_v, int* __restrict__ out_f) {
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    const unsigned cols = slices + 1, V = (stacks + 1) * cols;
    if (g < nv) {
        const unsigned k = (unsigned)g, i = k / V, q = k - i * V, a = q / cols, b = q - a * cols;
        const double ri = (double)r[i];
        const double xy = __dmul_rn(ri, __ldg(tab + a)), z = __dmul_rn(ri, __ldg(tab + stacks + 1 + a));
        const double* sector = tab + 2 * (stacks + 1);
        const double x = __dmul_rn(xy, __ldg(sector + b)), y = __dmul_rn(xy, __ldg(sector + cols + b));
        T* o = out_v + 3 * (size_t)k;
        o[0] = (T)__dadd_rn((double)p[3 * (size_t)i], x);
        o[1] = (T)__dadd_rn((double)p[3 * (size_t)i + 1], y);
        o[2] = (T)__dadd_rn((double)p[3 * (size_t)i + 2], z);
        return;
    }
    if (g >= (long long)nv + nf) return;
    const unsigned e = (unsigned)(g - nv), F = 2 * (stacks - 1) * slices, i = e / F;
    unsigned q = e - i * F, a, j;
    bool upper;   // the (k1, k2, k1 + 1) triangle, else the (k1 + 1, k2, k2 + 1) one
    if (q < slices) {
        a = 0; j = q; upper = false;
    } else {
        q -= slices;
        a = 1 + q / (2 * slices);
        const unsigned rem = q - (a - 1) * (2 * slices);
        if (a < stacks - 1) { j = rem >> 1; upper = (rem & 1) == 0; }
        else { j = rem; upper = true; }
    }
    const int k1 = (int)(i * V + a * cols + j), k2 = k1 + (int)cols;
    int* o = out_f + 3 * (size_t)e;
    o[0] = upper ? k1 : k1 + 1;
    o[1] = k2;
    o[2] = upper ? k1 + 1 : k2 + 1;
}

// ---- the per-(query, face) definition (DESIGN.md §3) ---------------------------------------------------------------
template <typename T>
struct MqHit { T d2, b0, b1, b2; };

template <typename T>
__device__ __forceinline__ T mq_dot(T ux, T uy, T uz, T wx, T wy, T wz) {
    using R = Real<T>;
    return R::add(R::add(R::mul(ux, wx), R::mul(uy, wy)), R::mul(uz, wz));
}
template <typename T>
__device__ __forceinline__ T mq_div(T a, T b);
template <> __device__ __forceinline__ float mq_div<float>(float a, float b) { return __fdiv_rn(a, b); }
template <> __device__ __forceinline__ double mq_div<double>(double a, double b) { return __ddiv_rn(a, b); }

// d^2 = ((px - cx)^2 + (py - cy)^2) + (pz - cz)^2
template <typename T>
__device__ __forceinline__ T mq_d2(const T p[3], T cx, T cy, T cz) {
    using R = Real<T>;
    const T dx = R::sub(p[0], cx), dy = R::sub(p[1], cy), dz = R::sub(p[2], cz);
    return R::add(R::add(R::mul(dx, dx), R::mul(dy, dy)), R::mul(dz, dz));
}

// Closest point of segment [x, y]: e = y - x, l = e.e; t = 0 when l is not positive, else (p - x).e / l clamped to
// [0, 1]; the point is x at t = 0, y at t = 1, else x + t e.  Returns d^2 and t.
template <typename T>
__device__ __forceinline__ T mq_segment(const T p[3], const T x[3], const T y[3], T& t) {
    using R = Real<T>;
    const T ex = R::sub(y[0], x[0]), ey = R::sub(y[1], x[1]), ez = R::sub(y[2], x[2]);
    const T l = mq_dot<T>(ex, ey, ez, ex, ey, ez);
    t = (T)0;
    if (l > (T)0) {
        t = mq_div<T>(mq_dot<T>(R::sub(p[0], x[0]), R::sub(p[1], x[1]), R::sub(p[2], x[2]), ex, ey, ez), l);
        t = t < (T)0 ? (T)0 : (t > (T)1 ? (T)1 : t);
    }
    if (t == (T)0) return mq_d2<T>(p, x[0], x[1], x[2]);
    if (t == (T)1) return mq_d2<T>(p, y[0], y[1], y[2]);
    return mq_d2<T>(p, R::add(x[0], R::mul(t, ex)), R::add(x[1], R::mul(t, ey)), R::add(x[2], R::mul(t, ez)));
}

// A degenerate face: the closest of its edges AB, BC, CA (the first on ties).
template <typename T>
__device__ __forceinline__ MqHit<T> mq_edges(const T p[3], const T a[3], const T b[3], const T c[3]) {
    using R = Real<T>;
    T t;
    MqHit<T> h;
    h.d2 = mq_segment<T>(p, a, b, t); h.b0 = R::sub((T)1, t); h.b1 = t; h.b2 = (T)0;
    T d2 = mq_segment<T>(p, b, c, t);
    if (d2 < h.d2) { h.d2 = d2; h.b0 = (T)0; h.b1 = R::sub((T)1, t); h.b2 = t; }
    d2 = mq_segment<T>(p, c, a, t);
    if (d2 < h.d2) { h.d2 = d2; h.b0 = t; h.b1 = (T)0; h.b2 = R::sub((T)1, t); }
    return h;
}

// n / d for an edge parameter: d >= n >= 0 here, and d = 0 only when n = 0 too.
template <typename T>
__device__ __forceinline__ T mq_ratio(T n, T d) { return d > (T)0 ? mq_div<T>(n, d) : (T)0; }

// Ericson's closest point on triangle abc, regions in his order: vertex A, vertex B, edge AB, vertex C, edge AC,
// edge BC, interior.  The interior is taken only when s = (va + vb) + vc > 0 and v = vb / s, w = vc / s satisfy
// v >= 0, w >= 0, v + w <= 1; otherwise, and for degenerate faces, the face is the union of its edges.
template <typename T>
__device__ __forceinline__ MqHit<T> closest_on_face(const T p[3], const T a[3], const T b[3], const T c[3], bool degenerate) {
    using R = Real<T>;
    if (degenerate) return mq_edges<T>(p, a, b, c);
    const T abx = R::sub(b[0], a[0]), aby = R::sub(b[1], a[1]), abz = R::sub(b[2], a[2]);
    const T acx = R::sub(c[0], a[0]), acy = R::sub(c[1], a[1]), acz = R::sub(c[2], a[2]);
    MqHit<T> h;
    const T apx = R::sub(p[0], a[0]), apy = R::sub(p[1], a[1]), apz = R::sub(p[2], a[2]);
    const T d1 = mq_dot<T>(abx, aby, abz, apx, apy, apz), d2 = mq_dot<T>(acx, acy, acz, apx, apy, apz);
    if (d1 <= (T)0 && d2 <= (T)0) {
        h.d2 = mq_d2<T>(p, a[0], a[1], a[2]); h.b0 = (T)1; h.b1 = (T)0; h.b2 = (T)0;
        return h;
    }
    const T bpx = R::sub(p[0], b[0]), bpy = R::sub(p[1], b[1]), bpz = R::sub(p[2], b[2]);
    const T d3 = mq_dot<T>(abx, aby, abz, bpx, bpy, bpz), d4 = mq_dot<T>(acx, acy, acz, bpx, bpy, bpz);
    if (d3 >= (T)0 && d4 <= d3) {
        h.d2 = mq_d2<T>(p, b[0], b[1], b[2]); h.b0 = (T)0; h.b1 = (T)1; h.b2 = (T)0;
        return h;
    }
    const T vc = R::sub(R::mul(d1, d4), R::mul(d3, d2));
    if (vc <= (T)0 && d1 >= (T)0 && d3 <= (T)0) {
        const T v = mq_ratio<T>(d1, R::sub(d1, d3));
        h.d2 = mq_d2<T>(p, R::add(a[0], R::mul(v, abx)), R::add(a[1], R::mul(v, aby)), R::add(a[2], R::mul(v, abz)));
        h.b0 = R::sub((T)1, v); h.b1 = v; h.b2 = (T)0;
        return h;
    }
    const T cpx = R::sub(p[0], c[0]), cpy = R::sub(p[1], c[1]), cpz = R::sub(p[2], c[2]);
    const T d5 = mq_dot<T>(abx, aby, abz, cpx, cpy, cpz), d6 = mq_dot<T>(acx, acy, acz, cpx, cpy, cpz);
    if (d6 >= (T)0 && d5 <= d6) {
        h.d2 = mq_d2<T>(p, c[0], c[1], c[2]); h.b0 = (T)0; h.b1 = (T)0; h.b2 = (T)1;
        return h;
    }
    const T vb = R::sub(R::mul(d5, d2), R::mul(d1, d6));
    if (vb <= (T)0 && d2 >= (T)0 && d6 <= (T)0) {
        const T w = mq_ratio<T>(d2, R::sub(d2, d6));
        h.d2 = mq_d2<T>(p, R::add(a[0], R::mul(w, acx)), R::add(a[1], R::mul(w, acy)), R::add(a[2], R::mul(w, acz)));
        h.b0 = R::sub((T)1, w); h.b1 = (T)0; h.b2 = w;
        return h;
    }
    const T va = R::sub(R::mul(d3, d6), R::mul(d5, d4));
    const T e43 = R::sub(d4, d3), e56 = R::sub(d5, d6);
    if (va <= (T)0 && e43 >= (T)0 && e56 >= (T)0) {
        const T w = mq_ratio<T>(e43, R::add(e43, e56));
        const T bcx = R::sub(c[0], b[0]), bcy = R::sub(c[1], b[1]), bcz = R::sub(c[2], b[2]);
        h.d2 = mq_d2<T>(p, R::add(b[0], R::mul(w, bcx)), R::add(b[1], R::mul(w, bcy)), R::add(b[2], R::mul(w, bcz)));
        h.b0 = (T)0; h.b1 = R::sub((T)1, w); h.b2 = w;
        return h;
    }
    const T s = R::add(R::add(va, vb), vc);
    if (s > (T)0) {
        const T v = mq_div<T>(vb, s), w = mq_div<T>(vc, s);
        if (v >= (T)0 && w >= (T)0 && R::add(v, w) <= (T)1) {
            h.d2 = mq_d2<T>(p, R::add(R::add(a[0], R::mul(abx, v)), R::mul(acx, w)),
                            R::add(R::add(a[1], R::mul(aby, v)), R::mul(acy, w)),
                            R::add(R::add(a[2], R::mul(abz, v)), R::mul(acz, w)));
            h.b0 = R::sub(R::sub((T)1, v), w); h.b1 = v; h.b2 = w;
            return h;
        }
    }
    return mq_edges<T>(p, a, b, c);
}

// ---- traversal ------------------------------------------------------------------------------------------------------
// Lower bound of |p - x|^2 over the fp32 box, rounded down throughout (p enters as [pl, ph] around its fp32 image).
__device__ __forceinline__ float mq_box_lb(const float pl[3], const float ph[3], const float lo[3], const float hi[3]) {
    float g[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = fmaxf(0.f, fmaxf(__fsub_rd(lo[k], ph[k]), __fsub_rd(pl[k], hi[k])));
    return __fadd_rd(__fadd_rd(__fmul_rd(g[0], g[0]), __fmul_rd(g[1], g[1])), __fmul_rd(g[2], g[2]));
}
// A box may be skipped only when no face in it can have a computed d^2 <= best (DESIGN.md §3): when
// rd(L (1 - 2^-21)) > ru(ru32(best) + 2^-140).
__device__ __forceinline__ bool mq_prune(float lb, float limit) { return __fmul_rd(lb, 1.f - 0x1p-21f) > limit; }
template <typename T>
__device__ __forceinline__ float mq_limit(T best) {
    return __fadd_ru(sizeof(T) == 4 ? (float)best : __double2float_ru((double)best), 0x1p-140f);
}

template <typename T>
__device__ __forceinline__ void mq_test_leaf(const Pt<T>* __restrict__ leaves, int leaf, const T p[3], T& best, long long& best_face,
                                             T bb[3], float& limit) {
    const Pt<T> A = leaves[3 * leaf], B = leaves[3 * leaf + 1], C = leaves[3 * leaf + 2];
    const T a[3] = {A.x, A.y, A.z}, b[3] = {B.x, B.y, B.z}, c[3] = {C.x, C.y, C.z};
    const MqHit<T> h = closest_on_face<T>(p, a, b, c, B.i != 0);
    const long long face = (long long)A.i;
    if (h.d2 < best || (h.d2 == best && face < best_face)) {
        best = h.d2; best_face = face; bb[0] = h.b0; bb[1] = h.b1; bb[2] = h.b2;
        limit = mq_limit<T>(best);
    }
}

// Query i in input order.  Nothing is written when the tree is empty (every face invalid: the caller raises).
// Per visit: one 64-byte node record; per face tested: three Pt<T> (48 B fp32, 96 B fp64).
template <typename T>
__global__ void __launch_bounds__(kThreads) mq_query_kernel(const T* __restrict__ q, long long nq, long long m,
                                                            const MqScratch* __restrict__ sc, const MqNode* __restrict__ nodes,
                                                            const Pt<T>* __restrict__ leaves, T* __restrict__ out_d,
                                                            void* __restrict__ out_fidx, int fidx_wide, T* __restrict__ out_bc) {
    const long long n = m - (long long)sc->bad;
    if (n < 1) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += (long long)gridDim.x * blockDim.x) {
        const T p[3] = {q[3 * i], q[3 * i + 1], q[3 * i + 2]};
        float pl[3], ph[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            pl[k] = sizeof(T) == 4 ? (float)p[k] : __double2float_rd((double)p[k]);
            ph[k] = sizeof(T) == 4 ? (float)p[k] : __double2float_ru((double)p[k]);
        }
        T best = Real<T>::inf(), bb[3] = {(T)0, (T)0, (T)0};
        long long best_face = -1;
        float limit = __int_as_float(0x7f800000);
        if (n == 1) {
            mq_test_leaf<T>(leaves, 0, p, best, best_face, bb, limit);
        } else {
            int stack[kMqStack];
            float stack_lb[kMqStack];
            int sp = 0, node = 0;
            while (true) {
                const float4* np_ = reinterpret_cast<const float4*>(nodes + node);
                const float4 q0 = __ldg(np_), q1 = __ldg(np_ + 1), q2 = __ldg(np_ + 2), q3 = __ldg(np_ + 3);
                const float lo0[3] = {q0.x, q0.y, q0.z}, hi0[3] = {q0.w, q1.x, q1.y};
                const float lo1[3] = {q1.z, q1.w, q2.x}, hi1[3] = {q2.y, q2.z, q2.w};
                const int c0 = __float_as_int(q3.x), c1 = __float_as_int(q3.y);
                const float l0 = mq_box_lb(pl, ph, lo0, hi0), l1 = mq_box_lb(pl, ph, lo1, hi1);
                bool k0 = !mq_prune(l0, limit), k1 = !mq_prune(l1, limit);
                if (k0 && c0 < 0) { mq_test_leaf<T>(leaves, ~c0, p, best, best_face, bb, limit); k0 = false; }
                if (k1 && c1 < 0) { mq_test_leaf<T>(leaves, ~c1, p, best, best_face, bb, limit); k1 = false; }
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
                    if (!mq_prune(stack_lb[sp], limit)) { node = stack[sp]; break; }
                }
                if (node < 0) break;
            }
        }
        // a non-finite query matches no face: it gets d = inf, fi = -1 (unspecified, DESIGN.md §7)
        out_d[i] = Real<T>::root(best);
        if (fidx_wide) ((long long*)out_fidx)[i] = best_face; else ((int*)out_fidx)[i] = (int)best_face;
        out_bc[3 * i] = bb[0]; out_bc[3 * i + 1] = bb[1]; out_bc[3 * i + 2] = bb[2];
    }
}

}  // namespace pcu
