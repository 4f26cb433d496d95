// mesh_geometry.cuh -- face areas, face and vertex normals of a triangle mesh (the reference's src/face_areas.cpp and
// src/mesh_normals.cpp), and the per-face and per-vertex pieces that Laplacian smoothing (laplacian.cuh) shares with
// them.  Results defined in DESIGN.md §3.
//
//   mg_face_kernel        one pass over the faces that writes whichever the caller asks for: the reference's face area
//                         (in v's precision), the unit normal (fp64, or rounded to v's type), the corner weights of
//                         the vertex normals, twice the area (face_area), half the cotangent of every corner, and the
//                         block partials of sum dblA and sum dblA * barycentre.  It counts the faces with a corner
//                         outside [0, #v).
//   mg_corner_kernel      one record per corner, key = vertex, idx = corner 3 t + k
//   radix sort (sort.cuh) stable, so every vertex's corners stay in ascending corner order
//   mg_incidence_kernel   first[v] = the first sorted position of v's corners (a CSR over the vertices), corner[j]
//   mg_vertex_normal_kernel  one thread per vertex: sum of w n_f over its corners in ascending (face, corner) order --
//                         the order of a sequential loop over f -- then normalised
// Reductions over the faces or vertices (reduce_grid) run on at most kMgBlocks CTAs: each CTA leaves its partial sums,
// and the last CTA to arrive adds them in CTA order, so two calls give the same bits and no floating-point atomic is
// used.
#pragma once
#include "common.cuh"
#include "meshsample.cuh"
#include "sort.cuh"

namespace pcu {

constexpr int kMgBlocks = 1024;                   // grid cap of the kernels that reduce
using MgRec = SortRec<unsigned long long, 1>;     // the records of sort.cuh's one-word sort

// What the host reads from a mesh-geometry call (zeroed per call).
struct MgRecord {
    unsigned long long bad;         // faces with a corner outside [0, #v)
    unsigned long long nonfinite;   // vertex coordinates that are not finite (smoothing only)
    long long nnz;                  // off-diagonal entries of the Laplacian (keep_offsets_kernel)
    unsigned ticket;                // arrivals of the current reduce_grid
    int zero_area;                  // a face pass with partials found a total dblA that is 0 or not finite
    double sums[4];                 // totals of the last face pass with partials: sum dblA, sum dblA * barycentre
};

// Sums v[0 .. K) over the block in a fixed order (a butterfly inside every warp, then the warps in order); the totals
// land in thread 0.  Block-wide.
template <int K>
__device__ __forceinline__ void block_sum(double v[K]) {
    __shared__ double warp_part[kThreads / 32][K];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] = __dadd_rn(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) warp_part[w][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double s = warp_part[0][k];
            for (int j = 1; j < kThreads / 32; ++j) s = __dadd_rn(s, warp_part[j][k]);
            v[k] = s;
        }
    __syncthreads();
}

// Grid-wide sums of v[0 .. K): every CTA stores its block_sum in partial[blockIdx.x]; the last CTA to arrive adds the
// gridDim.x partials (thread t takes CTAs t, t + kThreads, ... in order, then block_sum) and returns true, with the
// totals in its thread 0.  The other CTAs return false.  Deterministic for a given grid size.
template <int K>
__device__ __forceinline__ bool reduce_grid(double v[K], double* partial, unsigned* ticket) {
    __shared__ bool last;
    block_sum<K>(v);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) partial[(size_t)blockIdx.x * K + k] = v[k];
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return false;
    __threadfence();
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads)
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = __dadd_rn(v[k], __ldcg(partial + (size_t)b * K + k));
    block_sum<K>(v);
    if (threadIdx.x == 0) *ticket = 0u;
    return true;
}

// e1 = b - a, e2 = c - a, n = e1 x e2 in the order of face_area; returns |n| = sqrt((nx nx + ny ny) + nz nz).
__device__ __forceinline__ double face_cross(const double a[3], const double b[3], const double c[3], double n[3]) {
    const double e1x = __dsub_rn(b[0], a[0]), e1y = __dsub_rn(b[1], a[1]), e1z = __dsub_rn(b[2], a[2]);
    const double e2x = __dsub_rn(c[0], a[0]), e2y = __dsub_rn(c[1], a[1]), e2z = __dsub_rn(c[2], a[2]);
    n[0] = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
    n[1] = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
    n[2] = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(n[0], n[0]), __dmul_rn(n[1], n[1])), __dmul_rn(n[2], n[2])));
}

// (b - a) . (c - a) = ((x x + y y) + z z).
__device__ __forceinline__ double corner_dot(const double a[3], const double b[3], const double c[3]) {
    double s = 0.0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double p = __dmul_rn(__dsub_rn(b[d], a[d]), __dsub_rn(c[d], a[d]));
        s = d == 0 ? p : __dadd_rn(s, p);
    }
    return s;
}

// Max's (1999) corner weight |e1 x e2| / (|e1|^2 |e2|^2), e1 = b - a, e2 = c - a; 0 where |e1 x e2| = 0.
__device__ __forceinline__ double max_weight(const double a[3], const double b[3], const double c[3]) {
    const double A = face_area(a, b, c);
    return A == 0.0 ? 0.0 : __ddiv_rn(A, __dmul_rn(corner_dot(a, b, b), corner_dot(a, c, c)));
}

// The reference's face area (src/face_areas.cpp), operation for operation in T: edge lengths a = |v1 - v0|,
// b = |v2 - v1|, c = |v0 - v2| as sqrt((x x + y y) + z z), p = (a + b + c) 0.5, sqrt(((p max(p - a, 0)) max(p - b, 0))
// max(p - c, 0)), with max(x, 0) = x < 0 ? 0 : x as std::max returns it.
template <typename T>
__device__ __forceinline__ T reference_face_area(const T* p0, const T* p1, const T* p2) {
    using R = Real<T>;
    const T* q[4] = {p0, p1, p2, p0};
    T len[3];
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const T dx = R::sub(q[e + 1][0], q[e][0]), dy = R::sub(q[e + 1][1], q[e][1]), dz = R::sub(q[e + 1][2], q[e][2]);
        len[e] = R::root(R::add(R::add(R::mul(dx, dx), R::mul(dy, dy)), R::mul(dz, dz)));
    }
    const T p = R::mul(R::add(R::add(len[0], len[1]), len[2]), (T)0.5);
    T s = p;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const T d = R::sub(p, len[e]);
        s = R::mul(s, d < (T)0 ? (T)0 : d);
    }
    return R::root(s);
}

// The outputs of mg_face_kernel; a null pointer is not written.
template <typename T>
struct FaceOut {
    T* area;            // (m) the reference's face area, in T
    T* normal;          // (m, 3) unit normal, fp64 rounded once to T
    double* unit;       // (m, 3) unit normal in fp64
    double* weight;     // (m, 3) corner weights of the vertex normals: |e1 x e2| (weighting 1), the angle (weighting 2) or
                        // |e1 x e2| / (|e1|^2 |e2|^2), 0 where |e1 x e2| = 0 (weighting 3: Max's weights, curvature.cuh)
    int weighting;
    double* dbla;       // (m) face_area
    double* halfcot;    // (m, 3) cot / 2 of every corner's angle, 0 where dblA = 0
    double* partial;    // (gridDim.x, 4) block partials of sum dblA and sum dblA * barycentre -> MgRecord::sums
};

template <typename T>
__global__ void __launch_bounds__(kThreads) mg_face_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                           long long m, FaceOut<T> out, MgRecord* __restrict__ rec) {
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    unsigned nbad = 0u;
    for (long long t = (long long)blockIdx.x * kThreads + threadIdx.x; t < m; t += (long long)gridDim.x * kThreads) {
        long long c[3];
        bool bad = false;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            c[k] = load_index(f, 3 * t + k, fkind, nv, false);
            bad = bad || c[k] < 0;
        }
        if (bad) {   // the call fails; the outputs are still written
            ++nbad;
            c[0] = c[1] = c[2] = 0;
        }
        if (out.area) out.area[t] = bad ? (T)0 : reference_face_area<T>(v + 3 * c[0], v + 3 * c[1], v + 3 * c[2]);
        double p[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k) load_vertex<T>(v, c[k], p[k]);
        if (out.normal || out.unit) {
            double n[3];
            const double len = face_cross(p[0], p[1], p[2], n);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const double u = len == 0.0 ? 0.0 : __ddiv_rn(n[d], len);
                if (out.normal) out.normal[3 * t + d] = (T)u;
                if (out.unit) out.unit[3 * t + d] = u;
            }
        }
        if (out.weight)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double* a = p[k];
                const double* b = p[(k + 1) % 3];
                const double* e = p[(k + 2) % 3];
                out.weight[3 * t + k] = out.weighting == 1   ? face_area(p[0], p[1], p[2])
                                        : out.weighting == 2 ? atan2(face_area(a, b, e), corner_dot(a, b, e))
                                                             : max_weight(a, b, e);
            }
        if (out.dbla || out.halfcot || out.partial) {
            const double A = bad ? 0.0 : face_area(p[0], p[1], p[2]);
            if (out.dbla) out.dbla[t] = A;
            if (out.halfcot)
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    out.halfcot[3 * t + k] = A == 0.0 ? 0.0 : __dmul_rn(0.5, __ddiv_rn(corner_dot(p[k], p[(k + 1) % 3], p[(k + 2) % 3]), A));
            if (out.partial) {
                acc[0] = __dadd_rn(acc[0], A);
#pragma unroll
                for (int d = 0; d < 3; ++d)
                    acc[1 + d] = __dadd_rn(acc[1 + d], __dmul_rn(A, __ddiv_rn(__dadd_rn(__dadd_rn(p[0][d], p[1][d]), p[2][d]), 3.0)));
            }
        }
    }
    nbad = __reduce_add_sync(0xffffffffu, nbad);
    if ((threadIdx.x & 31) == 0 && nbad) atomicAdd(&rec->bad, (unsigned long long)nbad);
    if (out.partial && reduce_grid<4>(acc, out.partial, &rec->ticket) && threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) rec->sums[k] = acc[k];
        if (!(acc[0] > 0.0 && acc[0] <= 1.7976931348623157e308)) rec->zero_area = 1;
    }
}

// One record per corner: key = its vertex, idx = 3 t + k.  A corner outside [0, nv) gets key 0 (the call fails).
__global__ void __launch_bounds__(kThreads) mg_corner_kernel(const void* __restrict__ f, int fkind, long long corners, long long nv,
                                                             MgRec* __restrict__ recs) {
    const long long c = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (c >= corners) return;
    const long long x = load_index(f, c, fkind, nv, false);
    MgRec r;
    r.key[0] = x < 0 ? 0ull : (unsigned long long)x;
    r.idx = (unsigned long long)c;
    store_rec(recs + c, r);
}

// Over the n sorted records of a one-word key < nkeys, one thread per position i in [0, n]: first[k] = i for every
// key k in (key[i - 1], key[i]] (key[-1] = -1, key[n] = nkeys), so row k holds positions [first[k], first[k + 1]);
// item[i] = idx[i] >> item_shift when item is not null.
__global__ void __launch_bounds__(kThreads) mg_rows_kernel(const MgRec* __restrict__ sorted, long long n, long long nkeys, int* __restrict__ first,
                                                           int* __restrict__ item, int item_shift) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i > n) return;
    const long long prev = i == 0 ? -1 : (long long)sorted[i - 1].key[0];
    const long long cur = i < n ? (long long)sorted[i].key[0] : nkeys;
    for (long long k = prev + 1; k <= cur; ++k) first[k] = (int)i;
    if (item && i < n) item[i] = (int)(sorted[i].idx >> item_shift);
}

// One thread per vertex: s = sum over its corners c (ascending) of w_c n_f(c) (w = 1 when weight is null), then
// s / |s|, or 0 when |s| = 0; rounded once to T.
template <typename T>
__global__ void __launch_bounds__(kThreads) mg_vertex_normal_kernel(const int* __restrict__ first, const int* __restrict__ corner, long long nv,
                                                                    const double* __restrict__ unit, const double* __restrict__ weight,
                                                                    T* __restrict__ out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= nv) return;
    double s[3] = {0.0, 0.0, 0.0};
    for (int j = first[i], e = first[i + 1]; j < e; ++j) {
        const int c = __ldg(corner + j);
        const long long t = c / 3;
        const double w = weight ? __ldg(weight + c) : 1.0;
#pragma unroll
        for (int d = 0; d < 3; ++d) s[d] = __dadd_rn(s[d], weight ? __dmul_rn(w, __ldg(unit + 3 * t + d)) : __ldg(unit + 3 * t + d));
    }
    const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])), __dmul_rn(s[2], s[2])));
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * i + d] = (T)(len == 0.0 ? 0.0 : __ddiv_rn(s[d], len));
}

}  // namespace pcu
