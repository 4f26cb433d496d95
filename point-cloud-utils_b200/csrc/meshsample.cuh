// meshsample.cuh -- sampling points on triangle meshes (sample_mesh_random / sample_mesh_poisson_disk of the reference,
// src/sample_mesh.cpp) and barycentric interpolation (interpolate_barycentric_coords, point_cloud_utils/__init__.py).
//
// The reference draws with std::rand and libigl; the samples here are defined exactly instead (DESIGN.md §3, mesh
// samples), as pure functions of (v, f, seed):
//   face weight  A_f = |(b - a) x (c - a)| in fp64 (every operation rounded on its own, order in face_area), 0 when not
//                finite or when a corner is outside [0, #v);  S = 2^(62 - ceil(log2 m)) / max A (0 when max A = 0 or S
//                overflows);  w_f = floor(A_f * S) as uint64, so sum w_f < 2^63;  C = inclusive prefix sum of w (exact);
//                W = C[m - 1].
//   sample s     h(j) = mix64(mix64(3 s + j) ^ seed);  face = first f with C_f > mulhi64(h(0), W);
//                u1, u2 = (h(1) >> 11) 2^-53, (h(2) >> 11) 2^-53;  a = sqrt(u1);  bc = (1 - a, a (1 - u2), a u2) in fp64,
//                each rounded once to T.
// Row s of the output is sample s: no sort and no atomics decide anything.
#pragma once
#include "common.cuh"

namespace pcu {

constexpr int kMeshScanThreads = 256;
constexpr int kMeshScanTile = 4096;     // faces per CTA of the CDF scan (16 per thread)

// {W, S, faces with a corner out of range}: what the host reads to size and validate a call (pcu_b200_mesh_area).
struct MeshArea {
    unsigned long long total;
    double scale;
    unsigned long long bad;
};
struct MeshScratch {
    unsigned long long max_bits;   // bits of max A_f (non-negative doubles order like their bits)
    unsigned long long bad;
};

// Twice the triangle's area: e1 = b - a, e2 = c - a, n = (e1y e2z - e1z e2y, e1z e2x - e1x e2z, e1x e2y - e1y e2x),
// A = sqrt((nx nx + ny ny) + nz nz), everything fp64 and rounded per operation (no FMA).
__device__ __forceinline__ double face_area(const double a[3], const double b[3], const double c[3]) {
    const double e1x = __dsub_rn(b[0], a[0]), e1y = __dsub_rn(b[1], a[1]), e1z = __dsub_rn(b[2], a[2]);
    const double e2x = __dsub_rn(c[0], a[0]), e2y = __dsub_rn(c[1], a[1]), e2z = __dsub_rn(c[2], a[2]);
    const double nx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
    const double ny = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
    const double nz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
    const double A = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
    return A >= 0.0 && A <= 1.7976931348623157e308 ? A : 0.0;
}

template <typename T>
__device__ __forceinline__ void load_vertex(const T* v, long long i, double p[3]) {
    p[0] = (double)v[3 * i]; p[1] = (double)v[3 * i + 1]; p[2] = (double)v[3 * i + 2];
}

__device__ __forceinline__ double mesh_weight_scale(unsigned long long max_bits, long long m) {
    const int k = m > 1 ? 64 - __clzll((unsigned long long)(m - 1)) : 0;   // ceil(log2 m)
    const double amax = __longlong_as_double((long long)max_bits);
    const double s = __ddiv_rn(ldexp(1.0, 62 - k), amax);
    return amax > 0.0 && s <= 1.7976931348623157e308 ? s : 0.0;
}
__device__ __forceinline__ unsigned long long mesh_weight(unsigned long long area_bits, double s) {
    return (unsigned long long)floor(__dmul_rn(__longlong_as_double((long long)area_bits), s));   // < 2^(62-k) (1 + 2^-52)
}

// Per face: A_f (its bits, into `area`), the maximum and the count of faces with a corner out of range.
template <typename T>
__global__ void __launch_bounds__(kThreads) mesh_area_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f,
                                                             int fkind, long long m, unsigned long long* __restrict__ area,
                                                             MeshScratch* __restrict__ sc) {
    __shared__ unsigned long long warp_max[kThreads / 32];
    unsigned long long mx = 0;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (long long)gridDim.x * blockDim.x) {
        const long long i0 = load_index(f, 3 * t, fkind, nv, false), i1 = load_index(f, 3 * t + 1, fkind, nv, false),
                        i2 = load_index(f, 3 * t + 2, fkind, nv, false);
        double A = 0.0;
        if (i0 < 0 || i1 < 0 || i2 < 0) {
            atomicAdd(&sc->bad, 1ull);
        } else {
            double a[3], b[3], c[3];
            load_vertex<T>(v, i0, a); load_vertex<T>(v, i1, b); load_vertex<T>(v, i2, c);
            A = face_area(a, b, c);
        }
        const unsigned long long bits = (unsigned long long)__double_as_longlong(A);
        area[t] = bits;
        mx = bits > mx ? bits : mx;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, mx, o);
        mx = u > mx ? u : mx;
    }
    if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; ++w) mx = warp_max[w] > mx ? warp_max[w] : mx;
        if (mx != 0) atomicMax(&sc->max_bits, mx);
    }
}

__device__ __forceinline__ unsigned long long mesh_hash(unsigned long long seed, unsigned long long s, unsigned j) {
    return mix64(mix64(3ull * s + j) ^ seed);
}

// Samples s = 0 .. n-1 (or, with `rows`, s = rows[i] for i < *nrows: the kept rows of the Poisson-disk selection),
// written to row i of the outputs.  out_fidx (4- or 8-byte integers) and out_bc may be null; out_pos (may be null)
// receives fl_T((bc0 a + bc1 b) + bc2 c), fp64 from the unrounded coordinates, per axis.  W = 0 writes nothing.
template <typename T>
__global__ void __launch_bounds__(kThreads) mesh_sample_kernel(const unsigned long long* __restrict__ cdf, long long m,
                                                               const MeshArea* __restrict__ area, unsigned long long seed, long long n,
                                                               const int* __restrict__ rows, const long long* __restrict__ nrows,
                                                               const T* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                               void* __restrict__ out_fidx, int fidx_wide, T* __restrict__ out_bc,
                                                               T* __restrict__ out_pos) {
    const unsigned long long W = area->total;
    if (W == 0) return;
    const long long count = rows ? *nrows : n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long s = rows ? (unsigned long long)rows[i] : (unsigned long long)i;
        const unsigned long long u = __umul64hi(mesh_hash(seed, s, 0), W);   // < W = C[m - 1]
        long long lo = 0, hi = m - 1;
        while (lo < hi) {
            const long long mid = lo + ((hi - lo) >> 1);
            if (__ldg(cdf + mid) > u) hi = mid; else lo = mid + 1;
        }
        const double u1 = (double)(mesh_hash(seed, s, 1) >> 11) * 0x1p-53, u2 = (double)(mesh_hash(seed, s, 2) >> 11) * 0x1p-53;
        const double a = __dsqrt_rn(u1);
        const double b0 = __dsub_rn(1.0, a), b1 = __dmul_rn(a, __dsub_rn(1.0, u2)), b2 = __dmul_rn(a, u2);
        if (out_fidx) {
            if (fidx_wide) ((long long*)out_fidx)[i] = lo; else ((int*)out_fidx)[i] = (int)lo;
        }
        if (out_bc) { out_bc[3 * i] = (T)b0; out_bc[3 * i + 1] = (T)b1; out_bc[3 * i + 2] = (T)b2; }
        if (out_pos) {   // the corners are in range: a face with one outside weighs 0 and is never drawn
            double pa[3], pb[3], pc[3];
            load_vertex<T>(v, load_index(f, 3 * lo, fkind, nv, false), pa);
            load_vertex<T>(v, load_index(f, 3 * lo + 1, fkind, nv, false), pb);
            load_vertex<T>(v, load_index(f, 3 * lo + 2, fkind, nv, false), pc);
#pragma unroll
            for (int d = 0; d < 3; ++d)
                out_pos[3 * i + d] = (T)__dadd_rn(__dadd_rn(__dmul_rn(b0, pa[d]), __dmul_rn(b1, pb[d])), __dmul_rn(b2, pc[d]));
        }
    }
}

// out[i, d] = ((x0 b0 + x1 b1) + x2 b2), x_k = attr[f[fi[i], k], d], products and sums in the promoted type P with no
// FMA: numpy's (attribute[f[fi]] * bc[:, :, None]).sum(1) bit for bit.  Indices wrap like numpy's; a row with an index
// out of range is never loaded: it gets NaN and is counted in *bad.
template <typename A, typename B, typename P>
__global__ void __launch_bounds__(kThreads) interpolate_bary_kernel(const void* __restrict__ f, long long m, int fkind,
                                                                    const void* __restrict__ fi, long long n, int fikind,
                                                                    const B* __restrict__ bc, const A* __restrict__ attr, long long nv,
                                                                    long long dim, P* __restrict__ out, unsigned long long* __restrict__ bad) {
    using R = Real<P>;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n * dim; e += (long long)gridDim.x * blockDim.x) {
        const long long i = e / dim, d = e - i * dim;
        const long long face = load_index(fi, i, fikind, m, true);
        long long c[3] = {-1, -1, -1};
        if (face >= 0)
            for (int k = 0; k < 3; ++k) c[k] = load_index(f, 3 * face + k, fkind, nv, true);
        if (c[0] < 0 || c[1] < 0 || c[2] < 0) {
            out[e] = (P)__longlong_as_double(0x7ff8000000000000LL);
            if (d == 0) atomicAdd(bad, 1ull);
            continue;
        }
        const P x0 = (P)attr[c[0] * dim + d], x1 = (P)attr[c[1] * dim + d], x2 = (P)attr[c[2] * dim + d];
        const P b0 = (P)bc[3 * i], b1 = (P)bc[3 * i + 1], b2 = (P)bc[3 * i + 2];
        out[e] = R::add(R::add(R::mul(x0, b0), R::mul(x1, b1)), R::mul(x2, b2));
    }
}

}  // namespace pcu
