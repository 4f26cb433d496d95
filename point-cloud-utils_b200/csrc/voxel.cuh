// voxel.cuh -- voxel-grid down-sampling of a point cloud (SURVEY.md 8f, row N2).
//
// Replaces downsample_point_cloud_to_voxels (src/sample_point_cloud.cpp:163-244; binding :336-367; Python wrapper
// point_cloud_utils/__init__.py:123-200): every point goes to the voxel
//     index = int(floor((p - min_bound) / voxel_size))       per axis, in the cloud's precision (:205-206)
// and every voxel holding at least min_points_per_voxel points contributes the mean of its points (and of one
// attribute array) to the output.
//
// What is exact: the voxel of every point (same rounded subtraction, division and floor), hence the set of occupied
// voxels, the point count of each and the number of output rows.  That includes points whose quotient does not fit an
// int -- far outside explicit bounds, +-inf, NaN: the reference's int(...) on x86-64 gives INT_MIN for all of them, so
// on such an axis they share the INT_MIN layer of the grid here too.  What differs, and is stated: the reference walks
// a std::unordered_map, so its output ORDER is whatever libstdc++'s hash table iteration yields -- here voxels come out
// in the order of their first point in the input; and the reference sums in the cloud's precision point after point
// where this kernel accumulates in fp64 (atomics), so the means are within one float32 ulp of the exact mean of the
// voxel's points for float32 outputs, and within the fp64 summation bound for float64 ones
// (tests/test_voxel_grid_edges.py), rather than equal to the reference's rounded float sums.
//
// No sort: a hash table of point indices (open addressing, 32-bit CAS; a slot's key is the voxel of the point it
// holds, recomputed when probing) groups the points; per voxel an atomicMin keeps its first point, which is where the
// output row is emitted by an ordered compaction.
#pragma once
#include "common.cuh"
#include "compact.cuh"

namespace pcu {

template <typename T>
struct VoxelGrid {
    T min_bound[3];
    T size[3];
};

template <typename T>
__device__ __forceinline__ void voxel_of(const VoxelGrid<T>& g, const T* __restrict__ p, int (&v)[3]) {
    using R = Real<T>;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const T c = sizeof(T) == 4 ? (T)__fdiv_rn((float)R::sub(p[a], g.min_bound[a]), (float)g.size[a])
                                   : (T)__ddiv_rn((double)R::sub(p[a], g.min_bound[a]), (double)g.size[a]);
        // floor of a T value is exact in double.  int(...) as the reference's x86-64 build converts: a value outside
        // the int range, +-inf and NaN all give INT_MIN (a plain cast here would saturate, and turn NaN into 0)
        const double f = floor((double)c);
        v[a] = (f >= -2147483648.0 && f < 2147483648.0) ? (int)f : INT_MIN;
    }
}

__device__ __forceinline__ unsigned voxel_hash(const int (&v)[3]) {
    unsigned h = (unsigned)v[0] * 73856093u ^ (unsigned)v[1] * 19349663u ^ (unsigned)v[2] * 83492791u;
    h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
    return h;
}

constexpr int kVoxelEmpty = -1;

// Per-voxel accumulators, one record per hash slot.
struct VoxelAcc {
    double sum[3];
    int count;
    int first;      // smallest point index of the voxel
};

// pass 1: find / claim the slot of every point's voxel, accumulate.  table: `slots` ints, all kVoxelEmpty on entry;
// acc: `slots` records, zeroed except first = INT_MAX; attr (n, c) or null with attr_sum (slots, c) zeroed.
template <typename T, typename A>
__global__ void __launch_bounds__(kThreads) voxel_insert_kernel(const T* __restrict__ pts, long long n, VoxelGrid<T> g,
                                                                int* __restrict__ table, unsigned slots, VoxelAcc* __restrict__ acc,
                                                                int* __restrict__ slot_of, const A* __restrict__ attr, int c,
                                                                double* __restrict__ attr_sum) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int v[3];
    voxel_of<T>(g, pts + 3 * i, v);
    unsigned h = voxel_hash(v) % slots;
    for (;;) {
        int r = table[h];
        if (r == kVoxelEmpty) r = atomicCAS(table + h, kVoxelEmpty, (int)i);
        if (r == kVoxelEmpty) break;                 // claimed: point i represents this voxel's slot
        int w[3];
        voxel_of<T>(g, pts + 3ll * r, w);
        if (w[0] == v[0] && w[1] == v[1] && w[2] == v[2]) break;
        h = h + 1 == slots ? 0u : h + 1;
    }
    slot_of[i] = (int)h;
    VoxelAcc* a = acc + h;
    atomicAdd(&a->sum[0], (double)pts[3 * i]);
    atomicAdd(&a->sum[1], (double)pts[3 * i + 1]);
    atomicAdd(&a->sum[2], (double)pts[3 * i + 2]);
    atomicAdd(&a->count, 1);
    atomicMin(&a->first, (int)i);
    for (int k = 0; k < c; ++k) atomicAdd(attr_sum + (size_t)h * c + k, (double)attr[(size_t)i * c + k]);
}

__global__ void __launch_bounds__(kThreads) voxel_init_kernel(int* __restrict__ table, VoxelAcc* __restrict__ acc, unsigned slots) {
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots) return;
    table[s] = kVoxelEmpty;
    VoxelAcc a; a.sum[0] = a.sum[1] = a.sum[2] = 0.0; a.count = 0; a.first = 0x7fffffff;
    acc[s] = a;
}

// pass 2: a point emits an output row iff it is the first point of its voxel and the voxel is full enough
__global__ void __launch_bounds__(kThreads) voxel_flag_kernel(const int* __restrict__ slot_of, const VoxelAcc* __restrict__ acc,
                                                              long long n, int min_points, unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const VoxelAcc& a = acc[slot_of[i]];
    keep[i] = (a.first == (int)i && a.count >= min_points) ? 1 : 0;
}

// pass 3 (after keep_count / keep_offsets of compact.cuh): ordered scatter of the means
template <typename T, typename A>
__global__ void __launch_bounds__(kThreads) voxel_emit_kernel(const unsigned char* __restrict__ keep, long long n,
                                                              const unsigned* __restrict__ block_offset, const int* __restrict__ slot_of,
                                                              const VoxelAcc* __restrict__ acc, const double* __restrict__ attr_sum, int c,
                                                              T* __restrict__ out_pts, A* __restrict__ out_attr, int* __restrict__ out_count) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? keep[i] : 0u;
    const unsigned pos = keep_rank(mine, block_offset);
    if (mine) {
        const int h = slot_of[i];
        const VoxelAcc a = acc[h];
        const double cnt = (double)a.count;
        out_pts[3ll * pos] = (T)(a.sum[0] / cnt);
        out_pts[3ll * pos + 1] = (T)(a.sum[1] / cnt);
        out_pts[3ll * pos + 2] = (T)(a.sum[2] / cnt);
        for (int k = 0; k < c; ++k) out_attr[(size_t)pos * c + k] = (A)(attr_sum[(size_t)h * c + k] / cnt);
        if (out_count != nullptr) out_count[pos] = a.count;
    }
}

}  // namespace pcu
