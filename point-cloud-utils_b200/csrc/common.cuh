// common.cuh -- shared device-side vocabulary of the H100 nearest-neighbour path.
//
// Exact-arithmetic contract (the reason indices can be bit-identical to the reference):
// nanoflann's L2_Simple metric (external/nanoflann/nanoflann.hpp:496-507 in the reference) is
//     d2 = ((qx-px)^2 + (qy-py)^2) + (qz-pz)^2
// with every subtraction, product and sum rounded separately in the input precision.  nvcc would
// contract a*b+c into FFMA/DFMA, so every operation that feeds a comparison goes through the
// round-to-nearest intrinsics below, which the compiler never fuses.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

namespace pcu {

constexpr int kMaxGridDim = 2048;   // cells per axis, upper bound
constexpr int kThreads = 256;       // default CTA size of the streaming kernels
constexpr int kMaxLevels = 12;      // 2^11 = kMaxGridDim, plus one

// Index arrays come in four integer types, chosen at run time (pcu_b200_index_kind).
enum MeshIndexKind { kIdxI32 = 0, kIdxI64 = 1, kIdxU32 = 2, kIdxU64 = 3 };

// Entry i of an index array of kind `kind`, checked against [0, n): negative entries of a signed array wrap by n when
// `wrap` is set (numpy's indexing), and -1 stands for anything out of range.
__device__ __forceinline__ long long load_index(const void* a, long long i, int kind, long long n, bool wrap) {
    long long x;
    switch (kind) {
        case kIdxI32: x = ((const int*)a)[i]; break;
        case kIdxI64: x = ((const long long*)a)[i]; break;
        case kIdxU32: x = (long long)((const unsigned*)a)[i]; break;
        default: {
            const unsigned long long u = ((const unsigned long long*)a)[i];
            x = u >= (unsigned long long)n ? -1 - n : (long long)u;   // never wraps
        }
    }
    if (x < 0 && wrap) x += n;
    return x >= 0 && x < n ? x : -1;
}

// Programmatic dependent launch: every kernel of a call's chain is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so its CTAs may be scheduled while the previous
// kernel drains; this wait (first statement of every kernel) blocks until that kernel has completed
// and its writes are visible.  A no-op for ordinary launches.
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename T> struct Real;

template <> struct Real<float> {
    using bits_t = uint32_t;
    using index_t = int32_t;        // payload that rides in the 4th lane of a sorted point
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float root(float a) { return __fsqrt_rn(a); }
    static __device__ __forceinline__ float inf() { return __int_as_float(0x7f800000); }
    static __device__ __forceinline__ float largest() { return __int_as_float(0x7f7fffff); }   // FLT_MAX
    static __device__ __forceinline__ float vmax(float a, float b) { return fmaxf(a, b); }
    static __device__ __forceinline__ float vmin(float a, float b) { return fminf(a, b); }
    static __device__ __forceinline__ bits_t bits(float a) { return __float_as_uint(a); }
    static __device__ __forceinline__ float from_bits(bits_t b) { return __uint_as_float(b); }
    static constexpr bits_t kSign = 0x80000000u;
    static constexpr int kBits = 32;
};

template <> struct Real<double> {
    using bits_t = unsigned long long;
    using index_t = long long;
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double root(double a) { return __dsqrt_rn(a); }
    static __device__ __forceinline__ double inf() { return __longlong_as_double(0x7ff0000000000000LL); }
    static __device__ __forceinline__ double largest() { return __longlong_as_double(0x7fefffffffffffffLL); }   // DBL_MAX
    static __device__ __forceinline__ double vmax(double a, double b) { return fmax(a, b); }
    static __device__ __forceinline__ double vmin(double a, double b) { return fmin(a, b); }
    static __device__ __forceinline__ bits_t bits(double a) { return (bits_t)__double_as_longlong(a); }
    static __device__ __forceinline__ double from_bits(bits_t b) { return __longlong_as_double((long long)b); }
    static constexpr bits_t kSign = 0x8000000000000000ULL;
    static constexpr int kBits = 64;
};

// Order-preserving map between a float and an unsigned integer (total order, -inf .. +inf).
template <typename T>
__device__ __forceinline__ typename Real<T>::bits_t ordered(T v) {
    using R = Real<T>;
    typename R::bits_t u = R::bits(v);
    return (u & R::kSign) ? ~u : (u | R::kSign);
}
template <typename T>
__device__ __forceinline__ T unordered(typename Real<T>::bits_t u) {
    using R = Real<T>;
    return R::from_bits((u & R::kSign) ? (u & ~R::kSign) : ~u);
}

// A binned point: coordinates plus the row it had in the caller's array.  16 B (fp32) / 32 B (fp64)
// so one point is one (or two) 128-bit loads.
template <typename T> struct Pt;
template <> struct __align__(16) Pt<float> { float x, y, z; int32_t i; };
template <> struct __align__(32) Pt<double> { double x, y, z; long long i; };

template <typename T>
__device__ __forceinline__ Pt<T> load_pt(const Pt<T>* p);
template <>
__device__ __forceinline__ Pt<float> load_pt<float>(const Pt<float>* p) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    Pt<float> r; r.x = v.x; r.y = v.y; r.z = v.z; r.i = __float_as_int(v.w);
    return r;
}
template <>
__device__ __forceinline__ Pt<double> load_pt<double>(const Pt<double>* p) {
    const double2 a = __ldg(reinterpret_cast<const double2*>(p));
    const double2 b = __ldg(reinterpret_cast<const double2*>(p) + 1);
    Pt<double> r; r.x = a.x; r.y = a.y; r.z = b.x; r.i = __double_as_longlong(b.y);
    return r;
}
template <typename T>
__device__ __forceinline__ void store_pt(Pt<T>* dst, T x, T y, T z, long long i);
template <>
__device__ __forceinline__ void store_pt<float>(Pt<float>* dst, float x, float y, float z, long long i) {
    *reinterpret_cast<float4*>(dst) = make_float4(x, y, z, __int_as_float((int)i));
}
template <>
__device__ __forceinline__ void store_pt<double>(Pt<double>* dst, double x, double y, double z, long long i) {
    reinterpret_cast<double2*>(dst)[0] = make_double2(x, y);
    reinterpret_cast<double2*>(dst)[1] = make_double2(z, __longlong_as_double(i));
}

// The reference metric, operation for operation (query minus data).
template <typename T>
__device__ __forceinline__ T dist2(T qx, T qy, T qz, T px, T py, T pz) {
    using R = Real<T>;
    const T dx = R::sub(qx, px), dy = R::sub(qy, py), dz = R::sub(qz, pz);
    return R::add(R::add(R::mul(dx, dx), R::mul(dy, dy)), R::mul(dz, dz));
}
template <typename T>
__device__ __forceinline__ T sq_gap(T q, T wall) {  // lower bound for one axis, same rounding as the metric
    using R = Real<T>;
    const T d = R::sub(q, wall);
    return R::mul(d, d);
}

// 32-bit integer finaliser (a bijection): the counter-based hash behind the random choices of the ball normals'
// neighbour subsets and of the Poisson-disk sample's priorities.
__device__ __forceinline__ unsigned mix32(unsigned h) {
    h ^= h >> 16; h *= 0x7feb352du; h ^= h >> 15; h *= 0x846ca68bu; h ^= h >> 16;
    return h;
}

// splitmix64 (its +0x9E3779B97F4A7C15 step, then its finaliser; a bijection, mix64(0) = 0xE220A8397B1DCDAF): the
// counter-based hash behind the mesh samples' faces and barycentric coordinates.
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// Block-wide exclusive scan, kBlock threads: returns the exclusive prefix of v and sets *total to the block sum in
// every thread.  Ends with a barrier, so it may be called again right away (in a loop, on the same warp_sum).  V is
// the value type: 32-bit counts almost everywhere, 64-bit for the mesh samplers' face weights.
template <int kBlock, class V = unsigned>
__device__ __forceinline__ V block_exclusive_scan(V v, V* total) {
    static_assert(kBlock % 32 == 0 && kBlock <= 1024, "whole warps, at most 32 of them");
    constexpr int kWarps = kBlock / 32;
    __shared__ V warp_sum[kWarps];
    const int l = threadIdx.x & 31, w = threadIdx.x >> 5;
    V inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const V u = __shfl_up_sync(0xffffffffu, inc, o);
        if (l >= o) inc += u;
    }
    if (l == 31) warp_sum[w] = inc;
    __syncthreads();
    if (w == 0) {
        V s = l < kWarps ? warp_sum[l] : (V)0;
#pragma unroll
        for (int o = 1; o < kWarps; o <<= 1) {
            const V u = __shfl_up_sync(0xffffffffu, s, o);
            if (l >= o) s += u;
        }
        if (l < kWarps) warp_sum[l] = s;   // inclusive over warps
    }
    __syncthreads();
    const V before = w ? warp_sum[w - 1] : (V)0;
    *total = warp_sum[kWarps - 1];
    __syncthreads();
    return before + inc - v;
}

// Exclusive scan of `count` values, kBlock of them per round, with the running total carried between rounds:
// thread t handles i = t, t + kBlock, ...; load(i) gives value i and store(i, prefix, value) receives its exclusive
// prefix.  Returns the sum of all values to every thread.  Block-wide; ends with a barrier, so the stores are visible
// to the whole block on return.  The rounds are counted in the index type `I` of `count`: nvcc unrolls the loop over a
// signed count (the slab build's per-tile scan needs that) and keeps the one over an unsigned count rolled (fewer
// registers where the scan is the whole kernel).  V is the value type, as for block_exclusive_scan.
template <int kBlock, class V = unsigned, class I, class Load, class Store>
__device__ __forceinline__ V block_scan_rounds(I count, Load load, Store store) {
    V carry = 0;
    for (I b = 0; b < count; b += kBlock) {
        const I i = b + (I)threadIdx.x;
        const V v = i < count ? (V)load(i) : (V)0;
        V total;
        const V ex = carry + block_exclusive_scan<kBlock, V>(v, &total);
        if (i < count) store(i, ex, v);
        carry += total;
    }
    __syncthreads();
    return carry;
}

// Uniform grid over one cloud's bounding box.  Lives in device memory; written by grid_setup.
//   cell(p) = clamp(int(fl(fl(p - origin) * inv_h)), 0, dim-1)   -- monotone in p, so the walls
//   below are exact statements about where points of a given cell can lie:
//     wall_hi[a][j] = smallest representable value whose cell index along axis a is >= j
//     wall_lo[a][j] = largest  representable value whose cell index along axis a is <= j-1
//   (wall_lo[a][0] = -inf, wall_hi[a][dim] = +inf).
template <typename T>
struct GridHeader {
    T origin[3];
    T inv_h;
    T h;
    int dim[3];
    int ncells;
    int stride;     // entries per axis in the wall tables
    int pad;
};

// Shape of the occupancy pyramid over a grid (kept apart from GridHeader, which every block of the
// streaming kernels copies to shared memory).
struct PyramidShape {
    int levels;                       // level l (1..levels) halves the resolution l times; the top is 1x1x1
    int lvl_dim[kMaxLevels + 1][3];   // [0] = the grid's own dim
    int lvl_off[kMaxLevels + 1];      // offset of level l inside Cloud::pyramid (level 0 is cell_start itself)
};

template <typename T>
__device__ __forceinline__ int cell_of(T p, T origin, T inv_h, int dim) {
    using R = Real<T>;
    T t = R::mul(R::sub(p, origin), inv_h);
    t = R::vmin(R::vmax(t, (T)0), (T)(dim - 1));   // NaN -> 0
    return (int)t;
}

// One cloud as the kernels see it.
template <typename T>
struct Cloud {
    const T* raw;           // (n, 3) caller's points
    long long n;
    Pt<T>* sorted;          // n points in cell order
    unsigned* rank;         // n: arrival rank of each point inside its cell (cell-wise passes; null in the slab build)
    Pt<T>* part;            // n: the points partitioned by slab (slab build; null in the cell-wise passes)
    unsigned* slab_count;   // slabs: points per slab, then the partition cursors; zeroed per call (slab build)
    unsigned* slab_base;    // slabs + 1: first point of every slab in part / sorted (slab build)
    unsigned* slab_hist;    // slab_chunks * slabs: points per slab of every chunk (slab build)
    unsigned* cell_start;   // cell_cap + 1: counts, then exclusive prefix sums
    GridHeader<T>* grid;
    T* wall_lo;             // 3 * stride
    T* wall_hi;             // 3 * stride
    T* bbox_partial;        // bbox_blocks * 6
    unsigned long long* scan_state;  // per scan tile: status | value (decoupled look-back), zeroed per call
    unsigned* scan_ticket;           // [0] scan tiles / finished slab-histogram CTAs, [1] finished bbox CTAs,
                                     // [2] finished slab-sort CTAs; zeroed per call
    unsigned* occupied;     // number of non-empty cells (counted by the scan), zeroed per call
    unsigned* hint_out;     // host-mapped 8 words of feedback for the next call's grid sizing (grid.cuh), or null
    unsigned* pyramid;      // cell_cap + 64: point counts of the coarser levels (built only when needed)
    PyramidShape* shape;    // written by grid_setup
    int cell_cap;           // upper bound on ncells (host-known)
    int stride;             // wall table stride (host-known)
    int bbox_blocks;        // partial bounding boxes of this cloud (host-known, <= kMaxBBoxBlocks)
    int slabs;              // slab build: slabs of consecutive cells (host-known, <= kMaxSlabs)
    int slab_chunks;        // slab build: CTAs that partition the cloud, one contiguous chunk of points each
    float min_cell;        // lower limit of the cell size (0: none) -- radius searches ask for cells no finer than their reach
};

// How kernels receive the cloud descriptors: a device array (batches) or, for a single pair, by value
// in kernel-parameter space (constant bank: no dependent global loads at the start of every CTA).
template <typename T>
struct CloudsPtr {
    const Cloud<T>* p;
    __device__ __forceinline__ const Cloud<T>& operator[](int i) const { return p[i]; }
};
template <typename T>
struct CloudsVal {
    Cloud<T> v[2];
    __device__ __forceinline__ const Cloud<T>& operator[](int i) const { return v[i]; }
};

constexpr int kMaxBBoxBlocks = 1024;    // partial bounding boxes per cloud, upper bound
constexpr int kBBoxPerThread = 12;      // scalars each thread folds per pass (multiple of 3)
constexpr int kScanItems = 8;           // items per thread in the scan
constexpr int kScanThreads = 512;
constexpr int kScanTile = kScanItems * kScanThreads;
// one-CTA binning of small clouds (bin_small_kernel): the cell counters live in shared memory
constexpr int kSmallThreads = 1024;
constexpr int kSmallMaxCells = 50 * 1024;      // counters: 200 KB of the 227 KB a CTA may own
constexpr long long kSmallMaxPoints = 128 * 1024;
// slab build of larger clouds (grid.cuh)
constexpr int kSlabThreads = 512;               // threads of every slab kernel
constexpr int kSlabTile = 2048;                 // points per staged tile of the chunk walk (4 per thread)
constexpr long long kSlabChunkPoints = 16384;   // points per chunk CTA, until kMaxSlabChunks CTAs are reached
constexpr int kMaxSlabChunks = 128;             // chunk CTAs per cloud
constexpr int kSlabStageBytes = 64 * 1024;      // shared-memory staging of one slab's records
// Mean slab as a share of the staging buffer.  Fuller slabs mean fewer slabs: a cheaper tile scan and longer runs
// per (tile, slab) in the partition, fewer sort CTAs.  At 3/4 a uniform slab (3072 fp32 records, sd ~55) stays far
// below the buffer; a slab that does not fit takes the slower global-memory path (DESIGN.md §4).
constexpr double kSlabMeanFill = 0.75;
constexpr int kSlabMaxCells = 16 * 1024;        // cells per slab, upper bound (shared-memory counters)
constexpr int kMaxSlabs = 8192;                 // = 2^27 cells (the largest cell_cap) / kSlabMaxCells

}  // namespace pcu
