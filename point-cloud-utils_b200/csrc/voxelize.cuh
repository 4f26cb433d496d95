// voxelize.cuh -- triangle-mesh voxelization and 3-D flood fill (the reference's point_cloud_utils/_voxels.py,
// src/voxelize_triangle_mesh.cpp and src/flood_fill_3d.cpp).  Results defined in DESIGN.md §3.
//
// voxelize_triangle_mesh: voxel (i, j, k) is the box centred at o + (i, j, k) s (each product and sum rounded in fp64)
// with half-size s / 2; a face's candidates are the voxels of [ini, ino] per axis, ini = floor((min - o) / s),
// ino = ceil((max - o) / s); a candidate is kept when vx_tri_box (the reference's triBoxOverlap, operation for
// operation in fp64) accepts it.  Pipeline:
//   vx_bounds_kernel   one thread per face: bounds, candidate count (int64), error counts; block scan of the counts
//   vx_tiles_kernel    one CTA: exclusive scan of the tile sums -> a face's first candidate = tile offset + local prefix
//   vx_test_kernel     persistent CTAs walk the flat candidate space in slices of kVxSlice candidates; a slice's faces
//                      come from the prefix sums by binary search, so a face of 10^8 candidates and a million faces of
//                      ten candidates each spread over the SMs alike.  Run twice: counting (kVxCount), then, with the
//                      code buffer sized by that count, writing the kept voxels' Morton codes (kVxCodes).  A third mode
//                      (kVxGrid, make_mesh_watertight) sets the kept voxels' bytes in a dense 2^g-sided grid instead.
//   then the codes' sort (sort.cuh), their run heads (mc_heads_kernel) and vx_decode_kernel, which compacts the heads
//   (keep_rank) and decodes them into the (n, 3) int32 result.
//
// flood_fill_3d: voxel o (linear, z fastest) is adjacent to o +- 1, o +- d and o +- h d when that index is in [0, N),
// so steps past z = d - 1 or y = h - 1 wrap into the next row or slab, as in the reference.  Connected components of
// the voxels equal to the seed's value, by union-find on int32 parents (parent <= index, roots are the smallest index
// of their tree), in passes that do not depend on the region's shape:
//   ff_tile_kernel     union-find in shared memory over a 3-D tile (z fastest): the +1, +d, +h d edges inside it
//   ff_cross_kernel    the edges that leave a tile or wrap, united in global memory with atomicMin (union_find.cuh)
//   ff_out_kernel      out = fill where the voxel's root is the seed's, else the input value
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "meshquery.cuh"
#include "morton.cuh"
#include "sort.cuh"
#include "sparse_voxels.cuh"
#include "union_find.cuh"

namespace pcu {

// ---- voxelize_triangle_mesh ---------------------------------------------------------------------------------------
constexpr int kVxPerThread = 8;
constexpr int kVxSlice = kThreads * kVxPerThread;   // candidates per CTA per step of the persistent loop
// A total of candidates at or above this raises (2^63 less the rounding of a double sum of at most 2^31 terms).
constexpr double kVxMaxCandidates = 0x1p63 * (1.0 - 0x1p-20);

struct VxGeom { double o[3], s[3], h[3]; };          // origin, voxel size, half size (s / 2, exact)
struct VxFace { int ini[3]; int ny, nz; };            // ny = 0: the face tests nothing (an error face)

// What the host reads between the phases (zeroed per call).
struct VxCounts {
    unsigned long long bad_corner;   // faces with a corner outside [0, #v)
    unsigned long long bad_bounds;   // faces with a non-finite vertex or index bounds outside [INT32_MIN, INT32_MAX - 1]
    double cand_d;                   // the candidate total as a double sum (overflow check)
    unsigned long long cand;         // the candidate total (exact when cand_d < kVxMaxCandidates)
    unsigned long long accepted;     // accepted (face, voxel) pairs
    unsigned long long cursor;       // next free record of the emit pass
    long long unique;                // distinct codes (keep_offsets_kernel)
    unsigned long long occupied;     // kVxGrid: voxels whose byte this pass set first
};

// What vx_test_kernel does with an accepted candidate.
enum VxMode { kVxCount, kVxCodes, kVxGrid };

// ((a - b) x (c - b)) style helpers of triBoxOverlap (src/common/tribox.h), every operation rounded on its own
__device__ __forceinline__ bool vx_reject(double pa, double pb, double rad) {   // AXISTEST_*: min / max of two, then the test
    double mn, mx;
    if (pa < pb) { mn = pa; mx = pb; } else { mn = pb; mx = pa; }
    return mn > rad || mx < -rad;
}
__device__ __forceinline__ double vx_px(double a, double b, const double* v) { return __dsub_rn(__dmul_rn(a, v[1]), __dmul_rn(b, v[2])); }
__device__ __forceinline__ double vx_py(double a, double b, const double* v) { return __dadd_rn(__dmul_rn(-a, v[0]), __dmul_rn(b, v[2])); }
__device__ __forceinline__ double vx_pz(double a, double b, const double* v) { return __dsub_rn(__dmul_rn(a, v[0]), __dmul_rn(b, v[1])); }
__device__ __forceinline__ double vx_rad(double fa, double fb, double ha, double hb) { return __dadd_rn(__dmul_rn(fa, ha), __dmul_rn(fb, hb)); }
__device__ __forceinline__ bool vx_minmax_reject(double x0, double x1, double x2, double h) {   // FINDMINMAX, then the test
    double mn = x0, mx = x0;
    if (x1 < mn) mn = x1;
    if (x1 > mx) mx = x1;
    if (x2 < mn) mn = x2;
    if (x2 > mx) mx = x2;
    return mn > h || mx < -h;
}
__device__ __forceinline__ double vx_dot(const double* a, const double* b) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// triBoxOverlap(c, h, {a, b, d}) in the reference's order of tests and operations.
__device__ __forceinline__ bool vx_tri_box(const double c[3], const double h[3], const double a[3], const double b[3], const double d[3]) {
    double v0[3], v1[3], v2[3], e0[3], e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { v0[k] = __dsub_rn(a[k], c[k]); v1[k] = __dsub_rn(b[k], c[k]); v2[k] = __dsub_rn(d[k], c[k]); }
#pragma unroll
    for (int k = 0; k < 3; ++k) { e0[k] = __dsub_rn(v1[k], v0[k]); e1[k] = __dsub_rn(v2[k], v1[k]); e2[k] = __dsub_rn(v0[k], v2[k]); }
    double fx = fabs(e0[0]), fy = fabs(e0[1]), fz = fabs(e0[2]);
    if (vx_reject(vx_px(e0[2], e0[1], v0), vx_px(e0[2], e0[1], v2), vx_rad(fz, fy, h[1], h[2]))) return false;   // X01
    if (vx_reject(vx_py(e0[2], e0[0], v0), vx_py(e0[2], e0[0], v2), vx_rad(fz, fx, h[0], h[2]))) return false;   // Y02
    if (vx_reject(vx_pz(e0[1], e0[0], v2), vx_pz(e0[1], e0[0], v1), vx_rad(fy, fx, h[0], h[1]))) return false;   // Z12
    fx = fabs(e1[0]); fy = fabs(e1[1]); fz = fabs(e1[2]);
    if (vx_reject(vx_px(e1[2], e1[1], v0), vx_px(e1[2], e1[1], v2), vx_rad(fz, fy, h[1], h[2]))) return false;   // X01
    if (vx_reject(vx_py(e1[2], e1[0], v0), vx_py(e1[2], e1[0], v2), vx_rad(fz, fx, h[0], h[2]))) return false;   // Y02
    if (vx_reject(vx_pz(e1[1], e1[0], v0), vx_pz(e1[1], e1[0], v1), vx_rad(fy, fx, h[0], h[1]))) return false;   // Z0
    fx = fabs(e2[0]); fy = fabs(e2[1]); fz = fabs(e2[2]);
    if (vx_reject(vx_px(e2[2], e2[1], v0), vx_px(e2[2], e2[1], v1), vx_rad(fz, fy, h[1], h[2]))) return false;   // X2
    if (vx_reject(vx_py(e2[2], e2[0], v0), vx_py(e2[2], e2[0], v1), vx_rad(fz, fx, h[0], h[2]))) return false;   // Y1
    if (vx_reject(vx_pz(e2[1], e2[0], v2), vx_pz(e2[1], e2[0], v1), vx_rad(fy, fx, h[0], h[1]))) return false;   // Z12
#pragma unroll
    for (int k = 0; k < 3; ++k)
        if (vx_minmax_reject(v0[k], v1[k], v2[k], h[k])) return false;
    const double n[3] = {__dsub_rn(__dmul_rn(e0[1], e1[2]), __dmul_rn(e0[2], e1[1])),
                         __dsub_rn(__dmul_rn(e0[2], e1[0]), __dmul_rn(e0[0], e1[2])),
                         __dsub_rn(__dmul_rn(e0[0], e1[1]), __dmul_rn(e0[1], e1[0]))};
    double vmin[3], vmax[3];                          // planeBoxOverlap(n, v0, h)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (n[k] > 0.0) { vmin[k] = __dsub_rn(-h[k], v0[k]); vmax[k] = __dsub_rn(h[k], v0[k]); }
        else            { vmin[k] = __dsub_rn(h[k], v0[k]); vmax[k] = __dsub_rn(-h[k], v0[k]); }
    }
    if (vx_dot(n, vmin) > 0.0) return false;
    return vx_dot(n, vmax) >= 0.0;
}

// std::min / std::max of the reference's bounds (finite inputs: the caller has checked them)
__device__ __forceinline__ double vx_min3(double a, double b, double c) { const double bc = c < b ? c : b; return bc < a ? bc : a; }
__device__ __forceinline__ double vx_max3(double a, double b, double c) { const double bc = b < c ? c : b; return a < bc ? bc : a; }

template <typename T>
__global__ void __launch_bounds__(kThreads) vx_bounds_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                             long long m, const __grid_constant__ VxGeom g, VxFace* __restrict__ faces,
                                                             unsigned long long* __restrict__ local_start,
                                                             unsigned long long* __restrict__ tile_sum, VxCounts* __restrict__ counts) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    unsigned long long cnt = 0;
    double cnt_d = 0.0;
    if (t < m) {
        VxFace fc = {{0, 0, 0}, 0, 0};
        double a[3], b[3], c[3];
        cnt = 1;                                      // an error face holds one candidate that tests nothing
        if (!mq_corners<T>(v, nv, f, fkind, t, a, b, c)) {
            atomicAdd(&counts->bad_corner, 1ull);
        } else {
            bool ok = true;
            double q[6];                              // (min - o) / s, then (max - o) / s, per axis
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                ok = ok && isfinite(a[k]) && isfinite(b[k]) && isfinite(c[k]);
                q[k] = __dsub_rn(vx_min3(a[k], b[k], c[k]), g.o[k]);
                q[k + 3] = __dsub_rn(vx_max3(a[k], b[k], c[k]), g.o[k]);
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) q[k] = __ddiv_rn(q[k], g.s[k % 3]);
            double lo[3], hi[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                lo[k] = floor(q[k]);
                hi[k] = ceil(q[k + 3]);
                ok = ok && lo[k] >= -2147483648.0 && hi[k] <= 2147483646.0;   // also false for NaN
            }
            if (!ok) {
                atomicAdd(&counts->bad_bounds, 1ull);
            } else {
                const double ex = hi[0] - lo[0] + 1.0, ey = hi[1] - lo[1] + 1.0, ez = hi[2] - lo[2] + 1.0;   // exact
#pragma unroll
                for (int k = 0; k < 3; ++k) fc.ini[k] = (int)lo[k];
                fc.ny = (int)(long long)ey;             // at most 2^32 - 1: wraps, and is read back as unsigned
                fc.nz = (int)(long long)ez;
                cnt_d = ex * ey * ez;
                cnt = (unsigned long long)ex * (unsigned long long)ey * (unsigned long long)ez;   // exact unless cnt_d is too large
            }
        }
        faces[t] = fc;
    }
    unsigned long long total;
    const unsigned long long ex = block_exclusive_scan<kThreads, unsigned long long>(cnt, &total);
    if (t < m) local_start[t] = ex;
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
    double dtotal;
    block_exclusive_scan<kThreads, double>(cnt_d, &dtotal);
    if (threadIdx.x == 0 && dtotal != 0.0) atomicAdd(&counts->cand_d, dtotal);
}

// One CTA: tile offsets (exclusive, in place) and the candidate total.
__global__ void __launch_bounds__(1024) vx_tiles_kernel(unsigned long long* __restrict__ tile_sum, long long tiles, VxCounts* __restrict__ counts) {
    const unsigned long long all = block_scan_rounds<1024, unsigned long long>(
        (unsigned)tiles, [&](unsigned b) { return tile_sum[b]; }, [&](unsigned b, unsigned long long ex, unsigned long long) { tile_sum[b] = ex; });
    if (threadIdx.x == 0) counts->cand = all;
}

__device__ __forceinline__ unsigned long long vx_start(const unsigned long long* __restrict__ local_start,
                                                       const unsigned long long* __restrict__ tile_off, long long f) {
    return __ldg(tile_off + (f / kThreads)) + __ldg(local_start + f);
}

// Last face whose first candidate is <= c (faces hold at least one candidate each, so it holds c).
__device__ __forceinline__ long long vx_face_of(const unsigned long long* __restrict__ local_start,
                                                const unsigned long long* __restrict__ tile_off, long long m, unsigned long long c) {
    long long lo = 0, hi = m;                         // first face with start > c
    while (lo < hi) {
        const long long mid = lo + ((hi - lo) >> 1);
        if (vx_start(local_start, tile_off, mid) <= c) lo = mid + 1; else hi = mid;
    }
    return lo - 1;
}

// Persistent CTAs over the flat candidate space, kVxSlice candidates per step.  The slice's faces (at most kVxSlice)
// and their first candidates go to shared memory; candidate c of the slice finds its face there by binary search.
// kVxCount: adds the accepted count to counts->accepted.  kVxCodes: writes the accepted voxels' codes as sort records,
// at positions handed out per slice by one atomicAdd on counts->cursor (their order is the sort's business).  kVxGrid:
// sets byte (i 2^g + j) 2^g + k of `grid` (2^(3g) bytes, zero or one each, addressed as 32-bit words) to one for every
// accepted voxel inside [0, 2^g)^3 -- idempotent, so no order and no sort -- and adds the voxels whose byte it set
// first to counts->occupied.  Nothing runs when the bounds pass found an error or the total overflows.
template <typename T, int kMode>
__global__ void __launch_bounds__(kThreads) vx_test_kernel(const T* __restrict__ v, long long nv, const void* __restrict__ f, int fkind,
                                                           long long m, const __grid_constant__ VxGeom g, const VxFace* __restrict__ faces,
                                                           const unsigned long long* __restrict__ local_start,
                                                           const unsigned long long* __restrict__ tile_off, VxCounts* __restrict__ counts,
                                                           McRec* __restrict__ recs, unsigned* __restrict__ grid = nullptr, int lg = 0) {
    constexpr bool kEmit = kMode == kVxCodes;
    __shared__ unsigned long long s_start[kVxSlice + 1];
    __shared__ long long s_face[2];
    __shared__ unsigned long long s_base;
    __shared__ unsigned long long s_code[kEmit ? kVxPerThread : 1][kThreads];
    const bool ok = counts->bad_corner == 0 && counts->bad_bounds == 0 && counts->cand_d < kVxMaxCandidates;
    const unsigned long long total = ok ? counts->cand : 0ull;
    unsigned long long mine = 0;                     // kEmit = false: this thread's accepted candidates
    for (unsigned long long s0 = (unsigned long long)blockIdx.x * kVxSlice; s0 < total; s0 += (unsigned long long)gridDim.x * kVxSlice) {
        const unsigned long long s1 = min(total, s0 + kVxSlice);
        if (threadIdx.x < 2) s_face[threadIdx.x] = vx_face_of(local_start, tile_off, m, threadIdx.x ? s1 - 1 : s0);
        __syncthreads();
        const long long f0 = s_face[0];
        const int nface = (int)(s_face[1] - f0 + 1);
        for (int j = threadIdx.x; j < nface; j += kThreads) s_start[j] = vx_start(local_start, tile_off, f0 + j);
        __syncthreads();
        int kept = 0;
#pragma unroll 1
        for (int r = 0; r < kVxPerThread; ++r) {
            const unsigned long long c = s0 + (unsigned long long)(r * kThreads + threadIdx.x);
            if (c >= s1) break;
            int lo = 0, hi = nface;                   // last face of the slice with start <= c
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (s_start[mid] <= c) lo = mid; else hi = mid;
            }
            const long long t = f0 + lo;
            const VxFace fc = faces[t];
            if (fc.ny == 0) continue;
            const unsigned long long q = c - s_start[lo];
            const unsigned long long ny = (unsigned)fc.ny, nz = (unsigned)fc.nz;
            unsigned long long yz, dz;
            if (q < (1ull << 32) && nz < (1ull << 32)) { const unsigned q32 = (unsigned)q; yz = q32 / (unsigned)nz; dz = q32 - (unsigned)yz * (unsigned)nz; }
            else { yz = q / nz; dz = q - yz * nz; }
            const unsigned long long dx = yz / ny, dy = yz - dx * ny;
            const int idx[3] = {(int)(fc.ini[0] + (long long)dx), (int)(fc.ini[1] + (long long)dy), (int)(fc.ini[2] + (long long)dz)};
            double a[3], b[3], cc[3], ctr[3];
            mq_corners<T>(v, nv, f, fkind, t, a, b, cc);
#pragma unroll
            for (int k = 0; k < 3; ++k) ctr[k] = __dadd_rn(g.o[k], __dmul_rn((double)idx[k], g.s[k]));
            if (vx_tri_box(ctr, g.h, a, b, cc)) {
                if constexpr (kEmit) s_code[kept][threadIdx.x] = morton_encode3(idx[0], idx[1], idx[2]);
                if constexpr (kMode == kVxGrid) {
                    const unsigned side = 1u << lg;
                    if ((unsigned)idx[0] < side && (unsigned)idx[1] < side && (unsigned)idx[2] < side) {
                        const unsigned long long o = ((unsigned long long)idx[0] << (2 * lg)) | ((unsigned long long)idx[1] << lg) | (unsigned)idx[2];
                        const unsigned bit = 1u << (8 * (unsigned)(o & 3));
                        if (!(atomicOr(grid + (o >> 2), bit) & bit)) ++kept;
                    }
                    continue;
                }
                ++kept;
            }
        }
        if constexpr (kEmit) {
            unsigned total_kept;
            const unsigned before = block_exclusive_scan<kThreads>((unsigned)kept, &total_kept);
            if (threadIdx.x == 0) s_base = atomicAdd(&counts->cursor, (unsigned long long)total_kept);
            __syncthreads();
            const unsigned long long base = s_base + before;
            for (int j = 0; j < kept; ++j) {
                McRec rec;
                rec.key[0] = s_code[j][threadIdx.x];
                rec.idx = 0ull;
                store_rec(recs + base + j, rec);
            }
        } else {
            mine += (unsigned long long)kept;
        }
        __syncthreads();                             // s_start, s_face and s_code are reused by the next slice
    }
    if constexpr (!kEmit) {
        unsigned long long all;
        block_exclusive_scan<kThreads, unsigned long long>(mine, &all);
        if (threadIdx.x == 0 && all) atomicAdd(kMode == kVxGrid ? &counts->occupied : &counts->accepted, all);
    }
}

// After keep_count / keep_offsets over the run heads of the sorted codes: each head decodes into row rank(head).
__global__ void __launch_bounds__(kThreads) vx_decode_kernel(const McRec* __restrict__ recs, long long n, const unsigned char* __restrict__ head,
                                                             const unsigned* __restrict__ block_offset, int* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool mine = i < n && head[i];
    const unsigned pos = keep_rank(mine, block_offset);
    if (!mine) return;
    int x, y, z;
    morton_decode3(recs[i].key[0], x, y, z);
    out[3ull * pos] = x; out[3ull * pos + 1] = y; out[3ull * pos + 2] = z;
}

// ---- flood_fill_3d ------------------------------------------------------------------------------------------------
constexpr int kFfTileMax = 1024;                       // voxels per tile (tile sides are powers of two)
constexpr int kFfPerThread = kFfTileMax / kThreads;

// Grid w x h x d and its tiling: tiles of 2^lx x 2^ly x 2^lz voxels, tile index z fastest.
struct FfShape {
    long long w, h, d, n;                             // n = w h d < 2^31
    long long seed;                                   // linear index of the seed
    int lx, ly, lz;
    unsigned ty_n, tz_n;                              // tiles along y and z
};

// This CTA's tile: the grid coordinates of its first voxel.
struct FfTile { long long x0, y0, z0; };
__device__ __forceinline__ FfTile ff_tile(const FfShape& s) {
    const unsigned b = blockIdx.x;
    FfTile t;
    t.z0 = (long long)(b % s.tz_n) << s.lz;
    t.y0 = (long long)((b / s.tz_n) % s.ty_n) << s.ly;
    t.x0 = (long long)(b / (s.tz_n * s.ty_n)) << s.lx;
    return t;
}
// Voxel i (0 .. kFfTileMax) of the tile: grid coordinates, and whether it lies inside the tile and the grid.
struct FfVoxel { long long x, y, z, o; int ix, iy, iz; bool in; };
__device__ __forceinline__ FfVoxel ff_voxel(const FfShape& s, const FfTile& t, int i) {
    FfVoxel r;
    r.iz = i & ((1 << s.lz) - 1);
    r.iy = (i >> s.lz) & ((1 << s.ly) - 1);
    r.ix = i >> (s.lz + s.ly);
    r.x = t.x0 + r.ix;
    r.y = t.y0 + r.iy;
    r.z = t.z0 + r.iz;
    r.in = r.ix < (1 << s.lx) && r.x < s.w && r.y < s.h && r.z < s.d;
    r.o = (r.x * s.h + r.y) * s.d + r.z;
    return r;
}

// T's ==: IEEE for floats (NaN equals nothing, -0.0 equals 0.0)
template <typename T>
__device__ __forceinline__ bool ff_eq(const T* __restrict__ grid, long long o, T sv) { return __ldg(grid + o) == sv; }

// Parents are read through volatile loads: other threads change them while a union runs.
__device__ __forceinline__ int ff_find_shared(const int* lab, int x) {
    const volatile int* l = lab;
    while (l[x] != x) x = l[x];
    return x;
}
// Unites the trees of a and b: the larger root is pointed at the smaller one with atomicMin; when that root had
// meanwhile been given another parent, that parent is united with the smaller root in turn.
__device__ __forceinline__ void ff_union_shared(int* lab, int a, int b) {
    while (true) {
        a = ff_find_shared(lab, a);
        b = ff_find_shared(lab, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(&lab[a], b);
        if (old == a) return;
        a = old;
    }
}
// Tile-local components of the voxels equal to the seed's value; P[o] = the tile root's linear index (o for the others).
template <typename T>
__global__ void __launch_bounds__(kThreads) ff_tile_kernel(const T* __restrict__ grid, const __grid_constant__ FfShape s, int* __restrict__ P) {
    __shared__ int lab[kFfTileMax];
    __shared__ unsigned char eq[kFfTileMax];
    const T sv = __ldg(grid + s.seed);
    const FfTile tile = ff_tile(s);
    const int tz = 1 << s.lz, tyz = 1 << (s.ly + s.lz);
#pragma unroll
    for (int k = 0; k < kFfPerThread; ++k) {
        const int i = threadIdx.x + k * kThreads;
        const FfVoxel p = ff_voxel(s, tile, i);
        lab[i] = i;
        eq[i] = p.in && ff_eq(grid, p.o, sv);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kFfPerThread; ++k) {
        const int i = threadIdx.x + k * kThreads;
        if (!eq[i]) continue;
        const FfVoxel p = ff_voxel(s, tile, i);
        if (p.iz + 1 < tz && p.z + 1 < s.d && eq[i + 1]) ff_union_shared(lab, i, i + 1);
        if (p.iy + 1 < (1 << s.ly) && p.y + 1 < s.h && eq[i + tz]) ff_union_shared(lab, i, i + tz);
        if (p.ix + 1 < (1 << s.lx) && p.x + 1 < s.w && eq[i + tyz]) ff_union_shared(lab, i, i + tyz);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kFfPerThread; ++k) {
        const int i = threadIdx.x + k * kThreads;
        const FfVoxel p = ff_voxel(s, tile, i);
        if (!p.in) continue;
        P[p.o] = eq[i] ? (int)ff_voxel(s, tile, ff_find_shared(lab, i)).o : (int)p.o;
    }
}

// The forward edges the tile pass did not take: those leaving the tile, and the wraps past z = d - 1 and y = h - 1.
template <typename T>
__global__ void __launch_bounds__(kThreads) ff_cross_kernel(const T* __restrict__ grid, const __grid_constant__ FfShape s, int* __restrict__ P) {
    const T sv = __ldg(grid + s.seed);
    const FfTile tile = ff_tile(s);
#pragma unroll 1
    for (int k = 0; k < kFfPerThread; ++k) {
        const int i = threadIdx.x + k * kThreads;
        const FfVoxel p = ff_voxel(s, tile, i);
        if (!p.in) continue;
        const bool ez = (p.iz == (1 << s.lz) - 1 || p.z == s.d - 1) && p.o + 1 < s.n;
        const bool ey = (p.iy == (1 << s.ly) - 1 || p.y == s.h - 1) && p.o + s.d < s.n;
        const bool ex = p.ix == (1 << s.lx) - 1 && p.x + 1 < s.w;
        if (!(ez || ey || ex) || !ff_eq(grid, p.o, sv)) continue;
        if (ez && ff_eq(grid, p.o + 1, sv)) uf_union(P, (int)p.o, (int)(p.o + 1));
        if (ey && ff_eq(grid, p.o + s.d, sv)) uf_union(P, (int)p.o, (int)(p.o + s.d));
        if (ex && ff_eq(grid, p.o + s.h * s.d, sv)) uf_union(P, (int)p.o, (int)(p.o + s.h * s.d));
    }
}

// out[o] = fill for the voxels of the seed's component, grid[o] elsewhere.  fill == seed value: an unchanged copy
// (the reference never returns there).
template <typename T>
__global__ void __launch_bounds__(kThreads) ff_out_kernel(const T* __restrict__ grid, long long n, long long seed, T fill,
                                                          int* __restrict__ P, T* __restrict__ out) {
    __shared__ int s_root;
    const T sv = __ldg(grid + seed);
    if (threadIdx.x == 0) s_root = uf_find(P, (int)seed);
    __syncthreads();
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (o >= n) return;
    const T x = __ldg(grid + o);
    out[o] = (x == sv && !(fill == sv) && uf_find(P, (int)o) == s_root) ? fill : x;
}

}  // namespace pcu
