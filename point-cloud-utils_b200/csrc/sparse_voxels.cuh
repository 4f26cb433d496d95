// sparse_voxels.cuh -- marching cubes on a sparse voxel grid and the boundary of a sparse voxel grid.
//
// marching_cubes_sparse_voxel_grid (the reference's src/marching_cubes.cpp:35-85, which calls igl::marching_cubes):
// the result is defined in DESIGN.md §3.  Pipeline, one thread per cube or per slot (a crossing edge of a cube; slots
// are numbered cube by cube, edge by edge):
//   mc_classify_kernel   case byte of every cube, bad-index count, slots and triangles per CTA tile
//   mc_tiles_kernel      one CTA: exclusive scans of the tile totals -> first slot and first face of every tile
//   mc_slots_kernel      per slot the record {key = (min corner << b) | max corner, slot}, sorted by sort.cuh
//   mc_heads_kernel      (runtime.cu) run heads of the sorted keys (keep_count / keep_offsets number them: one run per vertex)
//   mc_runs_kernel       per slot its run; the run head (the run's smallest slot: the sort is stable) owns the run
//   mc_owner_kernel      the owners, counted in slot order (keep_count / keep_offsets), give each run its vertex id
//   mc_emit_kernel       owners write their vertex, cubes their faces
// A cube's first slot and first face are its tile's plus a block scan of the cube counts in the tile, recomputed from
// the case bytes wherever they are needed, so no per-cube offsets are stored.
//
// sparse_voxel_grid_boundary (src/sparse_voxel_grid.cpp:463-522): Morton codes of the voxels (the reference's
// safe_cast range check first), sorted; a voxel is on the boundary when one of its six face neighbours' codes
// (morton_add2, in the reference's offset order) is not among them.  Integer work only.
//
// Sparse voxel grids (sparse_voxel_grid_from_pointcloud, dilate / erode_sparse_voxel_grid,
// sparse_voxel_grid_to_hex_mesh; the reference's src/sparse_voxel_grid.cpp:78-460) and voxel_grid_geometry
// (src/mesh_for_voxels.cpp): results defined in DESIGN.md §3.  Each builds a set of code records and sorts it with
// sort.cuh; run heads (mc_heads_kernel) and the compaction of compact.cuh number the distinct codes:
//   svg_point_codes_kernel  {code, point} of every point (fp64 quantisation, range check)
//   svg_dilate_flag_kernel  per sorted voxel and neighbour offset: the missing neighbours this voxel owns
//   svg_dilate_write_kernel the owned neighbours' codes, compacted (already distinct; sorted afterwards)
//   svg_erode_flag_kernel   per voxel: all 26 neighbours present; svg_keep_voxels_kernel copies the kept rows
//   svg_corners_kernel      {corner code, 8 i + k} of every cube corner
//   svg_decode_kernel       distinct codes -> integer rows or hex vertices
//   svg_rank_kernel         run rank of every record scattered to its index (point_to_vox, cubes)
//   vg_geometry_kernel      the cube mesh of every voxel (no sort; sizes known in advance)
#pragma once
#include <type_traits>
#include "common.cuh"
#include "compact.cuh"
#include "morton.cuh"
#include "sort.cuh"
#include "mc_tables.h"

namespace pcu {

using McRec = SortRec<unsigned long long, 1>;

// What the host reads between the phases (zeroed per call).
struct McCounts {
    unsigned long long slots;   // crossing edges over all cubes
    unsigned long long faces;
    unsigned long long bad;     // cubes with a corner outside [0, n)
    long long verts;            // distinct keys (written by keep_offsets_kernel)
};

// Corner `end` (0: first, 1: second) of edge e: (0,1) (1,2) (2,3) (3,0) (4,5) (5,6) (6,7) (7,4) (0,4) (1,5) (2,6) (3,7),
// the numbering of tools/mc_tables.py.  Constant under an unrolled loop over e.
__host__ __device__ constexpr int mc_edge_corner(int e, int end) {
    return e < 8 ? (end ? (e & 4) + ((e + 1) & 3) : e) : (end ? e - 4 : e - 8);
}

// The 8 corner indices of cube c as unsigned 64-bit values, W-byte entries in 16-byte loads (rows are 32 or 64 bytes,
// the base 16-byte aligned).  Any entry >= n is out of range: negative signed entries are too, since n < 2^31 - 1.
template <int W>
__device__ __forceinline__ void mc_load_cube(const void* __restrict__ idx, long long c, unsigned long long (&v)[8]) {
    if (W == 4) {
        const uint4* p = reinterpret_cast<const uint4*>(idx) + 2 * c;
        const uint4 a = __ldg(p), b = __ldg(p + 1);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(idx) + 4 * c;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const ulonglong2 a = __ldg(p + k);
            v[2 * k] = a.x; v[2 * k + 1] = a.y;
        }
    }
}
template <int W>
__device__ __forceinline__ bool mc_in_range(unsigned long long v, long long n) {
    return (W == 4 ? (unsigned long long)(unsigned)v : v) < (unsigned long long)n;
}

// slots in bits 0-15, triangles in bits 16-31: a CTA's sums stay below 2^16 and 2^16 respectively
__device__ __forceinline__ unsigned mc_packed_counts(unsigned cs) {
    return (unsigned)__popc(__ldg(&kMcEdgeMask[cs])) | (unsigned)__ldg(&kMcTriCount[cs]) << 16;
}

template <typename T, typename S, int W>
__global__ void __launch_bounds__(kThreads) mc_classify_kernel(const S* __restrict__ scalars, long long n, const void* __restrict__ idx,
                                                               long long m, T iso, unsigned char* __restrict__ cases,
                                                               unsigned* __restrict__ tile_sum, McCounts* __restrict__ counts) {
    const long long c = (long long)blockIdx.x * kThreads + threadIdx.x;
    unsigned cs = 0;
    if (c < m) {
        unsigned long long v[8];
        mc_load_cube<W>(idx, c, v);
        bool ok = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) ok = ok && mc_in_range<W>(v[k], n);
        if (ok) {
#pragma unroll
            for (int k = 0; k < 8; ++k) cs |= ((T)__ldg(scalars + v[k]) > iso ? 1u : 0u) << k;   // NaN: not above
        } else {
            atomicAdd(&counts->bad, 1ull);
        }
        cases[c] = (unsigned char)cs;
    }
    unsigned total;
    block_exclusive_scan<kThreads>(c < m ? mc_packed_counts(cs) : 0u, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// One CTA: tile_slot0 / tile_face0 = exclusive prefix sums of the tiles' slots / faces; the totals into *counts.
__global__ void __launch_bounds__(1024) mc_tiles_kernel(const unsigned* __restrict__ tile_sum, long long tiles,
                                                        unsigned long long* __restrict__ tile_slot0,
                                                        unsigned long long* __restrict__ tile_face0, McCounts* __restrict__ counts) {
    const unsigned long long slots = block_scan_rounds<1024, unsigned long long>(
        (unsigned)tiles, [&](unsigned b) { return tile_sum[b] & 0xffffu; },
        [&](unsigned b, unsigned long long ex, unsigned long long) { tile_slot0[b] = ex; });
    const unsigned long long faces = block_scan_rounds<1024, unsigned long long>(
        (unsigned)tiles, [&](unsigned b) { return tile_sum[b] >> 16; },
        [&](unsigned b, unsigned long long ex, unsigned long long) { tile_face0[b] = ex; });
    if (threadIdx.x == 0) { counts->slots = slots; counts->faces = faces; }
}

// This thread's cube's case and first slot / first face (block-wide: every thread of the CTA calls it).
struct McCube { unsigned cs; unsigned long long slot0, face0; };
__device__ __forceinline__ McCube mc_cube_offsets(const unsigned char* __restrict__ cases, long long m,
                                                  const unsigned long long* __restrict__ tile_slot0,
                                                  const unsigned long long* __restrict__ tile_face0) {
    const long long c = (long long)blockIdx.x * kThreads + threadIdx.x;
    McCube r;
    r.cs = c < m ? cases[c] : 0u;
    unsigned total;
    const unsigned ex = block_exclusive_scan<kThreads>(mc_packed_counts(r.cs), &total);
    r.slot0 = tile_slot0[blockIdx.x] + (ex & 0xffffu);
    r.face0 = tile_face0[blockIdx.x] + (ex >> 16);
    return r;
}

template <int W>
__global__ void __launch_bounds__(kThreads) mc_slots_kernel(const void* __restrict__ idx, const unsigned char* __restrict__ cases, long long m,
                                                            const unsigned long long* __restrict__ tile_slot0,
                                                            const unsigned long long* __restrict__ tile_face0, int key_shift,
                                                            McRec* __restrict__ recs) {
    const McCube cube = mc_cube_offsets(cases, m, tile_slot0, tile_face0);
    const unsigned mask = __ldg(&kMcEdgeMask[cube.cs]);
    if (mask == 0u) return;
    unsigned long long v[8];
    mc_load_cube<W>(idx, (long long)blockIdx.x * kThreads + threadIdx.x, v);
    unsigned s = (unsigned)cube.slot0;           // the host has checked that slots fit 32 bits
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        if (mask >> e & 1u) {
            const unsigned long long a = v[mc_edge_corner(e, 0)], b = v[mc_edge_corner(e, 1)];
            McRec r;
            r.key[0] = (a < b ? a : b) << key_shift | (a < b ? b : a);
            r.idx = s;
            store_rec(recs + s, r);
            ++s;
        }
    }
}

// After keep_count / keep_offsets over `head`: run of every sorted record = heads at or before it, minus one.
__global__ void __launch_bounds__(kThreads) mc_runs_kernel(const McRec* __restrict__ recs, long long ns, const unsigned char* __restrict__ head,
                                                           const unsigned* __restrict__ block_offset, unsigned* __restrict__ slot_run,
                                                           unsigned char* __restrict__ owner) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < ns ? head[i] : 0u;
    const unsigned run = keep_rank<true>(mine, block_offset) - 1u;
    if (i >= ns) return;
    const unsigned long long slot = recs[i].idx;
    slot_run[slot] = run;
    owner[slot] = (unsigned char)mine;
}

// After keep_count / keep_offsets over `owner` (slot order): the owner of each run gives the run its vertex id.
__global__ void __launch_bounds__(kThreads) mc_owner_kernel(const unsigned char* __restrict__ owner, long long ns,
                                                            const unsigned* __restrict__ block_offset, const unsigned* __restrict__ slot_run,
                                                            unsigned* __restrict__ run_vid) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = s < ns ? owner[s] : 0u;
    const unsigned vid = keep_rank(mine, block_offset);
    if (mine) run_vid[slot_run[s]] = vid;
}

template <typename T> __device__ __forceinline__ T mc_div(T a, T b);
template <> __device__ __forceinline__ float mc_div<float>(float a, float b) { return __fdiv_rn(a, b); }
template <> __device__ __forceinline__ double mc_div<double>(double a, double b) { return __ddiv_rn(a, b); }

// Owner slots write their vertex (t = (iso - s_i) / (s_j - s_i), v = g_i + t (g_j - g_i), each operation rounded in T),
// every crossing cube its faces: vertex ids of its crossing edges, in the case's table order.
template <typename T, typename S, int W>
__global__ void __launch_bounds__(kThreads) mc_emit_kernel(const S* __restrict__ scalars, const T* __restrict__ coords, const void* __restrict__ idx,
                                                           const unsigned char* __restrict__ cases, long long m,
                                                           const unsigned long long* __restrict__ tile_slot0,
                                                           const unsigned long long* __restrict__ tile_face0, T iso,
                                                           const unsigned* __restrict__ slot_run, const unsigned* __restrict__ run_vid,
                                                           const unsigned char* __restrict__ owner, T* __restrict__ out_v,
                                                           void* __restrict__ out_f) {
    using R = Real<T>;
    __shared__ unsigned vid[12][kThreads];
    const McCube cube = mc_cube_offsets(cases, m, tile_slot0, tile_face0);
    const unsigned mask = __ldg(&kMcEdgeMask[cube.cs]);
    if (mask == 0u) return;
    unsigned long long v[8];
    mc_load_cube<W>(idx, (long long)blockIdx.x * kThreads + threadIdx.x, v);
    unsigned s = (unsigned)cube.slot0;           // the host has checked that slots fit 32 bits
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        if (mask >> e & 1u) {
            const unsigned id = __ldg(run_vid + __ldg(slot_run + s));
            vid[e][threadIdx.x] = id;
            if (__ldg(owner + s)) {
                const unsigned long long a = v[mc_edge_corner(e, 0)], b = v[mc_edge_corner(e, 1)];
                const T si = (T)__ldg(scalars + a), sj = (T)__ldg(scalars + b);
                const T t = mc_div<T>(R::sub(iso, si), R::sub(sj, si));
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const T gi = __ldg(coords + 3 * a + k), gj = __ldg(coords + 3 * b + k);
                    out_v[3ull * id + k] = R::add(gi, R::mul(t, R::sub(gj, gi)));
                }
            }
            ++s;
        }
    }
    const int nt = __ldg(&kMcTriCount[cube.cs]);
    const unsigned char* tri = kMcTris[cube.cs];
#pragma unroll 1
    for (int j = 0; j < 3 * nt; ++j) {
        const unsigned id = vid[__ldg(tri + j)][threadIdx.x];
        if constexpr (W == 4) reinterpret_cast<unsigned*>(out_f)[3ull * cube.face0 + j] = id;
        else reinterpret_cast<unsigned long long*>(out_f)[3ull * cube.face0 + j] = id;
    }
}

// ---- sparse_voxel_grid_boundary ----------------------------------------------------------------------------------
// safe_cast<Tfrom, int32_t> (sparse_voxel_grid.cpp:12-21) for a signed Tfrom: INT32_MIN and INT32_MAX are rejected too.
__device__ __forceinline__ bool svb_fits(long long x) { return x <= 2147483646ll && x >= -2147483647ll; }

template <typename I>
__device__ __forceinline__ unsigned long long svb_code(const I* __restrict__ g, long long i) {
    return morton_encode3((int)g[3 * i], (int)g[3 * i + 1], (int)g[3 * i + 2]);
}

// Codes of every voxel, as records for the sort; *bad counts voxels with a coordinate out of safe_cast's range.
template <typename I>
__global__ void __launch_bounds__(kThreads) svb_codes_kernel(const I* __restrict__ g, long long n, McRec* __restrict__ recs,
                                                             unsigned long long* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!svb_fits((long long)g[3 * i]) || !svb_fits((long long)g[3 * i + 1]) || !svb_fits((long long)g[3 * i + 2])) atomicAdd(bad, 1ull);
    McRec r;
    r.key[0] = svb_code<I>(g, i);
    r.idx = (unsigned long long)i;
    store_rec(recs + i, r);
}

// std::lower_bound of code q in the n sorted codes, and the reference's vector_binsearch test on it.
__device__ __forceinline__ long long svb_lower_bound(const McRec* __restrict__ sorted, long long n, unsigned long long q) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = lo + ((hi - lo) >> 1);
        if (__ldg(&sorted[mid].key[0]) < q) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ bool svb_missing(const McRec* __restrict__ sorted, long long n, unsigned long long q) {
    const long long lo = svb_lower_bound(sorted, n, q);
    return lo == n || __ldg(&sorted[lo].key[0]) != q;
}

// keep[i] = 1 when one of voxel i's six face neighbours (+x, -x, +y, -y, +z, -z: the reference's order) is missing
template <typename I>
__global__ void __launch_bounds__(kThreads) svb_flag_kernel(const I* __restrict__ g, long long n, const McRec* __restrict__ sorted,
                                                            unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long code = svb_code<I>(g, i);
    bool boundary = false;
    for (int o = 0; o < 6 && !boundary; ++o) {
        const int d = (o & 1) ? -1 : 1, a = o >> 1;
        const unsigned long long q = morton_add2(code, morton_encode3(a == 0 ? d : 0, a == 1 ? d : 0, a == 2 ? d : 0));
        boundary = svb_missing(sorted, n, q);
    }
    keep[i] = boundary ? 1 : 0;
}

// ---- sparse voxel grids: from points, dilation, erosion, hex mesh; voxel cube meshes ------------------------------
// Definitions in DESIGN.md §3.  A voxel is its 64-bit Morton code (morton.cuh); "sorted" is ascending code order.
// The 26 neighbour offsets, x slowest then y then z (the reference's table order without its three repeats):
// o in [0, 26) is cell c = o + (o >= 13) of the 3 x 3 x 3 block, offset (c / 9 - 1, c / 3 % 3 - 1, c % 3 - 1).
__device__ __forceinline__ int svg_axis(int o, int a) {
    const int c = o + (o >= 13 ? 1 : 0);
    return (a == 0 ? c / 9 : a == 1 ? c / 3 % 3 : c % 3) - 1;
}
__device__ __forceinline__ unsigned long long svg_offset(int o) {
    return morton_encode3(svg_axis(o, 0), svg_axis(o, 1), svg_axis(o, 2));
}

// The scaling of the point quantisation and of the hex vertices (host values, passed by value).
struct SvgPlace { double g[3], o[3]; };

// Per point: round((double(p) - o) / g) per axis (each operation rounded in fp64, C round: half away from zero), the
// reference's safe_cast<double, int32_t> (NaN passes it and converts to INT32_MIN, as x86-64 cvttsd2si does), its
// code as the record {code, point}.  *bad counts points with a coordinate outside [INT32_MIN + 1, INT32_MAX - 1].
template <typename T>
__global__ void __launch_bounds__(kThreads) svg_point_codes_kernel(const T* __restrict__ p, long long n, SvgPlace pl,
                                                                   McRec* __restrict__ recs, unsigned long long* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c[3];
    bool out = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double r = round(__ddiv_rn(__dsub_rn((double)p[3 * i + a], pl.o[a]), pl.g[a]));
        out = out || r > 2147483646.0 || r < -2147483647.0;
        c[a] = isnan(r) ? INT_MIN : (int)r;
    }
    if (out) atomicAdd(bad, 1ull);
    McRec rec;
    rec.key[0] = morton_encode3(c[0], c[1], c[2]);
    rec.idx = (unsigned long long)i;
    store_rec(recs + i, rec);
}

// Dilation, one thread per sorted voxel code j (duplicates after the first flag nothing): flag[o n + j] = 1 when
// neighbour q = code + offset o is missing from the grid and this voxel owns it, i.e. no earlier offset o' < o reaches
// q from a voxel of the grid (q - offset o' = code + offset o - offset o' present).  Every missing neighbour is thus
// flagged exactly once, and the flagged codes are already distinct.
__global__ void __launch_bounds__(kThreads) svg_dilate_flag_kernel(const McRec* __restrict__ sorted, long long n,
                                                                   unsigned char* __restrict__ flag) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const unsigned long long code = __ldg(&sorted[j].key[0]);
    const bool first = j == 0 || __ldg(&sorted[j - 1].key[0]) != code;
#pragma unroll 1
    for (int o = 0; o < 26; ++o) {
        bool owned = false;
        if (first && svb_missing(sorted, n, morton_add2(code, svg_offset(o)))) {
            owned = true;
#pragma unroll 1
            for (int e = 0; e < o && owned; ++e) {
                const unsigned long long d = morton_encode3(svg_axis(o, 0) - svg_axis(e, 0), svg_axis(o, 1) - svg_axis(e, 1),
                                                            svg_axis(o, 2) - svg_axis(e, 2));
                owned = svb_missing(sorted, n, morton_add2(code, d));
            }
        }
        flag[o * n + j] = owned ? 1 : 0;
    }
}

// After keep_count / keep_offsets over the 26 n flags: every flagged slot o n + j writes the record {code_j + offset
// o, rank} at its rank.
__global__ void __launch_bounds__(kThreads) svg_dilate_write_kernel(const McRec* __restrict__ sorted, long long n,
                                                                    const unsigned char* __restrict__ flag,
                                                                    const unsigned* __restrict__ block_offset, McRec* __restrict__ recs) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool mine = s < 26 * n && flag[s];
    const unsigned pos = keep_rank(mine, block_offset);
    if (!mine) return;
    const long long o = s / n, j = s - o * n;
    McRec rec;
    rec.key[0] = morton_add2(__ldg(&sorted[j].key[0]), svg_offset((int)o));
    rec.idx = pos;
    store_rec(recs + pos, rec);
}

// Erosion: keep[i] = 1 when all 26 neighbours of voxel i are in the grid.
template <typename I>
__global__ void __launch_bounds__(kThreads) svg_erode_flag_kernel(const I* __restrict__ g, long long n, const McRec* __restrict__ sorted,
                                                                  unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long code = svb_code<I>(g, i);
    bool all = true;
#pragma unroll 1
    for (int o = 0; o < 26 && all; ++o) all = !svb_missing(sorted, n, morton_add2(code, svg_offset(o)));
    keep[i] = all ? 1 : 0;
}

// The kept rows of g, verbatim and in order.
template <typename I>
__global__ void __launch_bounds__(kThreads) svg_keep_voxels_kernel(const I* __restrict__ g, const unsigned char* __restrict__ keep,
                                                                   long long n, const unsigned* __restrict__ block_offset,
                                                                   I* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool mine = i < n && keep[i];
    const unsigned pos = keep_rank(mine, block_offset);
    if (!mine) return;
    out[3ull * pos] = g[3 * i]; out[3ull * pos + 1] = g[3 * i + 1]; out[3ull * pos + 2] = g[3 * i + 2];
}

// Hex mesh: the 8 corner records {code + corner offset, 8 i + k} of voxel i, corners (0,0,0) (1,0,0) (1,1,0) (0,1,0)
// (0,0,1) (1,0,1) (1,1,1) (0,1,1) (marching_cubes_sparse_voxel_grid's order); *bad as in svb_codes_kernel.
template <typename I>
__global__ void __launch_bounds__(kThreads) svg_corners_kernel(const I* __restrict__ g, long long n, McRec* __restrict__ recs,
                                                               unsigned long long* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!svb_fits((long long)g[3 * i]) || !svb_fits((long long)g[3 * i + 1]) || !svb_fits((long long)g[3 * i + 2])) atomicAdd(bad, 1ull);
    const unsigned long long code = svb_code<I>(g, i);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        McRec rec;
        rec.key[0] = morton_add2(code, morton_encode3(((k + 1) >> 1) & 1, (k >> 1) & 1, k >> 2));
        rec.idx = 8ull * i + k;
        store_rec(recs + 8 * i + k, rec);
    }
}

// After keep_count / keep_offsets over the run heads of the sorted records: each head writes its decoded code as row
// rank(head) of out -- integer rows (O = int or long long), or hex vertices (O = float or double):
// ((double)c * g + o) - 0.5 * g per axis, each operation rounded in fp64, then one rounding to O.  head == nullptr:
// every record is a head (codes already distinct), rows in record order.
template <typename O>
__global__ void __launch_bounds__(kThreads) svg_decode_kernel(const McRec* __restrict__ recs, long long n, const unsigned char* __restrict__ head,
                                                              const unsigned* __restrict__ block_offset, SvgPlace pl, O* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool mine = i < n;
    unsigned long long pos = (unsigned long long)i;
    if (head) {
        mine = mine && head[i];
        pos = keep_rank(mine, block_offset);
    }
    if (!mine) return;
    int c[3];
    morton_decode3(recs[i].key[0], c[0], c[1], c[2]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if constexpr (std::is_floating_point<O>::value)
            out[3 * pos + a] = (O)__dsub_rn(__dadd_rn(__dmul_rn((double)c[a], pl.g[a]), pl.o[a]), __dmul_rn(0.5, pl.g[a]));
        else
            out[3 * pos + a] = (O)c[a];
    }
}

// After keep_count / keep_offsets over the run heads: each record's run (distinct codes at or before it, minus one)
// scattered to its index: point_to_vox[point], or cubes[8 i + k].
__global__ void __launch_bounds__(kThreads) svg_rank_kernel(const McRec* __restrict__ recs, long long n, const unsigned char* __restrict__ head,
                                                            const unsigned* __restrict__ block_offset, long long* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned run = keep_rank<true>(i < n && head[i], block_offset) - 1u;
    if (i < n) out[recs[i].idx] = (long long)run;
}

// voxel_grid_geometry (the reference's src/mesh_for_voxels.cpp generate_cube_mesh): thread t writes vertex row t
// (t < 8 n) and face row t (t < 12 n).  Vertex row 8 i + c, component k: float((((tbl_ck * (1 - gap) + 0.5 gap)
// + (double)ijk_ik) * s_k) + o_k), each operation rounded in fp64; face row 12 i + f: the table's face f plus 8 i.
struct VgGeom { double s[3], o[3], keep, shift; };   // keep = 1 - gap, shift = 0.5 gap (as the reference computes them)
__constant__ unsigned char kVgCorner[8] = {4, 5, 6, 7, 0, 1, 2, 3};   // bit 0: x, bit 1: y, bit 2: z of each table corner
__constant__ unsigned char kVgFaces[36] = {2, 7, 6, 2, 3, 7, 0, 4, 5, 0, 5, 1, 0, 2, 6, 0, 6, 4,
                                           1, 7, 3, 1, 5, 7, 0, 3, 2, 0, 1, 3, 4, 6, 7, 4, 7, 5};
template <typename I>
__global__ void __launch_bounds__(kThreads) vg_geometry_kernel(const I* __restrict__ ijk, long long n, VgGeom g, float* __restrict__ out_v,
                                                               int* __restrict__ out_f) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < 8 * n) {
        const long long i = t >> 3;
        const unsigned corner = __ldg(&kVgCorner[t & 7]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double tbl = (double)((corner >> k) & 1u);
            double x = __dadd_rn(__dmul_rn(tbl, g.keep), g.shift);
            x = __dadd_rn(x, (double)ijk[3 * i + k]);
            x = __dadd_rn(__dmul_rn(x, g.s[k]), g.o[k]);
            out_v[3 * t + k] = __double2float_rn(x);
        }
    }
    if (t < 12 * n) {
        const long long i = t / 12, f = t - 12 * i;
#pragma unroll
        for (int k = 0; k < 3; ++k) out_f[3 * t + k] = (int)__ldg(&kVgFaces[3 * f + k]) + (int)(8 * i);
    }
}

}  // namespace pcu
