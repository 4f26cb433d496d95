// mesh_topology.cuh -- connected components of a mesh and vertex removal (the reference's src/connected_components.cpp,
// src/remove_mesh_vertices.cpp and src/remove_unreferenced_mesh_vertices.cpp).  Results defined in DESIGN.md §3.
//
// connected_components: the graph has the vertices [0, n), n = max(f) + 1, and joins corner j to corner j + 1 of every
// face row (the same components as libigl's adjacency_matrix, which joins every pair of corners of a row).
//   cc_validate_kernel  persistent CTAs over the m c entries of f: max(f) and the entries outside [0, 2^31 - 2]
//   (the host reads them: first synchronisation; n sizes the buffers)
//   cc_init_kernel      P[v] = v
//   cc_hook_kernel      one thread per face row: uf_union of consecutive corners (union_find.cuh), so every root is
//                       the smallest vertex of its component
//   cc_flatten_kernel   root[v] = root of v; root flags
//   keep_count / keep_offsets over the flags (compact.cuh): the component count
//   cc_rank_kernel      rank[r] = number of roots below r: component j is the j-th in ascending order of its smallest
//                       vertex, the order in which the reference's outer loop starts its BFS runs
//   cc_label_kernel     cv[v] = rank[root[v]] (in place, in root), nv counted
//   cc_face_kernel      cf[i] = cv[f[i, 0]], nf counted
//   (the host reads the component count: second synchronisation), then cc_emit_kernel writes the four outputs in f's
//   width.
// The counts are warp-aggregated: the lanes of a warp that share a label add once, so a one-component mesh does not
// send every atomic to one address.
//
// remove_mesh_vertices / remove_unreferenced_mesh_vertices: order-preserving compactions (compact.cuh) of the kept
// vertices and, for the mask, of the kept faces; one synchronisation each, to read MtCounts.
//
// adjacency_list (the reference's src/adjacency_list.cpp, libigl's adjacency_list): the Laplacian's sparsity pattern
// (laplacian.cuh) over the rows [0, n), n = max(f) + 1, in CSR form:
//   cc_validate_kernel  max(f) and the entries outside [0, 2^31 - 2] (the host reads them: first synchronisation)
//   lap_edge_kernel     six directed-edge records per face, key (row << bits) | column, with nv = n
//   radix sort (sort.cuh), mc_heads_kernel (runtime.cu), keep_count / keep_offsets (compact.cuh): one entry per
//                       distinct (row, column) pair, ascending; the host reads their count nnz (second synchronisation)
//   adj_entries_kernel  entry e of every run: its column into the handle, its row as the key of mg_rows_kernel
//   mg_rows_kernel      (mesh_geometry.cuh) the row pointers: row i holds entries [rowptr[i], rowptr[i + 1])
//   adj_emit_kernel     both arrays in f's width.
// A face with a repeated corner gives the pair (a, a) and so a self-loop, as in libigl.
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "meshsample.cuh"
#include "mesh_geometry.cuh"
#include "union_find.cuh"

namespace pcu {

constexpr long long kCcMaxIndex = 0x7ffffffeLL;   // largest vertex index: parents stay int32, n <= 2^31 - 1

// What the host reads from connected_components (zeroed per call).
struct CcCounts {
    unsigned long long bad;   // entries of f outside [0, kCcMaxIndex]
    unsigned max_index;       // max(f) over the other entries
    unsigned pad;
    long long ncomp;          // components (keep_offsets_kernel)
};

// What the host reads from adjacency_list (zeroed per call).
struct AdjCounts {
    CcCounts valid;           // cc_validate_kernel's bad entries and max(f)
    long long nnz;            // distinct (row, column) pairs (keep_offsets_kernel)
};

// What the host reads from a vertex removal (zeroed per call).
struct MtCounts {
    long long kept_v;          // kept vertices (keep_offsets_kernel)
    long long kept_f;          // kept faces (remove_mesh_vertices)
    unsigned long long bad;    // faces with a corner outside [0, #v)
};

__global__ void __launch_bounds__(kThreads) cc_validate_kernel(const void* __restrict__ f, int fkind, long long total,
                                                               CcCounts* __restrict__ counts) {
    unsigned mx = 0u, bad = 0u;
    for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
        const long long x = load_index(f, e, fkind, kCcMaxIndex + 1, false);
        if (x < 0) ++bad;
        else mx = max(mx, (unsigned)x);
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
        if (mx) atomicMax(&counts->max_index, mx);
        if (bad) atomicAdd(&counts->bad, (unsigned long long)bad);
    }
}

__global__ void __launch_bounds__(kThreads) cc_init_kernel(int* __restrict__ P, long long n) {
    const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (v < n) P[v] = (int)v;
}

// Entries are valid (cc_validate_kernel) when this runs.
__global__ void __launch_bounds__(kThreads) cc_hook_kernel(const void* __restrict__ f, int fkind, long long m, int c, int* P) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    int a = (int)load_index(f, t * c, fkind, kCcMaxIndex + 1, false);
    for (int j = 1; j < c; ++j) {
        const int b = (int)load_index(f, t * c + j, fkind, kCcMaxIndex + 1, false);
        uf_union(P, a, b);
        a = b;
    }
}

// The roots go to their own array: P itself cannot hold them, because a concurrent uf_find may still store an
// ancestor that is not the root over P[v] after v's thread has stored the root there.
__global__ void __launch_bounds__(kThreads) cc_flatten_kernel(int* P, long long n, int* __restrict__ root, unsigned char* __restrict__ is_root) {
    const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (v >= n) return;
    const int r = uf_find(P, (int)v);
    root[v] = r;
    is_root[v] = r == (int)v;
}

__global__ void __launch_bounds__(kThreads) cc_rank_kernel(const unsigned char* __restrict__ is_root, long long n,
                                                           const unsigned* __restrict__ block_offset, int* __restrict__ rank) {
    const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = v < n && is_root[v];
    const unsigned pos = keep_rank(mine, block_offset);
    if (mine) rank[v] = (int)pos;
}

// counts[label] += 1 for the lanes with `in`, one atomic per distinct label of the warp.  Every lane of the warp calls it.
__device__ __forceinline__ void cc_count(bool in, int label, int* __restrict__ counts) {
    const unsigned peers = __match_any_sync(0xffffffffu, in ? label : -1);
    if (in && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&counts[label], __popc(peers));
}

// cv[v] = rank[root[v]], written over root[v] (each thread reads and writes its own entry only).
__global__ void __launch_bounds__(kThreads) cc_label_kernel(int* __restrict__ root, long long n, const int* __restrict__ rank,
                                                            int* __restrict__ nv) {
    const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool in = v < n;
    const int label = in ? __ldg(rank + root[v]) : 0;
    if (in) root[v] = label;
    cc_count(in, label, nv);
}

__global__ void __launch_bounds__(kThreads) cc_face_kernel(const void* __restrict__ f, int fkind, long long m, int c,
                                                           const int* __restrict__ cv, int* __restrict__ cf, int* __restrict__ nf) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool in = t < m;
    const int label = in ? __ldg(cv + load_index(f, t * c, fkind, kCcMaxIndex + 1, false)) : 0;
    if (in) cf[t] = label;
    cc_count(in, label, nf);
}

// The four results in f's width I (values are non-negative, so the unsigned kinds share the signed ones' bits).
template <typename I>
__global__ void __launch_bounds__(kThreads) cc_emit_kernel(const int* __restrict__ cv, long long n, const int* __restrict__ cf, long long m,
                                                           const int* __restrict__ nv, const int* __restrict__ nf, long long k,
                                                           I* __restrict__ out_cv, I* __restrict__ out_cf, I* __restrict__ out_nv,
                                                           I* __restrict__ out_nf) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) out_cv[i] = (I)cv[i];
    if (i < m) out_cf[i] = (I)cf[i];
    if (i < k) { out_nv[i] = (I)nv[i]; out_nf[i] = (I)nf[i]; }
}

// ---- adjacency_list -----------------------------------------------------------------------------------------------
// After keep_count / keep_offsets over the run heads of the sorted directed-edge records: entry e of every run, its row
// (for mg_rows_kernel's key) and its column.
__global__ void __launch_bounds__(kThreads) adj_entries_kernel(const MgRec* __restrict__ sorted, long long n, const unsigned char* __restrict__ head,
                                                               const unsigned* __restrict__ block_offset, int bits, MgRec* __restrict__ rows,
                                                               int* __restrict__ col) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < n && head[i];
    const unsigned e = keep_rank(mine, block_offset);
    if (!mine) return;
    const unsigned long long key = sorted[i].key[0];
    MgRec r;
    r.key[0] = key >> bits;
    r.idx = e;
    store_rec(rows + e, r);
    col[e] = (int)(key & ((1ull << bits) - 1ull));
}

// The n + 1 row pointers and the nnz columns in f's width I.
template <typename I>
__global__ void __launch_bounds__(kThreads) adj_emit_kernel(const int* __restrict__ rowptr, long long n, const int* __restrict__ col,
                                                            long long nnz, I* __restrict__ out_offsets, I* __restrict__ out_neighbors) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i <= n) out_offsets[i] = (I)rowptr[i];
    if (i < nnz) out_neighbors[i] = (I)col[i];
}

// ---- remove_mesh_vertices -----------------------------------------------------------------------------------------
// After keep_count / keep_offsets over the mask: the kept vertices to out_v in input order, and remap[i] = the new
// index of vertex i, or -1.
template <typename T>
__global__ void __launch_bounds__(kThreads) rmv_vertex_kernel(const T* __restrict__ v, long long nv, const unsigned char* __restrict__ mask,
                                                              const unsigned* __restrict__ block_offset, T* __restrict__ out_v,
                                                              int* __restrict__ remap) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < nv && mask[i] != 0;
    const unsigned pos = keep_rank(mine, block_offset);
    if (i >= nv) return;
    remap[i] = mine ? (int)pos : -1;
    if (mine) {
#pragma unroll
        for (int k = 0; k < 3; ++k) out_v[3ull * pos + k] = v[3 * i + k];
    }
}

// A face is kept when its three corners are; faces with a corner outside [0, nv) are counted (and not kept).
__global__ void __launch_bounds__(kThreads) rmv_face_flag_kernel(const void* __restrict__ f, int fkind, long long m, long long nv,
                                                                 const int* __restrict__ remap, unsigned char* __restrict__ keep,
                                                                 MtCounts* __restrict__ counts) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool bad = false, kept = false;
    if (t < m) {
        kept = true;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const long long x = load_index(f, 3 * t + k, fkind, nv, false);
            if (x < 0) bad = true;
            else kept = kept && __ldg(remap + x) >= 0;
        }
        kept = kept && !bad;
        keep[t] = kept;
    }
    const int nbad = __syncthreads_count(bad);
    if (threadIdx.x == 0 && nbad) atomicAdd(&counts->bad, (unsigned long long)nbad);
}

// After keep_count / keep_offsets over the face flags: the kept faces, re-indexed, in input order, in f's width I.
template <typename I>
__global__ void __launch_bounds__(kThreads) rmv_face_emit_kernel(const void* __restrict__ f, int fkind, long long m, long long nv,
                                                                 const unsigned char* __restrict__ keep, const unsigned* __restrict__ block_offset,
                                                                 const int* __restrict__ remap, I* __restrict__ out_f) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = t < m && keep[t];
    const unsigned pos = keep_rank(mine, block_offset);
    if (!mine) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) out_f[3ull * pos + k] = (I)__ldg(remap + load_index(f, 3 * t + k, fkind, nv, false));
}

// ---- remove_unreferenced_mesh_vertices ----------------------------------------------------------------------------
// used[x] = 1 for every corner x (flags zeroed before); faces with a corner outside [0, nv) are counted.
__global__ void __launch_bounds__(kThreads) rur_mark_kernel(const void* __restrict__ f, int fkind, long long m, long long nv,
                                                            unsigned char* __restrict__ used, MtCounts* __restrict__ counts) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool bad = false;
    if (t < m) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const long long x = load_index(f, 3 * t + k, fkind, nv, false);
            if (x < 0) bad = true;
            else used[x] = 1;
        }
    }
    const int nbad = __syncthreads_count(bad);
    if (threadIdx.x == 0 && nbad) atomicAdd(&counts->bad, (unsigned long long)nbad);
}

// After keep_count / keep_offsets over the flags: v_out = v[J], J = the referenced vertices in input order, and
// I[i] = the new index of vertex i, or -1 (all ones for the unsigned kinds), all in f's width I.
template <typename T, typename I>
__global__ void __launch_bounds__(kThreads) rur_vertex_kernel(const T* __restrict__ v, long long nv, const unsigned char* __restrict__ used,
                                                              const unsigned* __restrict__ block_offset, T* __restrict__ out_v,
                                                              I* __restrict__ out_j, I* __restrict__ out_i) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < nv && used[i];
    const unsigned pos = keep_rank(mine, block_offset);
    if (i >= nv) return;
    out_i[i] = mine ? (I)pos : (I)-1;
    if (mine) {
        out_j[pos] = (I)i;
#pragma unroll
        for (int k = 0; k < 3; ++k) out_v[3ull * pos + k] = v[3 * i + k];
    }
}

// f_out = I[f], one thread per entry (an entry outside [0, nv) writes -1; the call fails then).
template <typename I>
__global__ void __launch_bounds__(kThreads) rur_face_kernel(const void* __restrict__ f, int fkind, long long entries, long long nv,
                                                            const I* __restrict__ out_i, I* __restrict__ out_f) {
    const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (e >= entries) return;
    const long long x = load_index(f, e, fkind, nv, false);
    out_f[e] = x >= 0 ? out_i[x] : (I)-1;
}

}  // namespace pcu
