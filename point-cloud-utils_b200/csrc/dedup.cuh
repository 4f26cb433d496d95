// dedup.cuh -- removal of duplicated points / mesh vertices (SURVEY.md 8f, row N2, second half).
//
// Replaces deduplicate_point_cloud and deduplicate_mesh_vertices (src/remove_duplicates.cpp:108-176, the helpers
// :11-79).  The reference calls libigl (fetched at build time, not in the tree):
//     epsilon > 0 :  rV = igl::round(V / epsilon);  igl::unique_rows(rV, rSV, SVI, SVJ);  SV = V(SVI, :)
//     otherwise   :  igl::unique_rows(V, SV, SVI, SVJ)
// igl::unique_rows sorts the rows lexicographically (igl::sortrows, ascending), keeps one row per run of equal
// rows, and returns  SVI: for every unique row the index of an input row equal to it,  SVJ: for every input row the
// unique row it maps to.  The division happens in the cloud's precision (Eigen narrows the double epsilon to the
// matrix scalar), igl::round is std::round (halves away from zero).
//
// Exact here: the set and the ORDER of the unique rows, SVJ, the number of rows.  Stated difference: igl::sortrows is
// a std::sort of row indices (not stable), so WHICH of several equal rows the reference reports in SVI depends on its
// introsort; here it is always the first (smallest index), which is what a stable sort gives -- and therefore, for
// epsilon > 0, SV = V(SVI, :) is the first point of every cluster.  Every property the reference's own tests check
// (tests/test_examples.py:509-531: SV[SVJ] == V, V[SVI] == SV) holds either way.
//
// Pipeline: keys (order-preserving integer image of the rounded coordinates) -> radix sort (sort.cuh) -> run heads
// -> ordered compaction (compact.cuh) -> emit.
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "sort.cuh"

namespace pcu {

template <typename T> struct DedupRec;
template <> struct DedupRec<float> { using type = SortRec<uint32_t, 3>; };
template <> struct DedupRec<double> { using type = SortRec<unsigned long long, 3>; };

template <typename T> __device__ __forceinline__ T round_half_away(T v);
template <> __device__ __forceinline__ float round_half_away<float>(float v) { return roundf(v); }
template <> __device__ __forceinline__ double round_half_away<double>(double v) { return round(v); }
template <typename T> __device__ __forceinline__ T div_rn(T a, T b);
template <> __device__ __forceinline__ float div_rn<float>(float a, float b) { return __fdiv_rn(a, b); }
template <> __device__ __forceinline__ double div_rn<double>(double a, double b) { return __ddiv_rn(a, b); }

// eps > 0: key of round(p / eps), else of p.  -0 and +0 compare equal in the reference: both map to +0's key.
template <typename T>
__global__ void __launch_bounds__(kThreads) dedup_keys_kernel(const T* __restrict__ pts, long long n, T eps,
                                                              typename DedupRec<T>::type* __restrict__ recs) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typename DedupRec<T>::type r;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        T v = pts[3 * i + a];
        if (eps > (T)0) v = round_half_away<T>(div_rn<T>(v, eps));
        if (v == (T)0) v = (T)0;
        r.key[a] = ordered<T>(v);
    }
    r.idx = (typename Real<T>::bits_t)i;
    store_rec(recs + i, r);
}

// head[i] = 1 when sorted record i starts a run of equal keys
template <typename Rec>
__global__ void __launch_bounds__(kThreads) dedup_heads_kernel(const Rec* __restrict__ recs, long long n, unsigned char* __restrict__ head) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool h = i == 0;
    if (!h) {
        const Rec a = load_rec<Rec>(recs + i - 1), b = load_rec<Rec>(recs + i);
        h = a.key[0] != b.key[0] || a.key[1] != b.key[1] || a.key[2] != b.key[2];
    }
    head[i] = h ? 1 : 0;
}

// After keep_count / keep_offsets over `head`: unique id of every sorted record = heads at or before it, minus one.
//   svj[row] = unique id;  for heads: svi[unique id] = row (the smallest row of the run: the sort is stable) and
//   out_pts[unique id] = pts[row].
template <typename T, typename Rec>
__global__ void __launch_bounds__(kThreads) dedup_emit_kernel(const Rec* __restrict__ recs, long long n, const unsigned char* __restrict__ head,
                                                              const unsigned* __restrict__ block_offset, const T* __restrict__ pts,
                                                              T* __restrict__ out_pts, int* __restrict__ svi, int* __restrict__ svj) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? head[i] : 0u;
    const unsigned uid = keep_rank<true>(mine, block_offset) - 1u;   // heads up to and including this row
    if (i >= n) return;
    const long long row = (long long)recs[i].idx;
    svj[row] = (int)uid;
    if (mine) {
        svi[uid] = (int)row;
        out_pts[3ll * uid] = pts[3 * row];
        out_pts[3ll * uid + 1] = pts[3 * row + 1];
        out_pts[3ll * uid + 2] = pts[3 * row + 2];
    }
}

// Faces after the vertices were merged (src/remove_duplicates.cpp:58-77): a face is dropped when two of its
// corners map to the same unique vertex; the others are re-indexed, in their original order.
// keep[f] = 1 when face f survives; *bad counts faces with a corner outside [0, nv) (dropped; the host raises).
template <typename I>
__global__ void __launch_bounds__(kThreads) dedup_faces_flag_kernel(const I* __restrict__ faces, long long nf, int cols, long long nv,
                                                                    const int* __restrict__ svj, unsigned char* __restrict__ keep,
                                                                    unsigned* __restrict__ bad) {
    const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nf) return;
    bool ok = true;
    for (int c = 0; c < cols && ok; ++c) {
        const long long v = (long long)faces[f * cols + c];
        if (v < 0 || v >= nv) { ok = false; atomicAdd(bad, 1u); }
    }
    for (int c = 0; c < cols && ok; ++c)
        for (int c2 = c + 1; c2 < cols && ok; ++c2)
            if (svj[faces[f * cols + c]] == svj[faces[f * cols + c2]]) ok = false;
    keep[f] = ok ? 1 : 0;
}

template <typename I>
__global__ void __launch_bounds__(kThreads) dedup_faces_emit_kernel(const I* __restrict__ faces, long long nf, int cols,
                                                                    const int* __restrict__ svj, const unsigned char* __restrict__ keep,
                                                                    const unsigned* __restrict__ block_offset, I* __restrict__ out_faces) {
    const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = f < nf ? keep[f] : 0u;
    const unsigned dst = keep_rank(mine, block_offset);
    if (!mine) return;
    for (int c = 0; c < cols; ++c) out_faces[(size_t)dst * cols + c] = (I)svj[faces[f * cols + c]];
}

}  // namespace pcu
