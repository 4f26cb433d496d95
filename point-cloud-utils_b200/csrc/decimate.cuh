// decimate.cuh -- shortest-edge decimation of a triangle mesh in rounds of independent edge collapses (the reference's
// src/mesh_decimate.cpp, libigl's decimate).  Result defined in DESIGN.md §3.
//
// Vertex ids are the input's throughout; the current faces are int32 rows F[m] (a dead face keeps its last row), the
// live faces a compact list of face ids, the positions fp64.  One round, over the A live faces:
//   dc_records_kernel   six records per live face, {src, dst; opposite} for both directions of its three edges
//   radix sort of the 6 A records (sort.cuh) by (src, dst): the records of one directed edge form a run, and the runs
//                       of a vertex, in ascending dst, are its neighbour list (CSR over the run numbers)
//   dc_heads_kernel, keep_count / keep_offsets (compact.cuh): the run number of every run head
//   dc_runs_kernel      per run: src, dst, its one or two opposite vertices (-1: a boundary edge, whose second face is
//                       the one joined to the virtual vertex), beg / end of src's list, boundary edges per vertex
//   dc_valid_kernel     one thread per undirected edge (the run with src < dst): the link condition by a merge of the
//                       two sorted neighbour lists
//   keep_count / keep_offsets over the valid flags, dc_keys_kernel: the valid edges' {fp64 key bits (two words), run}
//                       in run order, padded to 3 A records with keys that sort last; radix sort by key (stable: ties
//                       in run order, which is (a, b) order)
//   dc_stamp_kernel     candidate p (rank p < K) atomicMins p into the stamp of every vertex of R(e)
//   dc_select_kernel    p is selected when it holds every stamp of R(e); flags 2p (selected) and 2p + 1 (selected
//                       and interior) so that a compaction scan over them counts the faces lower ranks remove
//   keep_count / keep_offsets, dc_apply_kernel: a selected edge is applied while those lower-ranked removals are
//                       below K; b merges into a, x[a] = (x[a] + x[b]) / 2
//   dc_faces_kernel     every live face relabelled through the merge map; it dies when two corners coincide
//   keep_count / keep_offsets, dc_live_kernel: the new live list; the count record is read (the round's one
//                       synchronisation)
// The input check (dc_faces_in_kernel, dc_verts_in_kernel) and the acceptance test of the first round's adjacency
// (dc_accept_kernel) synchronise once each before the rounds; the output (dc_mark_kernel, dc_vrank_kernel,
// dc_fout_kernel) once after them.
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "sort.cuh"

namespace pcu {

// {src, dst; opposite} of the adjacency sort, and {key high word, key low word; run} of the ranking sort.
using DcRec = SortRec<unsigned, 2>;

constexpr long long kDcMaxIds = 0x7fffffffLL - 1;   // vertices and faces: int32 ids, 6 m records below 2^32

// What the device tells the host: input check, acceptance, and the counts of a round (device-side compaction totals).
struct DcCounts {
    unsigned long long bad_corner, non_finite, rejected;
    long long runs, valid, alive, removable, nf_out, nv_out;
    unsigned long long applied, removed;
};

__device__ __forceinline__ long long dc_corner(const void* f, long long i, int kind) {
    switch (kind) {
        case kIdxI32: return ((const int*)f)[i];
        case kIdxI64: return ((const long long*)f)[i];
        case kIdxU32: return (long long)((const unsigned*)f)[i];
        default: {
            const unsigned long long u = ((const unsigned long long*)f)[i];
            return u > (unsigned long long)LLONG_MAX ? -1 : (long long)u;
        }
    }
}

// F (int32 rows), the first live list (every face) and the rejection of faces with a repeated corner.
__global__ void __launch_bounds__(kThreads) dc_faces_in_kernel(const void* __restrict__ f, int fkind, long long m, long long nv, int* __restrict__ F,
                                                               int* __restrict__ live, DcCounts* counts) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    long long c[3];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c[k] = dc_corner(f, 3 * t + k, fkind);
        bad |= c[k] < 0 || c[k] >= nv;
        F[3 * t + k] = (int)c[k];
    }
    if (bad) atomicAdd(&counts->bad_corner, 1ull);
    else if (c[0] == c[1] || c[1] == c[2] || c[0] == c[2]) atomicAdd(&counts->rejected, 1ull);
    live[t] = (int)t;
}

// Positions widened to fp64, the identity merge map.
template <typename T>
__global__ void __launch_bounds__(kThreads) dc_verts_in_kernel(const T* __restrict__ v, long long nv, double* __restrict__ x, int* __restrict__ map,
                                                               DcCounts* counts) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= nv) return;
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double d = (double)v[3 * i + k];
        bad |= !isfinite(d);
        x[3 * i + k] = d;
    }
    if (bad) atomicAdd(&counts->non_finite, 1ull);
    map[i] = (int)i;
}

// Corner k is opposite the edge from corner (k + 1) % 3 to corner (k + 2) % 3.
__global__ void __launch_bounds__(kThreads) dc_records_kernel(const int* __restrict__ F, const int* __restrict__ live, long long A, DcRec* __restrict__ rec) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= A) return;
    const long long t = live[i];
    const int c[3] = {F[3 * t], F[3 * t + 1], F[3 * t + 2]};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned u = (unsigned)c[(k + 1) % 3], w = (unsigned)c[(k + 2) % 3], o = (unsigned)c[k];
        DcRec r;
        r.key[0] = u; r.key[1] = w; r.idx = o;
        store_rec(rec + 6 * i + 2 * k, r);
        r.key[0] = w; r.key[1] = u;
        store_rec(rec + 6 * i + 2 * k + 1, r);
    }
}

__device__ __forceinline__ bool dc_same(const DcRec& a, const DcRec& b) { return a.key[0] == b.key[0] && a.key[1] == b.key[1]; }

__global__ void __launch_bounds__(kThreads) dc_heads_kernel(const DcRec* __restrict__ rec, long long n, unsigned char* __restrict__ head) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    head[i] = i == 0 || !dc_same(load_rec(rec + i - 1), load_rec(rec + i));
}

// The runs: rs / rd / o0 / o1 per run number, beg / end of every vertex's runs, nb = boundary edges per vertex (zeroed
// before).  A run of more than two records (an edge in three or more faces) is counted as a rejection.
__global__ void __launch_bounds__(kThreads) dc_runs_kernel(const DcRec* __restrict__ rec, long long n, const unsigned char* __restrict__ head,
                                                           const unsigned* __restrict__ offsets, int* __restrict__ rs, int* __restrict__ rd,
                                                           int* __restrict__ o0, int* __restrict__ o1, int* __restrict__ beg, int* __restrict__ end,
                                                           int* __restrict__ nb, DcCounts* counts) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < n && head[i];
    const unsigned j = keep_rank(mine, offsets);
    if (!mine) return;
    const DcRec r = load_rec(rec + i);
    long long q = i + 1;
    int second = -1;
    for (; q < n; ++q) {
        const DcRec s = load_rec(rec + q);
        if (!dc_same(s, r)) break;
        if (q == i + 1) second = (int)s.idx;
    }
    if (q - i > 2) atomicAdd(&counts->rejected, 1ull);
    const int src = (int)r.key[0];
    rs[j] = src;
    rd[j] = (int)r.key[1];
    o0[j] = (int)r.idx;
    o1[j] = second;
    if (i == 0 || load_rec(rec + i - 1).key[0] != r.key[0]) beg[src] = (int)j;
    if (q == n || load_rec(rec + q).key[0] != r.key[0]) end[src] = (int)j + 1;
    if (second < 0) atomicAdd(nb + src, 1);
}

// The first round's adjacency: every vertex has zero or two boundary edges.
__global__ void __launch_bounds__(kThreads) dc_accept_kernel(const int* __restrict__ nb, long long nv, DcCounts* counts) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i < nv && nb[i] != 0 && nb[i] != 2) atomicAdd(&counts->rejected, 1ull);
}

// fl(fl(fl(dx^2) + fl(dy^2)) + fl(dz^2)), dx = x[a] - x[b]
__device__ __forceinline__ double dc_key(const double* __restrict__ x, int a, int b) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double d = __dsub_rn(x[3 * a + k], x[3 * b + k]);
        s = k == 0 ? __dmul_rn(d, d) : __dadd_rn(s, __dmul_rn(d, d));
    }
    return s;
}

// Whether run w (a's run to some c) has opposite d.
__device__ __forceinline__ bool dc_has_opp(const int* __restrict__ o0, const int* __restrict__ o1, int w, int d) {
    return o0[w] == d || o1[w] == d;
}

// The link condition of DESIGN.md §3 for the undirected edge of run j (src < dst); flag[j] = valid, and 0 for every
// slot past the runs.
__global__ void __launch_bounds__(kThreads) dc_valid_kernel(long long n, const DcCounts* __restrict__ counts, const int* __restrict__ rs,
                                                            const int* __restrict__ rd, const int* __restrict__ o0, const int* __restrict__ o1,
                                                            const int* __restrict__ beg, const int* __restrict__ end, const int* __restrict__ nb,
                                                            unsigned char* __restrict__ flag) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j >= n) return;
    bool ok = false;
    if (j < counts->runs && rs[j] < rd[j]) {
        const int a = rs[j], b = rd[j], c = o0[j], d = o1[j];
        const bool interior = d >= 0;
        ok = interior ? c != d && !(nb[a] > 0 && nb[b] > 0) : true;
        int common = 0;
        for (int p = beg[a], q = beg[b], pe = end[a], qe = end[b]; ok && p < pe && q < qe;) {
            const int u = rd[p], w = rd[q];
            if (u < w) { ++p; continue; }
            if (w < u) { ++q; continue; }
            ++common;
            if (u == c) {   // interior: faces (a, c, d) and (b, c, d) both present; boundary: (a, c) and (b, c) both boundary
                ok = interior ? !(dc_has_opp(o0, o1, p, d) && dc_has_opp(o0, o1, q, d)) : !(o1[p] < 0 && o1[q] < 0);
            }
            ++p; ++q;
        }
        ok = ok && common == (interior ? 2 : 1);
    }
    flag[j] = ok;
}

// The valid edges' ranking records in run order at positions [0, V), and records that sort after every key at [V, P).
__global__ void __launch_bounds__(kThreads) dc_keys_kernel(long long n, long long P, const unsigned char* __restrict__ flag,
                                                           const unsigned* __restrict__ offsets, const DcCounts* __restrict__ counts,
                                                           const int* __restrict__ rs, const int* __restrict__ rd, const double* __restrict__ x,
                                                           DcRec* __restrict__ out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < n && flag[i];
    const unsigned p = keep_rank(mine, offsets);
    DcRec r;
    if (mine) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(dc_key(x, rs[i], rd[i]));
        r.key[0] = (unsigned)(bits >> 32); r.key[1] = (unsigned)bits; r.idx = (unsigned)i;
        store_rec(out + p, r);
    }
    if (i >= counts->valid && i < P) {
        r.key[0] = r.key[1] = r.idx = 0xffffffffu;
        store_rec(out + i, r);
    }
}

// Candidate p: every vertex of R(e) = {a, b} + N(a) + N(b) (the virtual vertex left out) takes the lowest rank.
__global__ void __launch_bounds__(kThreads) dc_stamp_kernel(long long P, const DcRec* __restrict__ ranked, const DcCounts* __restrict__ counts,
                                                            const int* __restrict__ rs, const int* __restrict__ rd, const int* __restrict__ beg,
                                                            const int* __restrict__ end, unsigned* __restrict__ stamp) {
    const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (p >= P || p >= counts->valid) return;
    const unsigned j = load_rec(ranked + p).idx, r = (unsigned)p;
    const int a = rs[j], b = rd[j];
    atomicMin(stamp + a, r);
    atomicMin(stamp + b, r);
    for (int q = beg[a]; q < end[a]; ++q) atomicMin(stamp + rd[q], r);
    for (int q = beg[b]; q < end[b]; ++q) atomicMin(stamp + rd[q], r);
}

__global__ void __launch_bounds__(kThreads) dc_select_kernel(long long P, const DcRec* __restrict__ ranked, const DcCounts* __restrict__ counts,
                                                             const int* __restrict__ rs, const int* __restrict__ rd, const int* __restrict__ o1,
                                                             const int* __restrict__ beg, const int* __restrict__ end,
                                                             const unsigned* __restrict__ stamp, unsigned char* __restrict__ rem) {
    const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (p >= P) return;
    bool sel = false, interior = false;
    if (p < counts->valid) {
        const unsigned j = load_rec(ranked + p).idx, r = (unsigned)p;
        const int a = rs[j], b = rd[j];
        sel = stamp[a] == r && stamp[b] == r;
        for (int q = beg[a]; sel && q < end[a]; ++q) sel = stamp[rd[q]] == r;
        for (int q = beg[b]; sel && q < end[b]; ++q) sel = stamp[rd[q]] == r;
        interior = o1[j] >= 0;
    }
    rem[2 * p] = sel;
    rem[2 * p + 1] = sel && interior;
}

// Thread 2p's exclusive rank over the removal flags is the number of faces the selected edges of lower rank remove.
__global__ void __launch_bounds__(kThreads) dc_apply_kernel(long long n2, long long K, const unsigned char* __restrict__ rem,
                                                            const unsigned* __restrict__ offsets, const DcRec* __restrict__ ranked,
                                                            const int* __restrict__ rs, const int* __restrict__ rd, double* __restrict__ x,
                                                            int* __restrict__ map, DcCounts* counts) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < n2 && rem[i];
    const unsigned before = keep_rank(mine, offsets);
    if (!mine || (i & 1) || (long long)before >= K) return;
    const unsigned j = load_rec(ranked + i / 2).idx;
    const int a = rs[j], b = rd[j];
    map[b] = a;
#pragma unroll
    for (int k = 0; k < 3; ++k) x[3 * a + k] = __dmul_rn(__dadd_rn(x[3 * a + k], x[3 * b + k]), 0.5);
    atomicAdd(&counts->applied, 1ull);
    atomicAdd(&counts->removed, rem[i + 1] ? 2ull : 1ull);
}

__global__ void __launch_bounds__(kThreads) dc_faces_kernel(int* __restrict__ F, const int* __restrict__ live, long long A, const int* __restrict__ map,
                                                            unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= A) return;
    const long long t = live[i];
    int c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c[k] = map[F[3 * t + k]];
        F[3 * t + k] = c[k];
    }
    keep[i] = c[0] != c[1] && c[1] != c[2] && c[0] != c[2];
}

__global__ void __launch_bounds__(kThreads) dc_live_kernel(const int* __restrict__ live, long long A, const unsigned char* __restrict__ keep,
                                                           const unsigned* __restrict__ offsets, int* __restrict__ out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < A && keep[i];
    const unsigned r = keep_rank(mine, offsets);
    if (mine) out[r] = live[i];
}

// The output's flags: alive[t] per input face, used[v] per vertex a live face references (both zeroed before).
__global__ void __launch_bounds__(kThreads) dc_mark_kernel(const int* __restrict__ F, const int* __restrict__ live, long long A,
                                                           unsigned char* __restrict__ alive, unsigned char* __restrict__ used) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= A) return;
    const long long t = live[i];
    alive[t] = 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) used[F[3 * t + k]] = 1;
}

// Vertex r of the output is the r-th used vertex: its id, its position, and the new label of that id.
__global__ void __launch_bounds__(kThreads) dc_vrank_kernel(long long nv, const unsigned char* __restrict__ used, const unsigned* __restrict__ offsets,
                                                            const double* __restrict__ x, int* __restrict__ label, int* __restrict__ vcorr,
                                                            double* __restrict__ xo) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < nv && used[i];
    const unsigned r = keep_rank(mine, offsets);
    if (!mine) return;
    label[i] = (int)r;
    vcorr[r] = (int)i;
#pragma unroll
    for (int k = 0; k < 3; ++k) xo[3 * (long long)r + k] = x[3 * i + k];
}

__global__ void __launch_bounds__(kThreads) dc_fout_kernel(long long m, const unsigned char* __restrict__ alive, const unsigned* __restrict__ offsets,
                                                           const int* __restrict__ F, const int* __restrict__ label, int* __restrict__ fcorr,
                                                           int* __restrict__ fo) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = t < m && alive[t];
    const unsigned r = keep_rank(mine, offsets);
    if (!mine) return;
    fcorr[r] = (int)t;
#pragma unroll
    for (int k = 0; k < 3; ++k) fo[3 * (long long)r + k] = label[F[3 * t + k]];
}

__device__ __forceinline__ void dc_put_index(void* out, long long i, int v, int wide) {
    if (wide) ((long long*)out)[i] = v;
    else ((int*)out)[i] = v;
}

// The result in the input's types: v_out rounded to T, f_out and the correspondences in f's width.
template <typename T>
__global__ void __launch_bounds__(kThreads) dc_emit_kernel(const double* __restrict__ xo, long long nvo, const int* __restrict__ fo,
                                                           const int* __restrict__ vcorr, const int* __restrict__ fcorr, long long nfo, int wide,
                                                           T* __restrict__ out_v, void* __restrict__ out_f, void* __restrict__ out_vc,
                                                           void* __restrict__ out_fc) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i < 3 * nvo) out_v[i] = (T)xo[i];
    if (i < 3 * nfo) dc_put_index(out_f, i, fo[i], wide);
    if (i < nvo) dc_put_index(out_vc, i, vcorr[i], wide);
    if (i < nfo) dc_put_index(out_fc, i, fcorr[i], wide);
}

}  // namespace pcu
