// orient.cuh -- consistent face orientation of a triangle mesh (the reference's src/orient_mesh_faces.cpp, libigl's
// bfs_orient over orientable_patches).  Result defined in DESIGN.md §3.
//
// Faces f and g are adjacent when they share an undirected edge that no third face has.  A pair is regular when its
// edge holds exactly two half-edges, one of each face, both faces have three distinct vertex ids and their opposite
// vertices differ: then bfs_orient's effect on it is a parity (g is flipped exactly when f and g traverse the edge in
// the same direction), whichever face it pops first.  Every patch made of regular pairs that is orientable comes out
// consistent with its smallest face, so it is answered by a union-find over doubled nodes f+ = 2f, f- = 2f + 1; the
// other ("collapsed") patches are replayed literally.
//   om_records_kernel   one thread per face: the records of its three half-edges {key = (min, max) of the endpoints'
//                       order-preserving unsigned images, payload = half-edge id e = k m + f}, P[2f] = 2f, P[2f+1] = 2f+1;
//                       32-bit words for the 32-bit kinds (16-byte records), 64-bit words for the others (32-byte ones)
//   radix sort of the 3 m records (sort.cuh): the half-edges of one undirected edge form a run of equal keys
//   om_runs_kernel      the thread at the head of each run counts its distinct faces (it reads at most 7 records: a
//                       run of at most two faces holds at most six half-edges).  A pair writes the neighbour slot of
//                       each of its half-edges and unites its doubled nodes (union_find.cuh): (f+, g+), (f-, g-) for a
//                       regular pair traversed in opposite directions, (f+, g-), (f-, g+) for one traversed in the same
//                       direction, all four for an irregular pair.  Every root is the smallest node of its tree, so
//                       r = find(2f) gives the patch's smallest face s = r >> 1 and the flip r & 1, and the patch is
//                       collapsed exactly when find(2s + 1) = 2s (non-orientable, or holding an irregular pair).
//   om_flatten_kernel   root[f] = find(2f); flag[f] = kOmSeed for a patch's smallest face, kOmCollapsedSeed for that
//                       of a collapsed patch
//   keep_count / keep_offsets over the flags (compact.cuh), cc_rank_kernel (mesh_topology.cuh): patch j is the j-th in
//                       ascending order of its smallest face
//   om_emit_kernel      the rows, reversed where flipped (never in a collapsed patch), and the patch ids in f's width
//   om_replay_kernel    one thread per collapsed patch: bfs_orient over the neighbour slots, in place on the emitted
//                       rows, with a linked-list queue that drops repeat pushes (the pops keep their order)
// Every buffer is sized by m: nothing is read back, and the host is never synchronised.
#pragma once
#include "common.cuh"
#include "meshsample.cuh"
#include "sort.cuh"
#include "union_find.cuh"

namespace pcu {

constexpr long long kOmMaxFaces = (1ll << 30) - 1;   // 2 m union-find nodes stay int32, 3 m records fit the sort's 32-bit positions
constexpr unsigned char kOmSeed = 1, kOmCollapsedSeed = 3;

// Records of the half-edge sort: key words (min, max) and the half-edge id, all of K = unsigned for the 32-bit kinds
// (3 m < 2^32 ids fit) and unsigned long long for the 64-bit ones.
template <typename K>
using OmRec = SortRec<K, 2>;

// Entry i of f as an order-preserving unsigned image (the sign bit flipped for the signed kinds; below 2^32 for the
// 32-bit kinds).  Only equality of images is used: bfs_orient compares vertex ids and never indexes with them, so every
// value is legal.
__device__ __forceinline__ unsigned long long om_id(const void* f, long long i, int kind) {
    switch (kind) {
        case kIdxI32: return (unsigned)((const int*)f)[i] ^ 0x80000000u;
        case kIdxI64: return ((const unsigned long long*)f)[i] ^ (1ull << 63);
        case kIdxU32: return ((const unsigned*)f)[i];
        default: return ((const unsigned long long*)f)[i];
    }
}

__device__ __forceinline__ void om_row(const void* f, long long t, int kind, unsigned long long r[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = om_id(f, 3 * t + k, kind);
}

template <typename K>
__device__ __forceinline__ bool om_same_key(const OmRec<K>& a, const OmRec<K>& b) {
    return a.key[0] == b.key[0] && a.key[1] == b.key[1];
}

// r[k] for a run-time k without indexing the array (which would put it in local memory).
__device__ __forceinline__ unsigned long long om_pick(const unsigned long long r[3], int k) {
    return k == 0 ? r[0] : k == 1 ? r[1] : r[2];
}

// Half-edge e = k m + f runs from corner (k + 1) % 3 of face f to corner (k + 2) % 3; corner k is opposite it.
template <typename K>
__global__ void __launch_bounds__(kThreads) om_records_kernel(const void* __restrict__ f, int fkind, long long m, OmRec<K>* __restrict__ rec,
                                                              int* __restrict__ P) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    unsigned long long c[3];
    om_row(f, t, fkind, c);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned long long a = c[(k + 1) % 3], b = c[(k + 2) % 3], lo = min(a, b), hi = max(a, b);
        OmRec<K> r;
        r.key[0] = (K)lo;
        r.key[1] = (K)hi;
        r.idx = (K)(k * m + t);
        store_rec(rec + k * m + t, r);
    }
    P[2 * t] = (int)(2 * t);
    P[2 * t + 1] = (int)(2 * t + 1);
}

// Face and corner slot of half-edge e.
__device__ __forceinline__ int om_slot(unsigned long long e, long long m, long long* face) {
    const int k = e >= (unsigned long long)(2 * m) ? 2 : e >= (unsigned long long)m ? 1 : 0;
    *face = (long long)e - k * m;
    return k;
}

// nb[e] (set to -1 before) = the other face of half-edge e's run when that run is a pair.
template <typename K>
__global__ void __launch_bounds__(kThreads) om_runs_kernel(const OmRec<K>* __restrict__ rec, long long n, long long m, const void* __restrict__ f,
                                                           int fkind, int* __restrict__ nb, int* P) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const OmRec<K> head = load_rec(rec + i);
    if (i > 0 && om_same_key(load_rec(rec + i - 1), head)) return;
    long long fa = -1, fb = -1, j = i;
    for (; j < n; ++j) {
        const OmRec<K> r = load_rec(rec + j);
        if (!om_same_key(r, head)) break;
        long long g;
        om_slot(r.idx, m, &g);
        if (g == fa || g == fb) continue;
        if (fa < 0) fa = g;
        else if (fb < 0) fb = g;
        else return;                        // a third face: the edge joins no faces
    }
    if (fb < 0) return;                     // a boundary edge
    for (long long q = i; q < j; ++q) {
        const unsigned long long e = rec[q].idx;
        long long g;
        om_slot(e, m, &g);
        nb[e] = (int)(g == fa ? fb : fa);
    }
    bool regular = j - i == 2;
    bool same_direction = false;
    if (regular) {
        long long f0, f1;
        const int k0 = om_slot(rec[i].idx, m, &f0), k1 = om_slot(rec[i + 1].idx, m, &f1);
        unsigned long long a[3], b[3];
        om_row(f, f0, fkind, a);
        om_row(f, f1, fkind, b);
        regular = a[0] != a[1] && a[1] != a[2] && a[0] != a[2] && b[0] != b[1] && b[1] != b[2] && b[0] != b[2] &&
                  om_pick(a, k0) != om_pick(b, k1);
        same_direction = om_pick(a, (k0 + 1) % 3) == om_pick(b, (k1 + 1) % 3);
    }
    const int pa = (int)(2 * fa), pb = (int)(2 * fb);
    if (!regular) {
        uf_union(P, pa, pa + 1);
        uf_union(P, pa, pb);
        uf_union(P, pb, pb + 1);
    } else if (same_direction) {
        uf_union(P, pa, pb + 1);
        uf_union(P, pa + 1, pb);
    } else {
        uf_union(P, pa, pb);
        uf_union(P, pa + 1, pb + 1);
    }
}

__global__ void __launch_bounds__(kThreads) om_flatten_kernel(int* P, long long m, int* __restrict__ root, unsigned char* __restrict__ flag) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    const int r = uf_find(P, (int)(2 * t));
    root[t] = r;
    unsigned char fl = 0;
    if (r == (int)(2 * t)) fl = uf_find(P, r + 1) == r ? kOmCollapsedSeed : kOmSeed;
    flag[t] = fl;
}

// Rows of f (I's bits), reversed where find(2f) is odd, and ids[f] = rank of the patch's smallest face.
template <typename I>
__global__ void __launch_bounds__(kThreads) om_emit_kernel(const I* __restrict__ f, long long m, const int* __restrict__ root,
                                                           const int* __restrict__ rank, I* __restrict__ out_f, I* __restrict__ out_c) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    const int r = root[t];
    const I a = f[3 * t], b = f[3 * t + 1], c = f[3 * t + 2];
    const bool flip = r & 1;
    out_f[3 * t] = flip ? c : a;
    out_f[3 * t + 1] = b;
    out_f[3 * t + 2] = flip ? a : c;
    out_c[t] = (I)__ldg(rank + (r >> 1));
}

// bfs_orient from the smallest face of each collapsed patch, on the rows om_emit_kernel wrote (unflipped there).  A
// face's neighbours are its distinct slots in ascending order; for each, its nine directed-edge comparisons with the
// popped face, in the edge order (1, 2), (2, 0), (0, 1), reverse its row on every match, and later comparisons see the
// reversed row.  enq (zeroed before) marks the faces ever pushed; next links the queue.
template <typename I>
__global__ void __launch_bounds__(kThreads) om_replay_kernel(const unsigned char* __restrict__ flag, long long m, const int* __restrict__ nb,
                                                             unsigned char* __restrict__ enq, int* __restrict__ next, I* ff) {
    const long long s = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (s >= m || flag[s] != kOmCollapsedSeed) return;
    int head = (int)s, tail = (int)s;
    enq[s] = 1;
    next[s] = -1;
    while (head >= 0) {
        const int f = head;
        head = next[f];
        const I a0 = ff[3ll * f], a1 = ff[3ll * f + 1], a2 = ff[3ll * f + 2];
        int x = nb[f], y = nb[m + f], z = nb[2 * m + f];
        if (x > y) { const int t = x; x = y; y = t; }
        if (y > z) { const int t = y; y = z; z = t; }
        if (x > y) { const int t = x; x = y; y = t; }
        const int nbr[3] = {x, y, z};
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const int n = nbr[q];
            if (n < 0 || (q > 0 && n == nbr[q - 1])) continue;
            I c[3] = {ff[3ll * n], ff[3ll * n + 1], ff[3ll * n + 2]};
            const I ef[3][2] = {{a1, a2}, {a2, a0}, {a0, a1}};
            bool flipped = false;
#pragma unroll
            for (int efi = 0; efi < 3; ++efi)
#pragma unroll
                for (int eni = 0; eni < 3; ++eni)
                    if (ef[efi][0] == c[(eni + 1) % 3] && ef[efi][1] == c[(eni + 2) % 3]) {
                        const I t = c[0]; c[0] = c[2]; c[2] = t;
                        flipped = !flipped;
                    }
            if (flipped) { ff[3ll * n] = c[0]; ff[3ll * n + 2] = c[2]; }
            if (!enq[n]) {
                enq[n] = 1;
                next[n] = -1;
                if (head < 0) head = n;
                else next[tail] = n;
                tail = n;
            }
        }
    }
}

}  // namespace pcu
