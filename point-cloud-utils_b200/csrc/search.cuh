// search.cuh -- exact nearest-neighbour sweeps over the cell-sorted clouds.
//
// Replaces nanoflann's per-query kd-tree descent (external/nanoflann/nanoflann.hpp:1545-1624,
// KNNResultSet :157-230) and the reductions the reference performs afterwards on the CPU
// (dists.maxCoeff, src/point_cloud_distance.cpp:221-225; norm(...).mean(),
// point_cloud_utils/__init__.py:112-113).
//
// Exactness argument (DESIGN.md "why the grid search is exact"): a query examines whole cells; a
// cell that was NOT examined only contains points whose coordinate along some axis lies beyond a
// wall (grid.cuh), and because fl(q - p), fl(d*d) and fl(a + b) are all monotone, the squared gap
// to that wall, computed with the very same rounded operations, is a lower bound of the
// reference-rounded distance to every such point.  A query is final only when its current k-th
// distance is STRICTLY below that bound, so exact ties are never hidden either.
#pragma once
#include "common.cuh"
#include "grid.cuh"
#include "../../include/pcu_b200.h"

namespace pcu {

template <typename T>
struct SweepPartial {
    double sum, sumsq;
    T max_d2;
    unsigned arg_q;     // caller-order row of the query attaining max_d2 (first one)
    unsigned arg_pos;   // its position in cell order (the witness search starts from there)
    unsigned arg_nn;    // its witness word (witness_word) when the pass that answered it knew it, else kWitnessUnknown
};

// One query-cloud -> dataset-cloud direction.
template <typename T>
struct Sweep {
    int qcloud, dcloud;
    int k;
    int squared;
    int main_blocks;             // partial slots [0, main_blocks) are written by the main kernel
    int far_blocks;              // partial slots [main_blocks, main_blocks + far_blocks) by the pyramid pass
    T* out_dist;                 // (n, k) or null
    long long* out_idx;          // (n, k) or null
    SweepPartial<T>* partial;    // main_blocks + far blocks slots, or null
    unsigned* far_list;          // sorted-order positions of queries the one-ring pass could not settle
    unsigned* vfar_list;         // ... and of those the ring walk gave up on (answered by the pyramid descent)
    unsigned* counters;          // [0] far queries, [1] tied, [2] very far, [3] finished CTAs of the last pass, [4] pair ticket
    long long* tie_list;         // caller-order rows whose answer depends on tie order
    pcu_b200_nn_stats* stats;    // or null
    // bidirectional calls: where the pair's Chamfer value goes (null: not wanted), the pair's two
    // statistics records and a zeroed ticket shared by the two sweeps of the pair
    T* value_out;
    pcu_b200_nn_stats* pair_stats;
    unsigned* pair_ticket;
};

template <typename T>
struct SweepsPtr {
    const Sweep<T>* p;
    __device__ __forceinline__ const Sweep<T>& operator[](int i) const { return p[i]; }
};
template <typename T>
struct SweepsVal {
    Sweep<T> v[2];
    __device__ __forceinline__ const Sweep<T>& operator[](int i) const { return v[i]; }
};

// The running nearest neighbour of one query.  d starts at the largest finite value, as nanoflann's KNNResultSet
// does (init), so a point whose rounded d^2 is exactly that value or overflows to +inf is never admitted and
// d < Real<T>::largest() holds exactly when a neighbour was found.  While d is still at its start value the tie
// branch of the offers may record a point at that distance in i and tie; found1() ignores both then.
template <typename T>
struct Best1 {
    T d;
    typename Real<T>::index_t i;
    bool tie;
};

template <typename T>
__device__ __forceinline__ bool found1(const Best1<T>& b) { return b.d < Real<T>::largest(); }

template <typename T> __device__ __forceinline__ typename Real<T>::index_t no_index();
template <> __device__ __forceinline__ int32_t no_index<float>() { return 0x7fffffff; }
template <> __device__ __forceinline__ long long no_index<double>() { return 0x7fffffffffffffffLL; }

// The Hausdorff witness of one answered query in one word: the neighbour's index in bits 0-30 (clouds hold fewer
// than 2^31 points; kWitnessNone when no point was found) and, in bit 31, whether tie order decided it.  A query
// without a neighbour never gets the tie bit, so no witness word equals kWitnessUnknown, which the main
// statistics pass writes: it tracks distances only.
constexpr unsigned kWitnessUnknown = 0xffffffffu;
constexpr unsigned kWitnessNone = 0x7fffffffu;
template <typename T>
__device__ __forceinline__ unsigned witness_word(const Best1<T>& b) {
    return found1<T>(b) ? (unsigned)b.i | (b.tie ? 0x80000000u : 0u) : kWitnessNone;
}

template <typename T>
__device__ __forceinline__ void offer1(Best1<T>& b, T d, typename Real<T>::index_t i) {
    if (d <= b.d) {
        if (d == b.d) { b.tie = true; b.i = i < b.i ? i : b.i; }
        else { b.d = d; b.i = i; b.tie = false; }
    }
}

// Same update as offer1 written with selects (no divergent branch inside the hot loop).
template <typename T>
__device__ __forceinline__ void offer1_select(Best1<T>& b, T d, typename Real<T>::index_t i, bool valid) {
    const bool lt = valid && d < b.d;
    const bool eq = valid && d == b.d;
    const typename Real<T>::index_t lower = i < b.i ? i : b.i;
    b.i = lt ? i : (eq ? lower : b.i);
    b.tie = !lt && (eq || b.tie);
    b.d = lt ? d : b.d;
}

template <typename T>
__device__ __forceinline__ void scan_run1(const Pt<T>* __restrict__ pts, unsigned a, unsigned b, T qx, T qy, T qz,
                                          Best1<T>& best) {
    for (unsigned j = a; j < b; ++j) {
        const Pt<T> p = load_pt<T>(pts + j);
        offer1<T>(best, dist2<T>(qx, qy, qz, p.x, p.y, p.z), p.i);
    }
}

// Visits the cells of the dataset grid around (qx,qy,qz) ring by ring (Chebyshev distance in cell
// units), starting at ring r0.  `visit(a, b, bound)` receives a contiguous run [a, b) of sorted
// points and a lower bound of the distance to all of them; `settled(lb)` is asked after each ring
// with the lower bound for everything not examined so far.
// Returns true when the search is complete (bound closed or whole grid examined), false when it
// stopped because `max_ring` rings were not enough.
template <typename T, typename Visit, typename Settled>
__device__ __forceinline__ bool expand_rings(const GridHeader<T>& g, const T* __restrict__ wall_lo,
                                             const T* __restrict__ wall_hi, const unsigned* __restrict__ cell_start,
                                             T qx, T qy, T qz, int r0, int max_ring, Visit&& visit, Settled&& settled) {
    using R = Real<T>;
    const int cx = cell_of<T>(qx, g.origin[0], g.inv_h, g.dim[0]);
    const int cy = cell_of<T>(qy, g.origin[1], g.inv_h, g.dim[1]);
    const int cz = cell_of<T>(qz, g.origin[2], g.inv_h, g.dim[2]);
    const int st = g.stride;
    const T* lo_x = wall_lo;           const T* hi_x = wall_hi;
    const T* lo_y = wall_lo + st;      const T* hi_y = wall_hi + st;
    const T* lo_z = wall_lo + 2 * st;  const T* hi_z = wall_hi + 2 * st;
    for (int r = r0; r <= max_ring; ++r) {
        const int xa = max(cx - r, 0), xb = min(cx + r, g.dim[0] - 1);
        const int ya = max(cy - r, 0), yb = min(cy + r, g.dim[1] - 1);
        const int za = max(cz - r, 0), zb = min(cz + r, g.dim[2] - 1);
        for (int z = za; z <= zb; ++z) {
            const T bz = z < cz ? sq_gap<T>(qz, lo_z[z + 1]) : (z > cz ? sq_gap<T>(qz, hi_z[z]) : (T)0);
            for (int y = ya; y <= yb; ++y) {
                const T by = y < cy ? sq_gap<T>(qy, lo_y[y + 1]) : (y > cy ? sq_gap<T>(qy, hi_y[y]) : (T)0);
                const unsigned row = (unsigned)((z * g.dim[1] + y) * g.dim[0]);
                const bool shell_row = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
                if (shell_row || r == 0) {
                    visit(cell_start[row + xa], cell_start[row + xb + 1], R::add(by, bz));
                } else {
                    if (cx - r >= 0) {
                        const T bx = sq_gap<T>(qx, lo_x[cx - r + 1]);
                        visit(cell_start[row + cx - r], cell_start[row + cx - r + 1], R::add(R::add(bx, by), bz));
                    }
                    if (cx + r <= g.dim[0] - 1) {
                        const T bx = sq_gap<T>(qx, hi_x[cx + r]);
                        visit(cell_start[row + cx + r], cell_start[row + cx + r + 1], R::add(R::add(bx, by), bz));
                    }
                }
            }
        }
        T lb = sq_gap<T>(qx, lo_x[xa]);
        lb = R::vmin(lb, sq_gap<T>(qx, hi_x[xb + 1]));
        lb = R::vmin(lb, sq_gap<T>(qy, lo_y[ya]));
        lb = R::vmin(lb, sq_gap<T>(qy, hi_y[yb + 1]));
        lb = R::vmin(lb, sq_gap<T>(qz, lo_z[za]));
        lb = R::vmin(lb, sq_gap<T>(qz, hi_z[zb + 1]));
        if (settled(lb)) return true;
        if (xa == 0 && ya == 0 && za == 0 && xb == g.dim[0] - 1 && yb == g.dim[1] - 1 && zb == g.dim[2] - 1) return true;
    }
    return false;
}

// ---------------------------------------------------------------------------------------------
// block-level reduction of the fused statistics
template <typename T>
struct MaxCand {
    T d2;           // -1: neutral element (q = 0xffffffff) or a query without neighbour
    unsigned q;     // caller-order row (clouds are limited to 2^31 - 1 points)
    unsigned pos;   // position in cell order
    unsigned nn;    // witness word of the query, or kWitnessUnknown
};
template <typename T>
__device__ __forceinline__ MaxCand<T> no_max() {
    MaxCand<T> mc; mc.d2 = (T)-1; mc.q = 0xffffffffu; mc.pos = 0u; mc.nn = kWitnessUnknown;
    return mc;
}
template <typename T>
__device__ __forceinline__ void take_max(MaxCand<T>& a, const MaxCand<T>& b) {
    // larger distance wins; equal distance -> lower query row (Eigen maxCoeff: first maximum); the witness
    // travels with the winner
    if (b.d2 > a.d2 || (b.d2 == a.d2 && b.q < a.q)) a = b;
}

// Warp-wide take_max; every lane returns the winner.
template <typename T>
__device__ __forceinline__ MaxCand<T> warp_take_max(MaxCand<T> mc) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        MaxCand<T> other;
        other.d2 = __shfl_xor_sync(0xffffffffu, mc.d2, o);
        other.q = __shfl_xor_sync(0xffffffffu, mc.q, o);
        other.pos = __shfl_xor_sync(0xffffffffu, mc.pos, o);
        other.nn = __shfl_xor_sync(0xffffffffu, mc.nn, o);
        take_max<T>(mc, other);
    }
    return mc;
}
// fp32: the order-preserving image of the distances (>= 0, or -1 for a query without neighbour) lets the hardware
// integer reductions (REDUX) do the work: max of the images, then min row among the lanes holding it.  The neutral
// element (-1, row 0xffffffff) loses to every candidate; a NaN never wins.
template <>
__device__ __forceinline__ MaxCand<float> warp_take_max<float>(MaxCand<float> mc) {
    const bool real = mc.d2 >= -1.f;
    const unsigned bits = real ? ordered<float>(mc.d2) : 0u;
    const unsigned top = __reduce_max_sync(0xffffffffu, bits);
    const bool holds = real && bits == top;
    const unsigned row = holds ? mc.q : 0xffffffffu;
    const unsigned first = __reduce_min_sync(0xffffffffu, row);
    const unsigned who = __ballot_sync(0xffffffffu, holds && row == first);
    if (who == 0u) return mc;         // every lane holds a NaN (non-finite coordinates)
    const int src = __ffs(who) - 1;
    MaxCand<float> out;
    out.d2 = unordered<float>(top);
    out.q = first;
    out.pos = __shfl_sync(0xffffffffu, mc.pos, src);
    out.nn = __shfl_sync(0xffffffffu, mc.nn, src);
    return out;
}

template <typename T>
__device__ __forceinline__ void block_reduce_stats(double sum, double sumsq, MaxCand<T> mc, SweepPartial<T>* out) {
    __shared__ double s_sum[kThreads / 32], s_sq[kThreads / 32];
    __shared__ MaxCand<T> s_mc[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sumsq += __shfl_xor_sync(0xffffffffu, sumsq, o);
    }
    mc = warp_take_max<T>(mc);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { s_sum[w] = sum; s_sq[w] = sumsq; s_mc[w] = mc; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < kThreads / 32; ++i) {   // fixed order: deterministic
            sum += s_sum[i]; sumsq += s_sq[i];
            take_max<T>(mc, s_mc[i]);
        }
        SweepPartial<T> p;
        p.sum = sum; p.sumsq = sumsq; p.max_d2 = mc.d2; p.arg_q = mc.q; p.arg_pos = mc.pos; p.arg_nn = mc.nn;
        *out = p;
    }
}

// kOut: write the query's neighbour to the caller's arrays.  kStats: fold its distance into the fused
// statistics.  In the statistics-only sweeps the hot loop tracks the minimum distance and nothing else:
// the only index the scalar metrics ever need is the neighbour of the ONE query that attains the
// Hausdorff maximum.  The slow passes know it and carry it with the maximum (`witness`: witness_word(best));
// the main pass passes kWitnessUnknown and conclude_sweep recovers it with one warp.
// A query without neighbour enters the Hausdorff maximum as -1, the distance the reference pads its row with, and
// makes the distance sums (hence the Chamfer distance) +inf (DESIGN.md section 3).
template <typename T, bool kOut, bool kStats>
__device__ __forceinline__ void finish_query1(const Sweep<T>& sw, bool have, const Best1<T>& best, long long row,
                                              unsigned pos, unsigned witness, double& sum, double& sumsq, MaxCand<T>& mc) {
    using R = Real<T>;
    if (!have) return;
    const bool found = found1<T>(best);
    const T root = R::root(best.d);
    if (kOut) {
        sw.out_idx[row] = found ? (long long)best.i : -1;
        sw.out_dist[row] = found ? (sw.squared ? best.d : root) : (T)-1;
        if (found && best.tie) sw.tie_list[atomicAdd(sw.counters + 1, 1u)] = row;
    }
    if (kStats) {
        sum += found ? (double)root : (double)R::inf();
        sumsq += found ? (double)best.d : (double)R::inf();
        MaxCand<T> c; c.d2 = found ? best.d : (T)-1; c.q = (unsigned)row; c.pos = pos; c.nn = witness;
        take_max<T>(mc, c);
    }
}

}  // namespace pcu
