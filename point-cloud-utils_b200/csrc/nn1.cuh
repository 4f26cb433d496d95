// nn1.cuh -- the k = 1 sweep (per-point outputs and / or fused Chamfer-Hausdorff statistics).
//
// This is the hot kernel of the path: it replaces the reference's per-query kd-tree descent
// (external/nanoflann/nanoflann.hpp:1545-1624) for every query of both directions of a Chamfer /
// Hausdorff call, and fuses the reductions the reference does afterwards on the CPU
// (src/point_cloud_distance.cpp:221-225, point_cloud_utils/__init__.py:112-113), so no per-point
// distance buffer is ever written for the scalar metrics.
#pragma once
#include <type_traits>
#include "search.cuh"

namespace pcu {

constexpr int kMaxRing = 2;   // rings the far pass examines before a query goes to the pyramid descent

// Per-thread table of the 9 rows (fixed y, z; three x-adjacent cells = one contiguous run of the
// sorted dataset) of a query's 3 x 3 x 3 neighbourhood, nearest rows first.  Indexed [row][thread]
// so that lanes hit distinct banks whatever row each lane is currently on.
// The query's own row (bound 0, always scanned first) stays in registers; the table holds the other
// eight.  That keeps the fp32 sweep at 25.9 KB of shared memory per CTA: six CTAs then fit the 164 KB
// carve-out instead of needing the 196 KB one, which leaves 92 KB instead of 60 KB of the SM's 256 KB
// to the L1 that serves the candidate loads.
template <typename T>
struct RowTable {
    unsigned begin[8][kThreads];
    unsigned end[8][kThreads];
    T bound[8][kThreads];
};

// Merges the running best of two lanes (after each lane has scanned disjoint cells).
template <typename T>
__device__ __forceinline__ void merge_best(Best1<T>& a, const Best1<T>& b) {
    if (b.d < a.d) a = b;
    else if (b.d == a.d) {
        a.tie = a.tie || b.tie || (b.i != a.i);
        a.i = b.i < a.i ? b.i : a.i;
    }
}

// Warp-cooperative ring walk for ONE query: each ring of cells is split over the lanes (one (y, z)
// row per lane and step), the lanes' results are merged, and the walk stops as soon as the wall bound
// closes (returns true) or kMaxRing rings have been examined (returns false unless the whole grid was
// covered).  All lanes return the same best.
template <typename T>
__device__ __forceinline__ bool warp_ring_search(const GridHeader<T>& g, const Cloud<T>& dc, const Pt<T>& q, int lane,
                                                 Best1<T>& best) {
    using R = Real<T>;
    const int st = g.stride;
    const T* lo_x = dc.wall_lo;           const T* hi_x = dc.wall_hi;
    const T* lo_y = dc.wall_lo + st;      const T* hi_y = dc.wall_hi + st;
    const T* lo_z = dc.wall_lo + 2 * st;  const T* hi_z = dc.wall_hi + 2 * st;
    const int cx = cell_of<T>(q.x, g.origin[0], g.inv_h, g.dim[0]);
    const int cy = cell_of<T>(q.y, g.origin[1], g.inv_h, g.dim[1]);
    const int cz = cell_of<T>(q.z, g.origin[2], g.inv_h, g.dim[2]);
    best.d = R::largest(); best.i = no_index<T>(); best.tie = false;
    for (int r = 0; r <= kMaxRing; ++r) {
        const int xa = max(cx - r, 0), xb = min(cx + r, g.dim[0] - 1);
        const int ya = max(cy - r, 0), yb = min(cy + r, g.dim[1] - 1);
        const int za = max(cz - r, 0), zb = min(cz + r, g.dim[2] - 1);
        const int ny = yb - ya + 1, nrows = ny * (zb - za + 1);
        for (int idx = lane; idx < nrows; idx += 32) {
            const int z = za + idx / ny, y = ya + idx % ny;
            const T bz = z < cz ? sq_gap<T>(q.z, lo_z[z + 1]) : (z > cz ? sq_gap<T>(q.z, hi_z[z]) : (T)0);
            const T by = y < cy ? sq_gap<T>(q.y, lo_y[y + 1]) : (y > cy ? sq_gap<T>(q.y, hi_y[y]) : (T)0);
            if (R::add(by, bz) > best.d) continue;
            const unsigned base = (unsigned)((z * g.dim[1] + y) * g.dim[0]);
            const bool shell_row = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
            if (shell_row || r == 0) {
                scan_run1<T>(dc.sorted, dc.cell_start[base + xa], dc.cell_start[base + xb + 1], q.x, q.y, q.z, best);
            } else {
                if (cx - r >= 0 && !(R::add(R::add(sq_gap<T>(q.x, lo_x[cx - r + 1]), by), bz) > best.d))
                    scan_run1<T>(dc.sorted, dc.cell_start[base + cx - r], dc.cell_start[base + cx - r + 1], q.x, q.y, q.z, best);
                if (cx + r <= g.dim[0] - 1 && !(R::add(R::add(sq_gap<T>(q.x, hi_x[cx + r]), by), bz) > best.d))
                    scan_run1<T>(dc.sorted, dc.cell_start[base + cx + r], dc.cell_start[base + cx + r + 1], q.x, q.y, q.z, best);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            Best1<T> other;
            other.d = __shfl_xor_sync(0xffffffffu, best.d, o);
            other.i = __shfl_xor_sync(0xffffffffu, best.i, o);
            other.tie = __shfl_xor_sync(0xffffffffu, (int)best.tie, o) != 0;
            merge_best<T>(best, other);
        }
        T lb = sq_gap<T>(q.x, lo_x[xa]);
        lb = R::vmin(lb, sq_gap<T>(q.x, hi_x[xb + 1]));
        lb = R::vmin(lb, sq_gap<T>(q.y, lo_y[ya]));
        lb = R::vmin(lb, sq_gap<T>(q.y, hi_y[yb + 1]));
        lb = R::vmin(lb, sq_gap<T>(q.z, lo_z[za]));
        lb = R::vmin(lb, sq_gap<T>(q.z, hi_z[zb + 1]));
        if (best.d < lb) return true;
        if (xa == 0 && ya == 0 && za == 0 && xb == g.dim[0] - 1 && yb == g.dim[1] - 1 && zb == g.dim[2] - 1) return true;
    }
    return false;
}

// Warp-cooperative search of ONE query's whole (2r + 1)^3 window of cells in a single round: one (y, z) row per
// lane, each row's x-run [cx - r, cx + r] (x-adjacent cells are one contiguous run of the sorted dataset) scanned
// whole with four candidate loads in flight, then one merge and one check of the window's wall bound.  The window
// is the union of rings 0 .. r and no row is skipped, so what it settles is exactly what warp_ring_search settles
// with r rings (DESIGN.md "why the grid search is exact"), in one dependent round instead of r + 1.  Returns true
// when the bound closed or the window covers the grid; all lanes return the same best.
template <typename T>
__device__ __forceinline__ bool warp_window_search(const GridHeader<T>& g, const Cloud<T>& dc, const Pt<T>& q, int lane,
                                                   int r, Best1<T>& best) {
    using R = Real<T>;
    const int st = g.stride;
    const int cx = cell_of<T>(q.x, g.origin[0], g.inv_h, g.dim[0]);
    const int cy = cell_of<T>(q.y, g.origin[1], g.inv_h, g.dim[1]);
    const int cz = cell_of<T>(q.z, g.origin[2], g.inv_h, g.dim[2]);
    const int xa = max(cx - r, 0), xb = min(cx + r, g.dim[0] - 1);
    const int ya = max(cy - r, 0), yb = min(cy + r, g.dim[1] - 1);
    const int za = max(cz - r, 0), zb = min(cz + r, g.dim[2] - 1);
    // the window's wall bound first, so that its loads are in flight while the rows are scanned
    T lb = sq_gap<T>(q.x, dc.wall_lo[xa]);
    lb = R::vmin(lb, sq_gap<T>(q.x, dc.wall_hi[xb + 1]));
    lb = R::vmin(lb, sq_gap<T>(q.y, dc.wall_lo[st + ya]));
    lb = R::vmin(lb, sq_gap<T>(q.y, dc.wall_hi[st + yb + 1]));
    lb = R::vmin(lb, sq_gap<T>(q.z, dc.wall_lo[2 * st + za]));
    lb = R::vmin(lb, sq_gap<T>(q.z, dc.wall_hi[2 * st + zb + 1]));
    best.d = R::largest(); best.i = no_index<T>(); best.tie = false;
    const int ny = yb - ya + 1, nrows = ny * (zb - za + 1);
    for (int idx = lane; idx < nrows; idx += 32) {
        const int z = za + idx / ny, y = ya + idx % ny;
        const unsigned base = (unsigned)((z * g.dim[1] + y) * g.dim[0]);
        const unsigned a = dc.cell_start[base + xa], b = dc.cell_start[base + xb + 1];
        for (unsigned j = a; j < b; j += 4) {
            Pt<T> p[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) p[u] = load_pt<T>(dc.sorted + min(j + u, b - 1));
#pragma unroll
            for (int u = 0; u < 4; ++u)
                offer1_select<T>(best, dist2<T>(q.x, q.y, q.z, p[u].x, p[u].y, p[u].z), p[u].i, j + u < b);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best1<T> other;
        other.d = __shfl_xor_sync(0xffffffffu, best.d, o);
        other.i = __shfl_xor_sync(0xffffffffu, best.i, o);
        other.tie = __shfl_xor_sync(0xffffffffu, (int)best.tie, o) != 0;
        merge_best<T>(best, other);
    }
    return best.d < lb ||
           (xa == 0 && ya == 0 && za == 0 && xb == g.dim[0] - 1 && yb == g.dim[1] - 1 && zb == g.dim[2] - 1);
}

// Main pass: one thread per (cell-sorted) query.
//   phase A (uniform): look up the 9 runs and the wall bound of each row;
//   phase B: ONE loop in which every trip a lane first steps to its next row if its run is exhausted
//     (skipping rows pruned by their bound) and then evaluates its next two candidates;
//   queries the 3 x 3 x 3 neighbourhood cannot settle (empty surroundings) go to the far list
//   (nn1_far_kernel below; doing them here, one warp each, cost more in registers and idle warps
//   than the extra launch -- measured).
// grid (ceil(max_n / kThreads), nsweeps).
template <typename T, typename CS, typename SS, bool kOut, bool kStats>
__global__ void __launch_bounds__(kThreads, sizeof(T) == 4 ? 6 : 4) nn1_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    using R = Real<T>;
    const Sweep<T> sw = sweeps[blockIdx.y];
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    if ((long long)blockIdx.x * blockDim.x >= qc.n) return;   // blocks beyond this sweep's queries
    __shared__ GridHeader<T> g;
    __shared__ RowTable<T> rows;
    if (threadIdx.x == 0) g = *dc.grid;
    __syncthreads();

    const int tid = threadIdx.x;
    const long long t = (long long)blockIdx.x * blockDim.x + tid;
    const bool active = t < qc.n;
    Best1<T> best; best.d = R::largest(); best.i = no_index<T>(); best.tie = false;
    bool settled = false;
    long long row = -1;
    if (active) {
        const Pt<T> q = load_pt<T>(qc.sorted + t);
        row = (long long)q.i;
        // wall tables indexed with unsigned 32-bit offsets off the two base pointers (axis a starts at a * stride)
        const T* __restrict__ wl = dc.wall_lo;
        const T* __restrict__ wh = dc.wall_hi;
        int cx = cell_of<T>(q.x, g.origin[0], g.inv_h, g.dim[0]);
        int cy = cell_of<T>(q.y, g.origin[1], g.inv_h, g.dim[1]);
        int cz = cell_of<T>(q.z, g.origin[2], g.inv_h, g.dim[2]);
        unsigned j = 0, e = 0;
        {   // phase A: the query's own row's run and the row table
            const int xa = max(cx - 1, 0), xb = min(cx + 1, g.dim[0] - 1);
            // gaps to the walls of the query's own cell along y and z
            const unsigned ust = (unsigned)g.stride;
            const T gy[3] = {(T)0, sq_gap<T>(q.y, __ldg(wl + (ust + (unsigned)cy))), sq_gap<T>(q.y, __ldg(wh + (ust + (unsigned)cy + 1u)))};
            const T gz[3] = {(T)0, sq_gap<T>(q.z, __ldg(wl + (2u * ust + (unsigned)cz))), sq_gap<T>(q.z, __ldg(wh + (2u * ust + (unsigned)cz + 1u)))};
            // (dy, dz) as indices into {0: same, 1: minus one, 2: plus one}; nearest rows first.  All index
            // arithmetic in unsigned 32 bits off one centre-row index (one IMAD.WIDE per load instead of a
            // 64-bit add chain), the in-range tests once per direction instead of once per row.
            const int order_y[9] = {0, 1, 2, 0, 0, 1, 2, 1, 2};
            const int order_z[9] = {0, 0, 0, 1, 2, 1, 1, 2, 2};
            const unsigned d0 = (unsigned)g.dim[0], slab = d0 * (unsigned)g.dim[1];
            const unsigned centre = ((unsigned)cz * (unsigned)g.dim[1] + (unsigned)cy) * d0;
            const bool ok_y[3] = {true, cy > 0, cy + 1 < g.dim[1]};
            const bool ok_z[3] = {true, cz > 0, cz + 1 < g.dim[2]};
            const unsigned off_y[3] = {0u, 0u - d0, d0};
            const unsigned off_z[3] = {0u, 0u - slab, slab};
            const unsigned* __restrict__ cs = dc.cell_start;
            const unsigned first_x = (unsigned)xa, past_x = (unsigned)xb + 1u;
#pragma unroll
            for (int s = 0; s < 9; ++s) {
                const int oy = order_y[s], oz = order_z[s];
                const unsigned base = centre + off_y[oy] + off_z[oz];
                unsigned a = 0, b = 0;
                if (ok_y[oy] && ok_z[oz]) {
                    a = __ldg(cs + (base + first_x));
                    b = __ldg(cs + (base + past_x));
                }
                if (s == 0) { j = a; e = b; }
                else {
                    rows.begin[s - 1][tid] = a;
                    rows.end[s - 1][tid] = b;
                    rows.bound[s - 1][tid] = R::add(gy[oy], gz[oz]);
                }
            }
        }
        int r = 0;
        for (;;) {
            // Every trip first steps to the next row if the current run is exhausted (predicated; a pruned
            // row leaves the lane idle for this trip) and THEN evaluates candidates, so the lanes of a
            // warp stay in one instruction stream: a lane that has just changed rows does not force a
            // separate pass over the candidate code for the lanes that have not (ncu had shown 8 of 32
            // lanes active there).  One step per trip, not two.
            if (j >= e && r < 8) {
                ++r;
                // a row whose bound exceeds the current best only holds strictly farther points
                const bool keep = !(rows.bound[r - 1][tid] > best.d);
                const unsigned nb = rows.begin[r - 1][tid], ne = rows.end[r - 1][tid];
                j = keep ? nb : 0u;
                e = keep ? ne : 0u;
            }
            const bool has = j < e;
            if (!has && r >= 8) break;
            if (has) {
                // two candidates per step: both loads are issued before either distance is needed
                const bool two = j + 1 < e;
                const Pt<T> p0 = load_pt<T>(dc.sorted + j);
                const Pt<T> p1 = load_pt<T>(dc.sorted + (two ? j + 1 : j));
                j += 2;
                const T d0 = dist2<T>(q.x, q.y, q.z, p0.x, p0.y, p0.z);
                const T d1 = dist2<T>(q.x, q.y, q.z, p1.x, p1.y, p1.z);
                if constexpr (kOut) {
                    offer1_select<T>(best, d0, p0.i, true);
                    offer1_select<T>(best, d1, p1.i, two);
                } else {   // statistics only: the minimum distance is all the scalar metrics need
                    best.d = R::vmin(best.d, R::vmin(d0, two ? d1 : d0));
                }
            }
        }
        if constexpr (std::is_same<CS, CloudsVal<T>>::value) {
            // The query's cell, recomputed from q and the shared header rather than kept live through the loop.
            // At the 40-register cap of six CTAs per SM, keeping it made the allocator load both candidates of a
            // trip of the by-value fp32 sweep (C3) into the same four registers, so each trip waited for two L1/L2
            // round trips in series (tools/sweep_sass.py shows the loads in flight).  The pointer-descriptor
            // sweeps had both loads in flight already and measured slower with the recomputation.
            cx = cell_of<T>(q.x, g.origin[0], g.inv_h, g.dim[0]);
            cy = cell_of<T>(q.y, g.origin[1], g.inv_h, g.dim[1]);
            cz = cell_of<T>(q.z, g.origin[2], g.inv_h, g.dim[2]);
        }
        const int xa = max(cx - 1, 0), xb = min(cx + 1, g.dim[0] - 1);
        const int ya = max(cy - 1, 0), yb = min(cy + 1, g.dim[1] - 1);
        const int za = max(cz - 1, 0), zb = min(cz + 1, g.dim[2] - 1);
        const unsigned ust = (unsigned)g.stride;
        T lb = sq_gap<T>(q.x, __ldg(wl + (unsigned)xa));
        lb = R::vmin(lb, sq_gap<T>(q.x, __ldg(wh + ((unsigned)xb + 1u))));
        lb = R::vmin(lb, sq_gap<T>(q.y, __ldg(wl + (ust + (unsigned)ya))));
        lb = R::vmin(lb, sq_gap<T>(q.y, __ldg(wh + (ust + (unsigned)yb + 1u))));
        lb = R::vmin(lb, sq_gap<T>(q.z, __ldg(wl + (2u * ust + (unsigned)za))));
        lb = R::vmin(lb, sq_gap<T>(q.z, __ldg(wh + (2u * ust + (unsigned)zb + 1u))));
        settled = best.d < lb;
        if (!settled) sw.far_list[atomicAdd(sw.counters, 1u)] = (unsigned)t;
    }
    double sum = 0.0, sumsq = 0.0;
    MaxCand<T> mc = no_max<T>();
    finish_query1<T, kOut, kStats>(sw, active && settled, best, row, (unsigned)t, kWitnessUnknown, sum, sumsq, mc);
    if (kStats) block_reduce_stats<T>(sum, sumsq, mc, sw.partial + blockIdx.x);
}

template <typename T> __device__ void build_pyramid(const Cloud<T>& dc);   // pyramid.cuh
template <typename T> struct Cloud;
template <typename T> __device__ void conclude_sweep(const Sweep<T>& sw, const Cloud<T>& qc, const Cloud<T>& dc, int nparts);   // pyramid.cuh
template <typename T> __device__ __forceinline__ SweepPartial<T> load_partial(const SweepPartial<T>* src);

// Slow pass for the queries the 3 x 3 x 3 neighbourhood could not settle (empty surroundings): one
// WARP per query, which scans the kMaxRing window in one round (warp_window_search; rings 0 and 1 alone cannot
// settle such a query, the main pass has just found so); what the window cannot settle goes to the very-far list.
// Every query it answers carries its witness (neighbour, tie flag) into the statistics.
// Its CTAs also fold the main pass's per-block statistics partials into their own (slot s belongs to
// CTA s mod gridDim), so the CTA that finishes last has only far_blocks partials left to combine: if the
// very-far list is empty -- the rule on overlapping clouds -- it concludes the sweep right here
// (statistics record, Hausdorff witness, Chamfer value; no further launch has anything to do);
// otherwise it builds the dataset's occupancy pyramid and the pyramid pass concludes.
// grid (sw.far_blocks, nsweeps), warp-stride loop over the far list.
template <typename T, typename CS, typename SS, bool kOut, bool kStats>
__global__ void __launch_bounds__(kThreads) nn1_far_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    const Sweep<T> sw = sweeps[blockIdx.y];
    const unsigned n_far = sw.counters[0];
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    const int lane = threadIdx.x & 31;
    const unsigned warps_total = gridDim.x * (kThreads / 32);
    if (blockIdx.x == 0 && threadIdx.x == 0) publish_far_hint<T>(dc, n_far, qc.n);
    double sum = 0.0, sumsq = 0.0;
    MaxCand<T> mc = no_max<T>();
    if (n_far > 0) {
        const GridHeader<T> g = *dc.grid;
        for (unsigned f = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); f < n_far; f += warps_total) {
            const unsigned qt = sw.far_list[f];
            const Pt<T> q = load_pt<T>(qc.sorted + qt);
            Best1<T> best;
            const bool ok = warp_window_search<T>(g, dc, q, lane, kMaxRing, best);
            if (!ok && lane == 0) sw.vfar_list[atomicAdd(sw.counters + 2, 1u)] = qt;
            finish_query1<T, kOut, kStats>(sw, ok && lane == 0, best, (long long)q.i, qt, witness_word<T>(best), sum, sumsq, mc);
        }
    }
    if (kStats) {
        const int main_used = (int)((qc.n + kThreads - 1) / kThreads);
        for (int s = blockIdx.x + threadIdx.x * gridDim.x; s < main_used; s += gridDim.x * blockDim.x) {
            const SweepPartial<T> p = load_partial<T>(sw.partial + s);
            sum += p.sum; sumsq += p.sumsq;
            MaxCand<T> c; c.d2 = p.max_d2; c.q = p.arg_q; c.pos = p.arg_pos; c.nn = p.arg_nn;
            take_max<T>(mc, c);
        }
        block_reduce_stats<T>(sum, sumsq, mc, sw.partial + sw.main_blocks + blockIdx.x);
    }
    __shared__ bool s_last;
    __syncthreads();   // every warp of this CTA has made its very-far appends before the CTA draws its ticket
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(sw.counters + 5, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        if (*(volatile unsigned*)(sw.counters + 2) > 0) build_pyramid<T>(dc);
        else if (kStats) conclude_sweep<T>(sw, qc, dc, sw.far_blocks);
    }
}

// Reads one per-block partial written by another CTA (possibly in this very launch): around L1.
template <typename T>
__device__ __forceinline__ SweepPartial<T> load_partial(const SweepPartial<T>* src) {
    SweepPartial<T> p;
    p.sum = __ldcg(&src->sum); p.sumsq = __ldcg(&src->sumsq); p.max_d2 = __ldcg(&src->max_d2);
    p.arg_q = __ldcg(&src->arg_q); p.arg_pos = __ldcg(&src->arg_pos); p.arg_nn = __ldcg(&src->arg_nn);
    return p;
}

// Combines the first `total` partials of the slow passes (far pass, which carries the main pass | pyramid
// pass) into one.  Called by ONE CTA.
template <typename T>
__device__ __forceinline__ void finalize_sweep(const Sweep<T>& sw, SweepPartial<T>* result /* shared */, int total) {
    double sum = 0.0, sumsq = 0.0;
    MaxCand<T> mc = no_max<T>();
    for (int s = threadIdx.x; s < total; s += blockDim.x) {
        const SweepPartial<T> p = load_partial<T>(sw.partial + sw.main_blocks + s);
        sum += p.sum; sumsq += p.sumsq;
        MaxCand<T> c; c.d2 = p.max_d2; c.q = p.arg_q; c.pos = p.arg_pos; c.nn = p.arg_nn;
        take_max<T>(mc, c);
    }
    block_reduce_stats<T>(sum, sumsq, mc, result);
    __syncthreads();
}

// chamfer = mean_x |x - NN_y(x)| + mean_y |y - NN_x(y)|  (point_cloud_utils/__init__.py:112-115)
__device__ __forceinline__ double chamfer_of64(const pcu_b200_nn_stats& a, const pcu_b200_nn_stats& b) {
    return a.sum_dist / (double)a.n_queries + b.sum_dist / (double)b.n_queries;
}
template <typename T>
__device__ __forceinline__ T chamfer_of(const pcu_b200_nn_stats& a, const pcu_b200_nn_stats& b) {
    return (T)chamfer_of64(a, b);
}

// stats: 2 per pair ([2p] = x->y, [2p+1] = y->x).  One block; pairs strided over its threads.
// Used by the batched entry point (per-pair values and their fp64 sum).
template <typename T>
__global__ void __launch_bounds__(kThreads) chamfer_value_kernel(const pcu_b200_nn_stats* __restrict__ stats,
                                                                 long long npairs, T* __restrict__ out_value,
                                                                 double* __restrict__ out_sum, int accumulate) {
    double acc = 0.0;
    for (long long p = threadIdx.x; p < npairs; p += blockDim.x) {
        const T vt = chamfer_of<T>(stats[2 * p], stats[2 * p + 1]);
        if (out_value) out_value[p] = vt;
        acc += (double)vt;
    }
    if (out_sum == nullptr) return;
    __shared__ double s[kThreads];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out_sum = accumulate ? *out_sum + s[0] : s[0];   // later slices of one call add up (stream order)
}

}  // namespace pcu
