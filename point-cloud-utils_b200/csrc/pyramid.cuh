// pyramid.cuh -- robust slow path for queries that are far from every dataset point.
//
// The ring walk (search.cuh / nn1.cuh) visits every cell of a ring whether it holds points or not, so
// a query at distance D from the data costs O((D/h)^3) cell visits -- fine for the stray query next to
// an empty patch, hopeless when the two clouds do not overlap at all (every query is "far").  Queries
// still unsettled after a few rings are therefore answered by a best-first-ish descent of an occupancy
// pyramid over the dataset grid (level l halves the resolution l times; a node stores how many points
// lie below it): empty space is skipped in O(1) per node and the search cost becomes logarithmic in
// the grid size.  Exactness is the same wall argument as everywhere else: a node is skipped only when
// the lower bound of the reference-rounded distance to its cell box is STRICTLY above the current best.
//
// The pyramid is built by the last CTA of the far pass (nn1.cuh), and only when that sweep has such
// queries: uniform random clouds never pay for it.
#pragma once
#include "search.cuh"
#include "nn1.cuh"

namespace pcu {

// Fills the levels of the dataset's occupancy pyramid; executed by ONE CTA (the far pass's last one).
template <typename T>
__device__ void build_pyramid(const Cloud<T>& dc) {
    __shared__ PyramidShape ps;
    for (int w = threadIdx.x; w < (int)(sizeof(PyramidShape) / sizeof(int)); w += blockDim.x)
        reinterpret_cast<int*>(&ps)[w] = reinterpret_cast<const int*>(dc.shape)[w];
    __syncthreads();
    for (int l = 1; l <= ps.levels; ++l) {
        const int nx = ps.lvl_dim[l][0], ny = ps.lvl_dim[l][1], nz = ps.lvl_dim[l][2];
        const int cx = ps.lvl_dim[l - 1][0], cy = ps.lvl_dim[l - 1][1], cz = ps.lvl_dim[l - 1][2];
        unsigned* out = dc.pyramid + ps.lvl_off[l];
        const unsigned* below = dc.pyramid + ps.lvl_off[l - 1];   // unused for l == 1
        for (int node = threadIdx.x; node < nx * ny * nz; node += blockDim.x) {
            const int x = node % nx, y = (node / nx) % ny, z = node / (nx * ny);
            unsigned total = 0;
            for (int dz = 0; dz < 2; ++dz)
                for (int dy = 0; dy < 2; ++dy) {
                    const int yy = 2 * y + dy, zz = 2 * z + dz;
                    if (yy >= cy || zz >= cz) continue;
                    const int row = (zz * cy + yy) * cx;
                    const int x0 = 2 * x, x1 = min(2 * x + 2, cx);
                    if (l == 1) total += dc.cell_start[row + x1] - dc.cell_start[row + x0];   // x-adjacent cells are contiguous
                    else for (int xx = x0; xx < x1; ++xx) total += __ldcg(below + row + xx);
                }
            out[node] = total;
        }
        __threadfence();
        __syncthreads();
    }
}

// Depth-first descent of the occupancy pyramid for one query, nearer children first.
//   worst()        current k-th distance: a node is entered unless its bound is STRICTLY above it
//   visit(a, b)    scan the sorted points [a, b) of one cell
template <typename T, typename Worst, typename Visit>
__device__ __forceinline__ void pyramid_descend(const GridHeader<T>& g, const PyramidShape& ps, const Cloud<T>& dc,
                                                const Pt<T>& q, Worst&& worst, Visit&& visit) {
    using R = Real<T>;
    const int st = g.stride;
    const T* lo[3] = {dc.wall_lo, dc.wall_lo + st, dc.wall_lo + 2 * st};
    const T* hi[3] = {dc.wall_hi, dc.wall_hi + st, dc.wall_hi + 2 * st};
    const T qv[3] = {q.x, q.y, q.z};
    int qc3[3];
    for (int a = 0; a < 3; ++a) qc3[a] = cell_of<T>(qv[a], g.origin[a], g.inv_h, g.dim[a]);
    // node = level (4 bits) | x (12) | y (12) | z (12)
    unsigned long long stack[8 * kMaxLevels + 8];
    int top = 0;
    stack[top++] = (unsigned long long)ps.levels << 36;
    while (top > 0) {
        const unsigned long long nd = stack[--top];
        const int l = (int)(nd >> 36), x = (int)((nd >> 24) & 0xfff), y = (int)((nd >> 12) & 0xfff), z = (int)(nd & 0xfff);
        const int c0[3] = {x << l, y << l, z << l};
        int pref = 0;   // bit a set: the query lies towards the upper half of the node along axis a
        T gap[3];
        for (int a = 0; a < 3; ++a) {
            const int c1 = min(((c0[a] >> l) + 1 << l) - 1, g.dim[a] - 1);
            gap[a] = qc3[a] < c0[a] ? sq_gap<T>(qv[a], hi[a][c0[a]])
                                    : (qc3[a] > c1 ? sq_gap<T>(qv[a], lo[a][c1 + 1]) : (T)0);
            if (l > 0 && qc3[a] >= c0[a] + (1 << (l - 1))) pref |= 1 << a;
        }
        if (R::add(R::add(gap[0], gap[1]), gap[2]) > worst()) continue;   // everything below is strictly farther
        if (l == 0) {
            const unsigned lin = (unsigned)((z * g.dim[1] + y) * g.dim[0] + x);
            visit(dc.cell_start[lin], dc.cell_start[lin + 1]);
            continue;
        }
        const int cl = l - 1;
        const int nx = ps.lvl_dim[cl][0], ny = ps.lvl_dim[cl][1], nz = ps.lvl_dim[cl][2];
        const unsigned* lvl = dc.pyramid + ps.lvl_off[cl];
        // children in order of increasing Hamming distance from the preferred octant; pushed in
        // reverse so that the nearest is popped first
        const int order[8] = {7, 6, 5, 3, 4, 2, 1, 0};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int ch = order[j] ^ pref;
            const int xx = 2 * x + (ch & 1), yy = 2 * y + ((ch >> 1) & 1), zz = 2 * z + ((ch >> 2) & 1);
            if (xx >= nx || yy >= ny || zz >= nz) continue;
            const unsigned lin = (unsigned)((zz * ny + yy) * nx + xx);
            const unsigned count = cl == 0 ? dc.cell_start[lin + 1] - dc.cell_start[lin] : lvl[lin];
            if (count == 0) continue;
            stack[top++] = ((unsigned long long)cl << 36) | ((unsigned long long)xx << 24) |
                           ((unsigned long long)yy << 12) | (unsigned long long)zz;
        }
    }
}

template <typename T>
__device__ __forceinline__ void load_shapes(const Cloud<T>& dc, GridHeader<T>& g, PyramidShape& ps) {
    if (threadIdx.x == 0) g = *dc.grid;
    for (int w = threadIdx.x; w < (int)(sizeof(PyramidShape) / sizeof(int)); w += blockDim.x)
        reinterpret_cast<int*>(&ps)[w] = reinterpret_cast<const int*>(dc.shape)[w];
    __syncthreads();
}

// Last step of a statistics sweep, run by ONE CTA once every partial of the sweep is in memory: folds the
// `nparts` per-CTA partials of the slow passes (which carry the main pass's partials, folded in by
// nn1_far_kernel) into the caller's pcu_b200_nn_stats, takes the Hausdorff witness -- the neighbour of the
// one query that attains the maximum, and whether it was decided by tie order -- and, for a bidirectional
// call, lets the sweep that finishes second write the pair's Chamfer value.
// A maximum answered by the far or the very-far pass carries its witness.  One answered by the main pass
// was settled inside its 3 x 3 x 3 cells, so a single warp finds the witness in one round over their 9 rows;
// the ring walk and the pyramid descent stay behind that round for whatever it cannot settle.
template <typename T>
__device__ void conclude_sweep(const Sweep<T>& sw, const Cloud<T>& qc, const Cloud<T>& dc, int nparts) {
    using R = Real<T>;
    __shared__ SweepPartial<T> result;
    finalize_sweep<T>(sw, &result, nparts);
    __shared__ GridHeader<T> wg;
    __shared__ PyramidShape wps;
    if (threadIdx.x == 0) wg = *dc.grid;
    __syncthreads();
    if (threadIdx.x < 32 && result.max_d2 >= (T)0) {
        Best1<T> wb; wb.d = R::largest(); wb.i = no_index<T>(); wb.tie = false;
        if (result.arg_nn != kWitnessUnknown) {
            const unsigned nn = result.arg_nn & kWitnessNone;
            wb.i = nn == kWitnessNone ? no_index<T>() : (typename Real<T>::index_t)nn;
            wb.tie = (result.arg_nn >> 31) != 0u;
        } else {
            const Pt<T> wq = load_pt<T>(qc.sorted + result.arg_pos);
            if (!warp_window_search<T>(wg, dc, wq, threadIdx.x, 1, wb) && !warp_ring_search<T>(wg, dc, wq, threadIdx.x, wb)) {
                // beyond the rings: the pyramid exists (this query was on the very-far list)
                wb.d = R::largest(); wb.i = no_index<T>(); wb.tie = false;
                for (int w = threadIdx.x; w < (int)(sizeof(PyramidShape) / sizeof(int)); w += 32)
                    reinterpret_cast<int*>(&wps)[w] = reinterpret_cast<const int*>(dc.shape)[w];
                __syncwarp();
                if (threadIdx.x == 0)
                    pyramid_descend<T>(wg, wps, dc, wq, [&]() { return wb.d; },
                                       [&](unsigned a, unsigned b) { scan_run1<T>(dc.sorted, a, b, wq.x, wq.y, wq.z, wb); });
            }
        }
        if (threadIdx.x == 0) {
            pcu_b200_nn_stats st;
            st.sum_dist = result.sum;
            st.sum_sq_dist = result.sumsq;
            st.max_sq_dist = (double)result.max_d2;
            st.argmax_query = (long long)result.arg_q;
            st.argmax_data = wb.i != no_index<T>() ? (long long)wb.i : -1;
            st.n_queries = qc.n;
            st.n_tied = -1;   // not tracked by the statistics-only sweep
            st.n_far = (long long)sw.counters[0];
            st.witness_tied = wb.tie ? 1 : 0;
            st.pair_value = result.sum / (double)qc.n;   // overwritten by the pair's value in bidirectional calls
            *sw.stats = st;
        }
    } else if (threadIdx.x == 0 && !(result.max_d2 >= (T)0)) {
        // no query found a neighbour (max_d2 = -1 from the first such query, as in the reference's padded
        // distances) or none produced a comparable distance (non-finite coordinates): the record is still
        // written, with no witness, so that callers never decode uninitialised memory
        pcu_b200_nn_stats st;
        st.sum_dist = result.sum;
        st.sum_sq_dist = result.sumsq;
        st.max_sq_dist = (double)result.max_d2;
        st.argmax_query = result.max_d2 == (T)-1 && result.arg_q != 0xffffffffu ? (long long)result.arg_q : -1;
        st.argmax_data = -1;
        st.n_queries = qc.n;
        st.n_tied = -1;
        st.n_far = (long long)sw.counters[0];
        st.witness_tied = 0;
        st.pair_value = result.sum / (double)qc.n;
        *sw.stats = st;
    }
    __syncthreads();
    if (sw.pair_stats != nullptr && sw.pair_ticket != nullptr && threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(sw.pair_ticket, 1u) == 1u) {   // the sweep of the pair that finishes second
            __threadfence();
            volatile pcu_b200_nn_stats* ps = sw.pair_stats;
            pcu_b200_nn_stats a, b;
            a.sum_dist = ps[0].sum_dist; a.n_queries = ps[0].n_queries;
            b.sum_dist = ps[1].sum_dist; b.n_queries = ps[1].n_queries;
            const double v = chamfer_of64(a, b);
            ps[0].pair_value = v;
            ps[1].pair_value = v;
            if (sw.value_out != nullptr) *sw.value_out = (T)v;
        }
    }
}

// k = 1: one thread per very-far query.  Nothing to do (and nothing done: the far pass has already
// concluded the sweep) when the very-far list is empty, which is the rule on overlapping clouds.
// grid (sw.far_blocks, nsweeps), thread-stride loop over the very-far list.
template <typename T, typename CS, typename SS, bool kOut, bool kStats>
__global__ void __launch_bounds__(kThreads) nn1_vfar_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    using R = Real<T>;
    const Sweep<T> sw = sweeps[blockIdx.y];
    const unsigned n_vfar = sw.counters[2];
    if (n_vfar == 0) return;
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    double sum = 0.0, sumsq = 0.0;
    MaxCand<T> mc = no_max<T>();
    {
        __shared__ GridHeader<T> g;
        __shared__ PyramidShape ps;
        load_shapes<T>(dc, g, ps);
        const unsigned step = gridDim.x * blockDim.x;
        for (unsigned f = blockIdx.x * blockDim.x + threadIdx.x; f < n_vfar; f += step) {
            const Pt<T> q = load_pt<T>(qc.sorted + sw.vfar_list[f]);
            Best1<T> best; best.d = R::largest(); best.i = no_index<T>(); best.tie = false;
            pyramid_descend<T>(g, ps, dc, q, [&]() { return best.d; },
                               [&](unsigned a, unsigned b) { scan_run1<T>(dc.sorted, a, b, q.x, q.y, q.z, best); });
            finish_query1<T, kOut, kStats>(sw, true, best, (long long)q.i, sw.vfar_list[f], witness_word<T>(best), sum, sumsq, mc);
        }
    }
    if (kStats) {
        block_reduce_stats<T>(sum, sumsq, mc, sw.partial + sw.main_blocks + sw.far_blocks + blockIdx.x);
        __shared__ bool s_last;
        if (threadIdx.x == 0) {
            __threadfence();
            s_last = atomicAdd(sw.counters + 3, 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (s_last) {
            __threadfence();
            conclude_sweep<T>(sw, qc, dc, 2 * sw.far_blocks);   // far pass (with the main pass folded in) | this pass
        }
    }
}

// Builds the pyramid of every sweep's dataset unconditionally (k > 32 path, which descends it for
// every query).  grid (1, nsweeps)
template <typename T, typename CS, typename SS>
__global__ void __launch_bounds__(kThreads) pyramid_build_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    const Cloud<T> dc = clouds[sweeps[blockIdx.y].dcloud];
    build_pyramid<T>(dc);
}

// k > 1 by pyramid descent: one thread per query, the (distance, index)-sorted list lives in the caller's
// output row (squared distances while searching).  kAll == false: the very-far list left by the ring
// passes (k <= 32); kAll == true: every query (k > 32, generic and slow -- large k is not a hot
// configuration).  grid (blocks, nsweeps), thread-stride loop.
template <typename T, typename CS, typename SS, bool kAll>
__global__ void __launch_bounds__(kThreads) knn_descend_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    using R = Real<T>;
    const Sweep<T> sw = sweeps[blockIdx.y];
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    const long long count = kAll ? qc.n : (long long)sw.counters[2];
    if (count == 0) return;
    __shared__ GridHeader<T> g;
    __shared__ PyramidShape ps;
    load_shapes<T>(dc, g, ps);
    const int k = sw.k;
    const long long step = (long long)gridDim.x * blockDim.x;
    for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < count; f += step) {
        const Pt<T> q = load_pt<T>(qc.sorted + (kAll ? f : (long long)sw.vfar_list[f]));
        const long long row = (long long)q.i;
        T* ld = sw.out_dist + row * k;
        long long* li = sw.out_idx + row * k;
        int have = 0;
        T worst = R::largest();   // nanoflann's KNNResultSet::init: a point at exactly this d^2 is never admitted
        long long worst_i = -1;   // no index passes the tie clause below until the list is full
        T rej = R::inf();
        pyramid_descend<T>(g, ps, dc, q, [&]() { return worst; },
            [&](unsigned a, unsigned b) {
                for (unsigned j = a; j < b; ++j) {
                    const Pt<T> p = load_pt<T>(dc.sorted + j);
                    const T d = dist2<T>(q.x, q.y, q.z, p.x, p.y, p.z);
                    const long long pi = (long long)p.i;
                    if (!(d < worst || (d == worst && pi < worst_i))) { rej = R::vmin(rej, d); continue; }
                    if (have == k) rej = R::vmin(rej, ld[k - 1]);
                    int s = have < k ? have : k - 1;
                    while (s > 0 && (ld[s - 1] > d || (ld[s - 1] == d && li[s - 1] > pi))) {
                        ld[s] = ld[s - 1]; li[s] = li[s - 1]; --s;
                    }
                    ld[s] = d; li[s] = pi;
                    if (have < k) ++have;
                    if (have == k) { worst = ld[k - 1]; worst_i = li[k - 1]; }
                }
            });
        bool tie = have == k && rej == worst;
        for (int s = 0; s + 1 < have; ++s) tie = tie || (ld[s] == ld[s + 1]);
        if (!sw.squared) for (int s = 0; s < have; ++s) ld[s] = R::root(ld[s]);
        for (int s = have; s < k; ++s) { ld[s] = (T)-1; li[s] = -1; }
        if (tie) sw.tie_list[atomicAdd(sw.counters + 1, 1u)] = row;
    }
}

}  // namespace pcu
