// topk.cuh -- k > 1 nearest-neighbour sweeps (warp top-k for k <= 32, generic list for larger k).
//
// Replaces nanoflann's KNNResultSet-driven search for k > 1 (external/nanoflann/nanoflann.hpp:157-230,
// :1545-1624 in the reference).  Shares the ring walk and its exactness argument with search.cuh.
#pragma once
#include "search.cuh"
#include "nn1.cuh"

namespace pcu {

// ---------------------------------------------------------------------------------------------
// One query answered by a whole warp (the slow pass of 2 <= k <= 32): lane j holds the j-th best
// (distance, index) pair, candidates are evaluated 32 at a time and inserted with shuffles.  Order
// inside the list is (distance, index) ascending, which is deterministic; queries whose answer depends
// on how the reference orders equal distances are reported in tie_list and re-answered by the kd-tree
// replay.  At most `max_ring` rings are walked; a query still open after that goes to the very-far list.
template <typename T>
__device__ __forceinline__ void knn_warp_one(const Sweep<T>& sw, const Cloud<T>& qc, const Cloud<T>& dc,
                                             const GridHeader<T>& g, long long t, int lane, int max_ring) {
    using R = Real<T>;
    using index_t = typename R::index_t;
    const int k = sw.k;
    const Pt<T> q = load_pt<T>(qc.sorted + t);

    // empty slots and the k-th distance start at the largest finite value (nanoflann's KNNResultSet::init): a point
    // at exactly that d^2, or at +inf, is never admitted, and the tie clause only applies once the list is full
    T dl = R::largest();
    index_t il = no_index<T>();
    T worst = R::largest();
    index_t worst_i = no_index<T>();
    T rej = R::inf();   // smallest distance that was turned away or pushed out (uniform across lanes)
    const unsigned kmask = k >= 32 ? 0xffffffffu : ((1u << k) - 1u);

    auto visit = [&](unsigned a, unsigned b, T bound) {
        if (bound > worst) return;
        for (unsigned base = a; base < b; base += 32) {
            const unsigned j = base + lane;
            const bool valid = j < b;
            T d = R::inf();
            index_t pi = no_index<T>();
            if (valid) {
                const Pt<T> p = load_pt<T>(dc.sorted + j);
                d = dist2<T>(q.x, q.y, q.z, p.x, p.y, p.z);
                pi = p.i;
            }
            const bool pass = valid && (d < worst || (d == worst && pi < worst_i && worst_i != no_index<T>()));
            // distances that never enter the list still matter for the tie flag
            T turned = (valid && !pass) ? d : R::inf();
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) turned = R::vmin(turned, __shfl_xor_sync(0xffffffffu, turned, o));
            rej = R::vmin(rej, turned);
            unsigned mask = __ballot_sync(0xffffffffu, pass);
            while (mask) {
                const int src = __ffs(mask) - 1;
                mask &= mask - 1;
                const T cd = __shfl_sync(0xffffffffu, d, src);
                const index_t ci = __shfl_sync(0xffffffffu, pi, src);
                if (!(cd < worst || (cd == worst && ci < worst_i && worst_i != no_index<T>()))) { rej = R::vmin(rej, cd); continue; }
                const bool before = (dl < cd) || (dl == cd && il < ci);
                const int pos = __popc(__ballot_sync(0xffffffffu, before) & kmask);
                const T pushed = __shfl_sync(0xffffffffu, dl, k - 1);
                const T up_d = __shfl_up_sync(0xffffffffu, dl, 1);
                const index_t up_i = __shfl_up_sync(0xffffffffu, il, 1);
                if (lane < k) {
                    if (lane > pos) { dl = up_d; il = up_i; }
                    else if (lane == pos) { dl = cd; il = ci; }
                }
                rej = R::vmin(rej, pushed);
                worst = __shfl_sync(0xffffffffu, dl, k - 1);
                worst_i = __shfl_sync(0xffffffffu, il, k - 1);
            }
        }
    };
    const bool settled = expand_rings<T>(g, dc.wall_lo, dc.wall_hi, dc.cell_start, q.x, q.y, q.z, 0, max_ring, visit,
                                         [&](T lb) { return worst < lb; });
    if (!settled) {   // rings grow cubically with the distance to the data: the pyramid descent takes over
        if (lane == 0) sw.vfar_list[atomicAdd(sw.counters + 2, 1u)] = (unsigned)t;
        return;
    }

    const long long row = (long long)q.i;
    if (lane < k) {
        const bool found = il != no_index<T>();
        sw.out_idx[row * k + lane] = found ? (long long)il : -1;
        sw.out_dist[row * k + lane] = found ? (sw.squared ? dl : R::root(dl)) : (T)-1;
    }
    const T next_d = __shfl_down_sync(0xffffffffu, dl, 1);
    const bool dup = lane < k - 1 && dl == next_d && il != no_index<T>();
    const bool edge = (rej == worst) && (worst_i != no_index<T>());
    const unsigned any = __ballot_sync(0xffffffffu, dup || edge);
    if (any && lane == 0) sw.tie_list[atomicAdd(sw.counters + 1, 1u)] = row;
}

// Slow pass of 2 <= k <= 32: warp-stride loop over the far list left by knn_thread_kernel, at most
// kMaxRing rings per query; the CTA that finishes last builds the occupancy pyramid if some query is
// still open (knn_descend_kernel then answers it).  grid (far_blocks, nsweeps)
template <typename T, typename CS, typename SS>
__global__ void __launch_bounds__(kThreads) knn_warp_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    const Sweep<T> sw = sweeps[blockIdx.y];
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    const int lane = threadIdx.x & 31;
    const unsigned n_far = sw.counters[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) publish_far_hint<T>(dc, n_far, qc.n);
    if (n_far > 0) {
        const GridHeader<T> g = *dc.grid;
        const unsigned warps_total = gridDim.x * (kThreads / 32);
        for (unsigned f = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); f < n_far; f += warps_total)
            knn_warp_one<T>(sw, qc, dc, g, (long long)sw.far_list[f], lane, kMaxRing);
    }
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(sw.counters + 5, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        if (*(volatile unsigned*)(sw.counters + 2) > 0) build_pyramid<T>(dc);
    }
}

// ---------------------------------------------------------------------------------------------
// 2 <= k <= 32, main pass: ONE THREAD per query with its (distance, index)-sorted list held in
// registers.  An insertion is a fully unrolled compare/select chain (~6 instructions per slot), and
// because 32 queries share every issued instruction, the cost per query is a small fraction of the
// warp-per-query scheme above, which remains the slow pass for the queries this kernel cannot settle
// within the 3 x 3 x 3 neighbourhood.
//
// Slots: K = capacity (power of two >= k).  The K - k surplus slots are filled with a key that is
// smaller than every real key, so they sit at the front of the ascending list for ever and the k-th
// best is always slot K - 1 -- a compile-time register, no dynamic indexing.  Empty slots hold a key at the
// largest finite distance that no candidate at that distance (or at +inf) is less than: as in nanoflann's
// KNNResultSet, only a point strictly nearer than the largest finite value is ever admitted.
template <typename T> struct ListKey;
template <> struct ListKey<float> {
    unsigned long long v;   // (distance bits << 32) | index : distances are >= +0, bits order like values
    static __device__ __forceinline__ ListKey make(float d, int i) {
        ListKey k; k.v = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)i; return k;
    }
    static __device__ __forceinline__ ListKey dead() { ListKey k; k.v = 0ull; return k; }
    static __device__ __forceinline__ ListKey empty() { ListKey k; k.v = 0x7f7fffffull << 32; return k; }   // (FLT_MAX, 0)
    __device__ __forceinline__ bool less(const ListKey& o) const { return v < o.v; }
    __device__ __forceinline__ float dist() const { return __uint_as_float((unsigned)(v >> 32)); }
    __device__ __forceinline__ long long index() const { return (long long)(int)(unsigned)v; }
    __device__ __forceinline__ bool is_empty() const { return v == 0x7f7fffffull << 32; }
};
template <> struct ListKey<double> {
    double d; long long i;
    static __device__ __forceinline__ ListKey make(double d, long long i) { ListKey k; k.d = d; k.i = i; return k; }
    static __device__ __forceinline__ ListKey dead() { ListKey k; k.d = -1.0; k.i = -1; return k; }
    static __device__ __forceinline__ ListKey empty() {   // (DBL_MAX, -1)
        ListKey k; k.d = __longlong_as_double(0x7fefffffffffffffLL); k.i = -1; return k;
    }
    __device__ __forceinline__ bool less(const ListKey& o) const { return d < o.d || (d == o.d && i < o.i); }
    __device__ __forceinline__ double dist() const { return d; }
    __device__ __forceinline__ long long index() const { return i; }
    __device__ __forceinline__ bool is_empty() const { return d == __longlong_as_double(0x7fefffffffffffffLL); }
};

template <typename T, int K>
__device__ __forceinline__ void list_insert(ListKey<T> (&a)[K], const ListKey<T>& key) {
    bool lt[K];
#pragma unroll
    for (int s = 0; s < K; ++s) lt[s] = key.less(a[s]);
#pragma unroll
    for (int s = K - 1; s >= 1; --s) a[s] = lt[s - 1] ? a[s - 1] : (lt[s] ? key : a[s]);
    a[0] = lt[0] ? key : a[0];
}

// grid (ceil(max_n / kThreads), nsweeps)
template <typename T, typename CS, typename SS, int K>
__global__ void __launch_bounds__(kThreads) knn_thread_kernel(const __grid_constant__ CS clouds, const __grid_constant__ SS sweeps) {
    grid_dependency_wait();
    using R = Real<T>;
    const Sweep<T> sw = sweeps[blockIdx.y];
    const Cloud<T> qc = clouds[sw.qcloud];
    const Cloud<T> dc = clouds[sw.dcloud];
    if ((long long)blockIdx.x * blockDim.x >= qc.n) return;
    __shared__ GridHeader<T> g;
    __shared__ RowTable<T> rows;
    if (threadIdx.x == 0) g = *dc.grid;
    __syncthreads();
    const int tid = threadIdx.x;
    const long long t = (long long)blockIdx.x * blockDim.x + tid;
    if (t >= qc.n) return;
    const int k = sw.k;
    const Pt<T> q = load_pt<T>(qc.sorted + t);
    const int st = g.stride;
    const T* lo_x = dc.wall_lo;           const T* hi_x = dc.wall_hi;
    const T* lo_y = dc.wall_lo + st;      const T* hi_y = dc.wall_hi + st;
    const T* lo_z = dc.wall_lo + 2 * st;  const T* hi_z = dc.wall_hi + 2 * st;
    const int cx = cell_of<T>(q.x, g.origin[0], g.inv_h, g.dim[0]);
    const int cy = cell_of<T>(q.y, g.origin[1], g.inv_h, g.dim[1]);
    const int cz = cell_of<T>(q.z, g.origin[2], g.inv_h, g.dim[2]);
    const int xa = max(cx - 1, 0), xb = min(cx + 1, g.dim[0] - 1);
    const T gy[3] = {(T)0, sq_gap<T>(q.y, __ldg(lo_y + cy)), sq_gap<T>(q.y, __ldg(hi_y + cy + 1))};
    const T gz[3] = {(T)0, sq_gap<T>(q.z, __ldg(lo_z + cz)), sq_gap<T>(q.z, __ldg(hi_z + cz + 1))};
    const int order_y[9] = {0, 1, 2, 0, 0, 1, 2, 1, 2};
    const int order_z[9] = {0, 0, 0, 1, 2, 1, 1, 2, 2};
    // unsigned 32-bit index arithmetic off the centre row, range tests once per direction (as in nn1_kernel)
    const unsigned d0 = (unsigned)g.dim[0], slab = d0 * (unsigned)g.dim[1];
    const unsigned centre = ((unsigned)cz * (unsigned)g.dim[1] + (unsigned)cy) * d0;
    const bool ok_y[3] = {true, cy > 0, cy + 1 < g.dim[1]};
    const bool ok_z[3] = {true, cz > 0, cz + 1 < g.dim[2]};
    const unsigned off_y[3] = {0u, 0u - d0, d0};
    const unsigned off_z[3] = {0u, 0u - slab, slab};
    const unsigned* __restrict__ cs = dc.cell_start;
    const unsigned first_x = (unsigned)xa, past_x = (unsigned)xb + 1u;
    unsigned j = 0, e = 0;   // the own row's run; the other eight go to the table
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
    ListKey<T> list[K];
#pragma unroll
    for (int s = 0; s < K; ++s) list[s] = s < K - k ? ListKey<T>::dead() : ListKey<T>::empty();
    T rej = R::inf();   // smallest distance turned away or pushed out: equal to the k-th => order-dependent answer
    // Candidates that beat the current k-th are first parked in a small per-lane queue.  An insertion
    // costs ~6 instructions per list slot and is paid by the whole warp whenever ANY lane inserts, so
    // the warp inserts in rounds -- one parked candidate per lane -- only when some lane's queue is
    // full: the number of rounds follows the busiest lane instead of the union of all lanes.
    constexpr int kPark = 4;
    ListKey<T> park[kPark];
    int parked = 0;
    auto insert_round = [&]() {
        if (parked > 0) {
            const ListKey<T> key = park[0];
#pragma unroll
            for (int u = 0; u + 1 < kPark; ++u) park[u] = park[u + 1];
            --parked;
            if (key.less(list[K - 1])) {
                if (!list[K - 1].is_empty()) rej = R::vmin(rej, list[K - 1].dist());
                list_insert<T, K>(list, key);
            } else {
                rej = R::vmin(rej, key.dist());
            }
        }
    };
    auto offer = [&](T d, typename R::index_t i, bool valid) {
        const ListKey<T> key = ListKey<T>::make(d, i);
        const bool pass = valid && key.less(list[K - 1]);
        if (valid && !pass) rej = R::vmin(rej, d);
        if (pass) {
#pragma unroll
            for (int u = 0; u < kPark; ++u) if (u == parked) park[u] = key;
            ++parked;
        }
        if (__any_sync(__activemask(), parked == kPark)) insert_round();
    };
    int r = 0;
    for (;;) {
        if (j < e) {
            // two candidates per step: both loads are in flight before either distance is needed
            const bool two = j + 1 < e;
            const Pt<T> p0 = load_pt<T>(dc.sorted + j);
            const Pt<T> p1 = load_pt<T>(dc.sorted + (two ? j + 1 : j));
            j += 2;
            const T d0 = dist2<T>(q.x, q.y, q.z, p0.x, p0.y, p0.z);
            const T d1 = dist2<T>(q.x, q.y, q.z, p1.x, p1.y, p1.z);
            offer(d0, p0.i, true);
            offer(d1, p1.i, two);
        } else {
            if (++r >= 9) break;
            // skip a row only if all of it is strictly farther than the current k-th distance
            if (!(rows.bound[r - 1][tid] > list[K - 1].dist())) { j = rows.begin[r - 1][tid]; e = rows.end[r - 1][tid]; }
        }
    }
    while (parked > 0) insert_round();
    const int ya = max(cy - 1, 0), yb = min(cy + 1, g.dim[1] - 1);
    const int za = max(cz - 1, 0), zb = min(cz + 1, g.dim[2] - 1);
    T lb = sq_gap<T>(q.x, __ldg(lo_x + xa));
    lb = R::vmin(lb, sq_gap<T>(q.x, __ldg(hi_x + xb + 1)));
    lb = R::vmin(lb, sq_gap<T>(q.y, __ldg(lo_y + ya)));
    lb = R::vmin(lb, sq_gap<T>(q.y, __ldg(hi_y + yb + 1)));
    lb = R::vmin(lb, sq_gap<T>(q.z, __ldg(lo_z + za)));
    lb = R::vmin(lb, sq_gap<T>(q.z, __ldg(hi_z + zb + 1)));
    const T worst = list[K - 1].dist();
    const bool full = !list[K - 1].is_empty();
    if (!(full && worst < lb)) {   // not provably complete within one ring: hand over to the warp pass
        sw.far_list[atomicAdd(sw.counters, 1u)] = (unsigned)t;
        return;
    }
    const long long row = (long long)q.i;
    bool tie = rej == worst;
#pragma unroll
    for (int s = 0; s < K; ++s) {
        if (s >= K - k) {
            const int c = s - (K - k);
            const T d = list[s].dist();
            sw.out_idx[row * k + c] = list[s].index();
            sw.out_dist[row * k + c] = sw.squared ? d : R::root(d);
            if (s + 1 < K) tie = tie || (d == list[s + 1].dist());
        }
    }
    if (tie) sw.tie_list[atomicAdd(sw.counters + 1, 1u)] = row;
}

}  // namespace pcu
