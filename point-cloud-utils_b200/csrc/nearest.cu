// nearest.cu -- the nearest-neighbour family: the grid build and its plan, k nearest neighbours, the fused k = 1
// statistics (Chamfer, Hausdorff) and their witness replay, prepared clouds, batched Chamfer, normals, Poisson-disk
// downsampling, algebraic point set surfaces, and their device and host C entry points.
//
// It owns no algorithmic decisions that depend on the data: grid shapes, far-query lists and tie lists are produced
// and consumed on the device, so a device-pointer call enqueues a fixed sequence of launches and returns without
// synchronising.
#include "runtime.cuh"
#include "grid.cuh"
#include "search.cuh"
#include "nn1.cuh"
#include "topk.cuh"
#include "pyramid.cuh"
#include "kdreplay.cuh"
#include "normals.cuh"
#include "apss.cuh"
#include "poisson.cuh"

using namespace pcu;
using namespace pcu_internal;

namespace {

// Descriptor-taking kernels exist in two flavours: descriptors by value in parameter space (single
// pair: `plan.by_value`) or in a device array (batches).  K<T, CloudsX<T>, SweepsX<T>[, extra...]>.
#define PCU_LAUNCH_CS(K, grid, block, ...)                                                                                   \
    PCU_TRY(plan.by_value                                                                                                    \
                ? launch_pdl(K<T, CloudsVal<T>, SweepsVal<T>, ##__VA_ARGS__>, grid, block, 0, stream, plan.cv, plan.sv) \
                : launch_pdl(K<T, CloudsPtr<T>, SweepsPtr<T>, ##__VA_ARGS__>, grid, block, 0, stream, plan.cp, plan.sp))

// Per-field byte strides between consecutive pairs of a batch (side 0 = first cloud of each pair,
// side 1 = second cloud; direction 0 = first -> second, direction 1 = second -> first).
struct CloudStrides { size_t raw, sorted, rank, part, slab_count, slab_base, slab_hist, cell_start, grid, wall_lo, wall_hi, bbox_partial, scan_state, scan_ticket, occupied, pyramid, shape; };
struct SweepStrides { size_t out_dist, out_idx, partial, far_list, vfar_list, counters, tie_list; };

template <typename U>
__device__ __forceinline__ U* advance(U* p, size_t bytes) {
    return p ? reinterpret_cast<U*>(reinterpret_cast<unsigned char*>(const_cast<typename std::remove_const<U>::type*>(p)) + bytes) : p;
}

// Writes the cloud / sweep descriptors of every pair of a batch.  They are generated on the device
// from two prototypes, so a call never stages descriptors through host memory that a later call
// could overwrite while this one is still queued.
template <typename T>
struct DescriptorArgs {
    Cloud<T> cloud[2];
    Sweep<T> sweep[2];
    CloudStrides cs[2];
    SweepStrides ss[2];
    long long batch;
    int nsweeps;
    pcu_b200_nn_stats* stats;
    T* value_out;   // per-pair Chamfer values (bidirectional calls), or null
};

template <typename T>
__global__ void descriptors_kernel(const __grid_constant__ DescriptorArgs<T> a, Cloud<T>* clouds, Sweep<T>* sweeps) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.batch) return;
    for (int s = 0; s < 2; ++s) {
        Cloud<T> c = a.cloud[s];
        const CloudStrides& st = a.cs[s];
        c.raw = advance(c.raw, p * st.raw);
        c.sorted = advance(c.sorted, p * st.sorted);
        c.rank = advance(c.rank, p * st.rank);
        c.part = advance(c.part, p * st.part);
        c.slab_count = advance(c.slab_count, p * st.slab_count);
        c.slab_base = advance(c.slab_base, p * st.slab_base);
        c.slab_hist = advance(c.slab_hist, p * st.slab_hist);
        c.cell_start = advance(c.cell_start, p * st.cell_start);
        c.grid = advance(c.grid, p * st.grid);
        c.wall_lo = advance(c.wall_lo, p * st.wall_lo);
        c.wall_hi = advance(c.wall_hi, p * st.wall_hi);
        c.bbox_partial = advance(c.bbox_partial, p * st.bbox_partial);
        c.scan_state = advance(c.scan_state, p * st.scan_state);
        c.scan_ticket = advance(c.scan_ticket, p * st.scan_ticket);
        c.occupied = advance(c.occupied, p * st.occupied);
        if (p != 0) c.hint_out = nullptr;   // the first pair of a batch speaks for all of them
        c.pyramid = advance(c.pyramid, p * st.pyramid);
        c.shape = advance(c.shape, p * st.shape);
        clouds[2 * p + s] = c;
    }
    for (int d = 0; d < a.nsweeps; ++d) {
        Sweep<T> w = a.sweep[d];
        const SweepStrides& st = a.ss[d];
        w.qcloud = (int)(2 * p + d);
        w.dcloud = (int)(2 * p + 1 - d);
        w.out_dist = advance(w.out_dist, p * st.out_dist);
        w.out_idx = advance(w.out_idx, p * st.out_idx);
        w.partial = advance(w.partial, p * st.partial);
        w.far_list = advance(w.far_list, p * st.far_list);
        w.vfar_list = advance(w.vfar_list, p * st.vfar_list);
        w.counters = advance(w.counters, p * st.counters);
        w.tie_list = advance(w.tie_list, p * st.tie_list);
        w.stats = a.stats ? a.stats + p * a.nsweeps + d : nullptr;
        w.pair_stats = a.stats ? a.stats + p * a.nsweeps : nullptr;
        w.pair_ticket = advance(a.sweep[0].counters, p * a.ss[0].counters) + 4;
        w.value_out = (a.nsweeps == 2 && a.value_out) ? a.value_out + p : nullptr;
        sweeps[p * a.nsweeps + d] = w;
    }
}

}  // namespace

// A cloud binned once (pcu_b200_cloud_prepare_*): its cell-sorted points, cell table, grid header, wall tables and
// pyramid buffers live in one private device block, described by the same Cloud<T> record the kernels take.
struct pcu_b200_cloud {
    int device = 0;
    int is_f64 = 0;
    long long n = 0;
    unsigned char* block = nullptr;
    size_t bytes = 0;
    Cloud<float> desc32{};
    Cloud<double> desc64{};
    const void* raw = nullptr;   // the handle's own copy of the caller's (n, 3) array (inside block)
    int knn_k = 1;               // the k the cell size was chosen for
    int leaf = 0;                // > 0: the block also holds the reference-tree replica built with this leaf size
    KdReplayBuffers<float> kd32{};
    KdReplayBuffers<double> kd64{};
};
template <typename T> KdReplayBuffers<T>& cloud_tree(pcu_b200_cloud* c);
template <> KdReplayBuffers<float>& cloud_tree<float>(pcu_b200_cloud* c) { return c->kd32; }
template <> KdReplayBuffers<double>& cloud_tree<double>(pcu_b200_cloud* c) { return c->kd64; }

namespace {

int cell_cap_for(long long n, double occupancy) {
    double c = (double)n / occupancy;
    if (c < 1.0) c = 1.0;
    if (c > (double)(1 << 27)) c = (double)(1 << 27);
    return (int)c;
}

float occupancy_for(const pcu_b200_workspace* ws, int k) {
    if (ws->opts.cell_occupancy > 0.f) return ws->opts.cell_occupancy;
    // k = 1: 1.5 points per cell (on C3 the sweep then visits fewer candidates while the scan over more cells and the
    // far pass grow by less; 1.0 leaves too many queries to the far pass)
    if (k <= 1) return 1.5f;
    // k > 1 (thread-per-query lists), chosen on 2 x 10^6 queries against 10^6 uniform points (tools/knn_occupancy.py):
    // fewer points per cell mean fewer candidates in the 27 cells but more queries left to the slow warp pass; the
    // trade-off is 3 at k = 4, 4 at k = 8, 7 at k = 16, 12 at k = 32.  Piecewise linear through those points.
    static const float ks[] = {2.f, 4.f, 8.f, 16.f, 32.f}, occ[] = {2.f, 3.f, 4.f, 7.f, 12.f};
    const float kf = (float)k;
    if (kf <= ks[0]) return occ[0];
    for (int i = 1; i < 5; ++i)
        if (kf <= ks[i]) return occ[i - 1] + (occ[i] - occ[i - 1]) * (kf - ks[i - 1]) / (ks[i] - ks[i - 1]);
    return 0.375f * kf;     // k > 32: the generic pyramid path, same slope as the last segment
}

// What one call works on: `batch` independent pairs (first cloud: n points, second: m points).
template <typename T>
struct PlanSpec {
    long long batch = 1;
    const T* a = nullptr;   // (batch, n, 3)
    const T* b = nullptr;   // (batch, m, 3)
    long long n = 0, m = 0;
    int nsweeps = 1;        // 1: first -> second;  2: both directions
    int k = 1;
    int squared = 0;
    bool want_stats = false;
    bool want_out = false;
    float occupancy = 2.f;
    float cell_mult[2] = {1.f, 1.f};   // grid refinement from the previous call's fill statistics
    unsigned* hint_dev = nullptr;      // 2 x 4 words of host-mapped memory, or null
    int binning = 0;                // pcu_b200_options::binning
    bool prepared_second = false;   // the second cloud is a pcu_b200_cloud: its descriptor replaces the carved one, it is not binned
    T* out_dist = nullptr;          // want_out (batch == 1)
    long long* out_idx = nullptr;
    pcu_b200_nn_stats* stats = nullptr;   // caller's device buffer, or null -> carved from the arena
    T* value_out = nullptr;               // per-pair Chamfer values (nsweeps == 2), or null
    long long replay_points = 0;
    int sm_count = 0;                     // the device's SMs (prepare_plan): sizes the far pass
};

// Scratch layout of one call.  Every per-cloud / per-sweep buffer is an array over the batch with
// a uniform stride, so descriptors can be generated on the device.
template <typename T>
struct Plan {
    DescriptorArgs<T> args{};
    Cloud<T>* d_clouds = nullptr;
    Sweep<T>* d_sweeps = nullptr;
    bool by_value = false;        // single pair: descriptors travel in kernel-parameter space
    CloudsVal<T> cv{};
    SweepsVal<T> sv{};
    CloudsPtr<T> cp{};
    SweepsPtr<T> sp{};
    pcu_b200_nn_stats* d_stats = nullptr;
    unsigned char* zero_begin = nullptr;   // zeroed per call: [cell counters | scan states, tickets, sweep counters]
    size_t zero_bytes = 0;
    size_t zero_cells_bytes = 0;           // leading part that only the multi-launch grid build needs zeroed
    bool one_cta_binning = false;          // bin_small_kernel instead of the five grid-wide passes
    bool slab_build = false;               // slab_hist / slab_partition / slab_sort instead of the cell-wise passes
    int max_slabs = 1, max_slab_chunks = 1;
    size_t slab_hist_smem = 0, slab_part_smem = 0, slab_sort_smem = 0;   // dynamic shared memory of the slab kernels
    long long max_n = 0;
    int max_cap = 0;
    int max_bbox_blocks = 1;
    int far_blocks = 1;
    int nclouds = 0, nsweeps_total = 0;
    KdReplayBuffers<T> replay{};

    template <typename U>
    static U* take_strided(Carver& cv, size_t count_per_item, long long batch, size_t& stride_bytes) {
        stride_bytes = align_up(count_per_item * sizeof(U));
        return reinterpret_cast<U*>(cv.take<unsigned char>(stride_bytes * (size_t)batch));
    }

    // Carves (or, with a null base, just measures) the layout.
    void layout(Carver& cv, const PlanSpec<T>& sp) {
        const long long B = sp.batch;
        nclouds = (int)(2 * B);
        nsweeps_total = (int)(B * sp.nsweeps);
        d_clouds = cv.take<Cloud<T>>((size_t)nclouds);
        d_sweeps = cv.take<Sweep<T>>((size_t)nsweeps_total);
        d_stats = sp.stats ? sp.stats : (sp.want_stats ? cv.take<pcu_b200_nn_stats>((size_t)nsweeps_total) : nullptr);
        args = DescriptorArgs<T>{};
        args.batch = B;
        args.nsweeps = sp.nsweeps;
        args.stats = sp.want_stats ? d_stats : nullptr;
        args.value_out = sp.value_out;
        const long long sizes[2] = {sp.n, sp.m};
        const T* raws[2] = {sp.a, sp.b};
        max_n = std::max(sp.n, sp.m);
        max_cap = 0;
        max_bbox_blocks = 1;
        // far pass (warp-stride loop over the far list): two CTAs per SM over all sweeps, at least four per sweep
        far_blocks = (int)std::max<long long>(4, 2LL * sp.sm_count / std::max<long long>(1, B * sp.nsweeps));
        // zeroed region first: cell counters and sweep counters
        const size_t zero_from = cv.off;
        for (int s = 0; s < 2; ++s) {
            Cloud<T>& cl = args.cloud[s];
            cl.raw = raws[s];
            cl.n = sizes[s];
            cl.cell_cap = cell_cap_for(sizes[s], sp.occupancy / sp.cell_mult[s]);
            cl.hint_out = sp.hint_dev ? sp.hint_dev + 8 * s : nullptr;
            cl.stride = std::min(kMaxGridDim, cl.cell_cap) + 1;
            cl.bbox_blocks = (int)std::min<long long>(kMaxBBoxBlocks, std::max<long long>(1, (3 * sizes[s] + 2 * kThreads * kBBoxPerThread - 1) / (2 * kThreads * kBBoxPerThread)));
            max_bbox_blocks = std::max(max_bbox_blocks, cl.bbox_blocks);
            args.cs[s].raw = (size_t)3 * sizes[s] * sizeof(T);
            cl.cell_start = take_strided<unsigned>(cv, (size_t)cl.cell_cap + 1, B, args.cs[s].cell_start);
            max_cap = std::max(max_cap, cl.cell_cap);
        }
        zero_cells_bytes = cv.off - zero_from;
        // One CTA per cloud when the counters fit in shared memory and the clouds are small: five dependent
        // launches then cost more than one CTA's serial passes (tools/binning_time.py compares the two; at 65536
        // points one SM takes longer than the grid-wide passes, so larger clouds keep the grid-wide passes
        // whatever the batch size).
        const bool fits = max_cap + 1 <= kSmallMaxCells && max_n <= kSmallMaxPoints;
        one_cta_binning = !sp.prepared_second && fits && (sp.binning == 2 || (sp.binning == 0 && max_n <= 8192));
        // The slab build for batches and for single pairs above 65536 points: below that, one pair's cell-wise
        // passes are a few microseconds faster (tools/binning_time.py; DESIGN.md §4).
        slab_build = !one_cta_binning && (sp.binning == 3 || (sp.binning == 0 && (B > 1 || max_n > 65536)));
        max_slabs = max_slab_chunks = 1;
        slab_part_smem = 0;
        int max_slab_cells = 1;
        for (int s = 0; s < 2; ++s) {
            Cloud<T>& cl = args.cloud[s];
            cl.scan_state = take_strided<unsigned long long>(cv, ((size_t)cl.cell_cap + 1 + kScanTile - 1) / kScanTile + 1, B,
                                                             args.cs[s].scan_state);
            cl.scan_ticket = take_strided<unsigned>(cv, 3, B, args.cs[s].scan_ticket);
            cl.occupied = take_strided<unsigned>(cv, 1, B, args.cs[s].occupied);
            if (slab_build) {
                // a slab holds kSlabMeanFill of the staging buffer on average, and at most kSlabMaxCells cells
                const long long per_slab = (long long)(kSlabMeanFill * kSlabStageBytes) / (long long)sizeof(Pt<T>);
                const long long want = std::max((sizes[s] + per_slab - 1) / per_slab, ((long long)cl.cell_cap + kSlabMaxCells - 1) / kSlabMaxCells);
                cl.slabs = (int)std::min<long long>(kMaxSlabs, std::max(1LL, want));
                cl.slab_chunks = (int)std::min<long long>(kMaxSlabChunks, (sizes[s] + kSlabChunkPoints - 1) / kSlabChunkPoints);
                cl.slab_count = take_strided<unsigned>(cv, (size_t)cl.slabs, B, args.cs[s].slab_count);
                max_slabs = std::max(max_slabs, cl.slabs);
                max_slab_chunks = std::max(max_slab_chunks, cl.slab_chunks);
                max_slab_cells = std::max(max_slab_cells, (cl.cell_cap + cl.slabs - 1) / cl.slabs);
                slab_part_smem = std::max(slab_part_smem, pcu::slab_part_smem<T>(cl.slabs));
            }
        }
        slab_hist_smem = pcu::slab_hist_smem<T>(max_slabs);
        slab_sort_smem = (size_t)kSlabStageBytes + (size_t)max_slab_cells * sizeof(unsigned);
        for (int d = 0; d < sp.nsweeps; ++d)
            args.sweep[d].counters = take_strided<unsigned>(cv, 8, B, args.ss[d].counters);
        zero_begin = cv.base ? cv.base + zero_from : nullptr;
        zero_bytes = cv.off - zero_from;
        for (int s = 0; s < 2; ++s) {
            Cloud<T>& cl = args.cloud[s];
            CloudStrides& st = args.cs[s];
            cl.sorted = take_strided<Pt<T>>(cv, (size_t)cl.n, B, st.sorted);
            if (slab_build) {
                cl.part = take_strided<Pt<T>>(cv, (size_t)cl.n, B, st.part);
                cl.slab_base = take_strided<unsigned>(cv, (size_t)cl.slabs + 1, B, st.slab_base);
                cl.slab_hist = take_strided<unsigned>(cv, (size_t)cl.slab_chunks * cl.slabs, B, st.slab_hist);
            } else {
                cl.rank = take_strided<unsigned>(cv, (size_t)cl.n, B, st.rank);
            }
            cl.grid = take_strided<GridHeader<T>>(cv, 1, B, st.grid);
            cl.wall_lo = take_strided<T>(cv, (size_t)3 * cl.stride, B, st.wall_lo);
            cl.wall_hi = take_strided<T>(cv, (size_t)3 * cl.stride, B, st.wall_hi);
            cl.bbox_partial = take_strided<T>(cv, (size_t)cl.bbox_blocks * 6, B, st.bbox_partial);
            cl.pyramid = take_strided<unsigned>(cv, (size_t)cl.cell_cap + 64, B, st.pyramid);
            cl.shape = take_strided<PyramidShape>(cv, 1, B, st.shape);
        }
        for (int d = 0; d < sp.nsweeps; ++d) {
            Sweep<T>& sw = args.sweep[d];
            SweepStrides& st = args.ss[d];
            sw.k = sp.k;
            sw.squared = sp.squared;
            const long long nq = sizes[d];
            sw.main_blocks = (int)((nq + kThreads - 1) / kThreads);
            sw.far_blocks = far_blocks;
            sw.far_list = take_strided<unsigned>(cv, (size_t)nq, B, st.far_list);
            sw.vfar_list = take_strided<unsigned>(cv, (size_t)nq, B, st.vfar_list);
            if (sp.want_out) {
                sw.tie_list = take_strided<long long>(cv, (size_t)nq, B, st.tie_list);
                sw.out_dist = sp.out_dist;   // batch == 1 on this path
                sw.out_idx = sp.out_idx;
            }
            if (sp.want_stats)
                sw.partial = take_strided<SweepPartial<T>>(cv, (size_t)sw.main_blocks + 2 * far_blocks, B, st.partial);
        }
        if (sp.replay_points > 0) replay.carve(cv, sp.replay_points);
        // descriptor sources
        this->cp.p = d_clouds;
        this->sp.p = d_sweeps;
        by_value = B == 1;
        if (by_value) {
            for (int s = 0; s < 2; ++s) this->cv.v[s] = args.cloud[s];
            for (int d = 0; d < sp.nsweeps; ++d) {
                Sweep<T> w = args.sweep[d];
                w.qcloud = d; w.dcloud = 1 - d;
                w.stats = args.stats ? args.stats + d : nullptr;
                w.pair_stats = args.stats;
                w.pair_ticket = args.sweep[0].counters + 4;
                w.value_out = (sp.nsweeps == 2) ? args.value_out : nullptr;
                this->sv.v[d] = w;
            }
        }
    }
};

template <typename T>
int upload_descriptors(Plan<T>& plan, cudaStream_t stream) {
    if (plan.by_value) return PCU_B200_OK;   // nothing to upload: descriptors ride along with every launch
    const unsigned blocks = (unsigned)((plan.args.batch + 127) / 128);
    PCU_LAUNCH(descriptors_kernel<T>, blocks, 128, stream, plan.args, plan.d_clouds, plan.d_sweeps);
    return PCU_B200_OK;
}

// Grid-sizing feedback.  A grid sized for `occupancy` points per cell of the bounding BOX fills only a
// few of its cells when the cloud is a surface (or any thin set), and those hold many points each, so
// every query wades through long candidate runs.  The binning kernels report how many cells were
// non-empty; when the same shapes come again on this workspace (a loss evaluated every iteration, a
// benchmark loop) and the non-empty cells held well over the target, the grid gets more cells --
// assuming the non-empty count grows like h^-2 (a surface), so r times fewer points per non-empty cell
// cost r^1.5 times more cells -- up to 32 times the default; a refined grid that turns out too fine for
// the data it now sees (few points per non-empty cell, or many queries left unsettled by their 27
// cells) shrinks again.  Box-filling clouds never trigger it
// (uniform data sits at 0.9 of the threshold), results never depend on it.
template <typename T>
void apply_grid_feedback(pcu_b200_workspace* ws, PlanSpec<T>& spec) {
    const long long key[5] = {spec.n, spec.m, spec.k, (long long)sizeof(T), spec.batch};
    if (!ws->hint_host) return;
    bool same = true;
    for (int i = 0; i < 5; ++i) same = same && key[i] == ws->hint_key[i];
    if (!same) {
        for (int i = 0; i < 5; ++i) ws->hint_key[i] = key[i];
        ws->cell_mult[0] = ws->cell_mult[1] = 1.f;
        ws->cell_mult_ceiling[0] = ws->cell_mult_ceiling[1] = 32.f;
        for (int i = 0; i < 16; ++i) ws->hint_host[i] = 0u;
    } else {
        const long long sizes[2] = {spec.n, spec.m};
        for (int s = 0; s < 2; ++s) {
            volatile unsigned* h = ws->hint_host + 8 * s;
            const unsigned cap = h[0], nonempty = h[1], pts = h[2], valid = h[3];
            if (!valid || nonempty == 0u || pts != (unsigned)sizes[s]) continue;
            if (cap != (unsigned)cell_cap_for(sizes[s], spec.occupancy / ws->cell_mult[s])) continue;   // measured under another grid
            const double per_cell = (double)pts / (double)nonempty;
            const double r = per_cell / (1.3 * (double)spec.occupancy);
            // share of the queries searched against this cloud that the 3 x 3 x 3 cells could not settle:
            // many of them means the cells are too fine for where the queries are (or the clouds are far
            // apart), and finer cells only deepen the slow passes
            const double far_share = (h[6] && h[5]) ? (double)h[4] / (double)h[5] : 0.0;
            double m = (double)ws->cell_mult[s];
            if (far_share > 0.05) {
                if (m > 1.0) ws->cell_mult_ceiling[s] = (float)std::max(1.0, 0.6 * m);   // do not come back up here
                m *= 0.35;
            } else if (r > 1.6) m *= r * std::sqrt(r);                             // dead band 0.8 .. 1.6
            else if (r < 0.8) m *= (r / 0.8) * std::sqrt(r / 0.8);
            m = std::min((double)ws->cell_mult_ceiling[s], m);
            ws->cell_mult[s] = m < 1.5 ? 1.f : (float)m;
            h[3] = 0u; h[6] = 0u;   // consumed
        }
    }
    spec.cell_mult[0] = ws->cell_mult[0];
    spec.cell_mult[1] = ws->cell_mult[1];
    spec.hint_dev = ws->hint_dev;
}

template <typename T>
int prepare_plan(pcu_b200_workspace* ws, Plan<T>& plan, PlanSpec<T>& spec, cudaStream_t stream) {
    apply_grid_feedback(ws, spec);
    spec.sm_count = ws->sm_count;
    return carve_scratch(ws, kArena, stream, [&](Carver& cv) { plan.layout(cv, spec); });
}

// Kernels whose dynamic shared-memory limit is raised above the default, one group of four bits each in
// pcu_b200_workspace::smem_raised.
enum SmemKernel { kSmemBinSmall, kSmemSlabHist, kSmemSlabPartition, kSmemSlabSort };

// Raises the dynamic shared-memory limit of `kernel` (kernel `which`, instantiated for Clouds<T>) to `bytes`, once per
// workspace: bit 4 * which + 2 * (T is double) + (Clouds is CloudsVal) of ws->smem_raised records that it is done.
template <template <typename> class Clouds, typename T>
int raise_smem_limit(pcu_b200_workspace* ws, SmemKernel which, void (*kernel)(Clouds<T>), size_t bytes) {
    const unsigned bit = 1u << (4 * which + (sizeof(T) == 8 ? 2 : 0) + (std::is_same<Clouds<T>, CloudsVal<T>>::value ? 1 : 0));
    if (!(ws->smem_raised & bit)) {
        PCU_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        ws->smem_raised |= bit;
    }
    return PCU_B200_OK;
}

// bbox -> grid -> cell order of `clouds` (gridDim.y = ny) by the slab build or the cell-wise passes, each stage
// followed by its mark.  Descriptors by value take the bounding box and the grid set-up in one launch
// (bbox_partial_kernel's kSetup); descriptors in a device array (batches) set up their grids in a launch of its own.
template <typename T, typename CS>
int launch_grid_build(pcu_b200_workspace* ws, const Plan<T>& plan, const CS& clouds, unsigned ny, cudaStream_t stream) {
    constexpr bool by_value = std::is_same<CS, CloudsVal<T>>::value;
    PCU_TRY(launch_pdl(bbox_partial_kernel<T, CS, by_value>, dim3(plan.max_bbox_blocks, ny), kThreads, 0, stream, clouds));
    if constexpr (!by_value) PCU_TRY(launch_pdl(grid_setup_kernel<T, CS>, dim3(1, ny), kThreads, 0, stream, clouds));
    mark(ws, 2, stream);
    if (plan.slab_build) {
        const size_t part_most = std::max(slab_part_smem<T>(kMaxSlabs), slab_part_smem<T>(kSlabTile));
        PCU_TRY(raise_smem_limit(ws, kSmemSlabHist, slab_hist_kernel<T, CS>, slab_hist_smem<T>(kMaxSlabs)));
        PCU_TRY(raise_smem_limit(ws, kSmemSlabPartition, slab_partition_kernel<T, CS>, part_most));
        PCU_TRY(raise_smem_limit(ws, kSmemSlabSort, slab_sort_kernel<T, CS>, (size_t)kSlabStageBytes + kSlabMaxCells * sizeof(unsigned)));
        const dim3 chunks((unsigned)plan.max_slab_chunks, ny), slabs((unsigned)plan.max_slabs, ny);
        PCU_TRY(launch_pdl(slab_hist_kernel<T, CS>, chunks, kSlabThreads, plan.slab_hist_smem, stream, clouds));
        mark(ws, 3, stream);
        PCU_TRY(launch_pdl(slab_partition_kernel<T, CS>, chunks, kSlabThreads, plan.slab_part_smem, stream, clouds));
        mark(ws, 4, stream);
        PCU_TRY(launch_pdl(slab_sort_kernel<T, CS>, slabs, kSlabThreads, plan.slab_sort_smem, stream, clouds));
        mark(ws, 5, stream);
        return PCU_B200_OK;
    }
    const unsigned bin_blocks = (unsigned)((plan.max_n + kThreads - 1) / kThreads);
    const unsigned scan_blocks = (unsigned)(((long long)plan.max_cap + 1 + kScanTile - 1) / kScanTile);
    PCU_TRY(launch_pdl(cell_count_kernel<T, CS>, dim3(bin_blocks, ny), kThreads, 0, stream, clouds));
    mark(ws, 3, stream);
    PCU_TRY(launch_pdl(scan_lookback_kernel<T, CS>, dim3(scan_blocks, ny), kScanThreads, 0, stream, clouds));
    mark(ws, 4, stream);
    PCU_TRY(launch_pdl(scatter_kernel<T, CS>, dim3(bin_blocks, ny), kThreads, 0, stream, clouds));
    mark(ws, 5, stream);
    return PCU_B200_OK;
}

// bbox -> grid -> cell order (slab build, cell-wise passes or one CTA per cloud) for every cloud of the plan
// `ready` (host entry points, single pairs): two events, recorded on the copy stream when the first / the second
// cloud has arrived on the device.  The first cloud is then binned -- all five passes -- while the second is
// still crossing PCIe, and only the second cloud's passes follow its copy.
// `between` (host entry points; may be null): host work to do once the first cloud's passes have been enqueued and
// before the second cloud's `ready` event is waited for -- the staged copy of the second cloud, which keeps the host
// busy, so that the GPU bins the first cloud meanwhile.  It records ready[1] itself.
template <typename T>
int enqueue_binning(pcu_b200_workspace* ws, const Plan<T>& plan, cudaStream_t stream, const cudaEvent_t* ready = nullptr,
                    bool first_only = false, const std::function<int()>* between = nullptr) {
    // one cloud after the other (single pairs whose clouds arrive one by one, or whose second cloud is prepared)
    const bool per_cloud = (ready != nullptr || first_only) && plan.by_value && !plan.one_cta_binning;
    if (!per_cloud) {
        if (between != nullptr) PCU_TRY((*between)());   // the other build paths take both clouds at once
        if (ready != nullptr) {
            PCU_CUDA(cudaStreamWaitEvent(stream, ready[0], 0));
            if (!first_only) PCU_CUDA(cudaStreamWaitEvent(stream, ready[1], 0));
        }
    }
    // the cell-wise passes count into cell_start; the other builds write every entry of it and need only the
    // counters after it zeroed
    const size_t zero_skip = plan.slab_build || plan.one_cta_binning ? plan.zero_cells_bytes : 0;
    PCU_CUDA(cudaMemsetAsync(plan.zero_begin + zero_skip, 0, plan.zero_bytes - zero_skip, stream));
    if (plan.one_cta_binning) {
        const size_t smem = ((size_t)plan.max_cap + 1) * sizeof(unsigned), most = (size_t)kSmallMaxCells * sizeof(unsigned);
        if (plan.by_value) {
            PCU_TRY(raise_smem_limit(ws, kSmemBinSmall, bin_small_kernel<T, CloudsVal<T>>, most));
            PCU_TRY(launch_pdl(bin_small_kernel<T, CloudsVal<T>>, dim3(plan.nclouds), kSmallThreads, smem, stream, plan.cv));
        } else {
            PCU_TRY(raise_smem_limit(ws, kSmemBinSmall, bin_small_kernel<T, CloudsPtr<T>>, most));
            PCU_TRY(launch_pdl(bin_small_kernel<T, CloudsPtr<T>>, dim3(plan.nclouds), kSmallThreads, smem, stream, plan.cp));
        }
        for (int stage = 2; stage <= 5; ++stage) mark(ws, stage, stream);   // the whole build shows up as "bbox+grid"
        return PCU_B200_OK;
    }
    if (!per_cloud) {
        const unsigned ny = (unsigned)plan.nclouds;
        return plan.by_value ? launch_grid_build(ws, plan, plan.cv, ny, stream) : launch_grid_build(ws, plan, plan.cp, ny, stream);
    }
    for (int s = 0; s < (first_only ? 1 : 2); ++s) {   // first_only: the second cloud is a prepared one
        if (s == 1 && between != nullptr) PCU_TRY((*between)());
        if (ready != nullptr) PCU_CUDA(cudaStreamWaitEvent(stream, ready[s], 0));
        CloudsVal<T> one;
        one.v[0] = plan.cv.v[s];
        one.v[1] = plan.cv.v[s];
        PCU_TRY(launch_grid_build(ws, plan, one, 1, stream));
    }
    if (first_only && between != nullptr) PCU_TRY((*between)());
    return PCU_B200_OK;
}

template <typename T>
int check_cloud_args(const void* a, long long n, const void* b, long long m) {
    if (!a || !b) return fail(PCU_B200_INVALID_ARGUMENT, "null point-cloud pointer");
    if (n <= 0 || m <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT,
                    "Invalid input set with zero elements: both clouds must have shape (n, 3) with n > 0 "
                    "(got %lld and %lld rows)", n, m);
    // rows, cell prefixes and list entries are 32-bit throughout the pipeline, whatever the coordinate type
    const long long lim = 0x7fffffffLL;
    if (n >= lim || m >= lim)
        return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld, %lld rows; at most 2^31 - 2 are supported)", n, m);
    return PCU_B200_OK;
}

template <typename T> const Cloud<T>& cloud_desc(const pcu_b200_cloud* c);
template <> const Cloud<float>& cloud_desc<float>(const pcu_b200_cloud* c) { return c->desc32; }
template <> const Cloud<double>& cloud_desc<double>(const pcu_b200_cloud* c) { return c->desc64; }

// ---- fused k = 1 statistics -------------------------------------------------------------------
// nsweeps == 1: query -> dataset.  nsweeps == 2: x -> y and y -> x over the same two binned clouds.

template <typename T>
int stats_device(pcu_b200_workspace* ws, const T* a, long long n, const T* b, long long m, bool both,
                 pcu_b200_nn_stats* out_stats, T* out_value, cudaStream_t stream, const cudaEvent_t* ready = nullptr,
                 const pcu_b200_cloud* prepared = nullptr, const std::function<int()>* between = nullptr) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (prepared != nullptr) {
        if (prepared->is_f64 != (sizeof(T) == 8 ? 1 : 0)) return fail(PCU_B200_INVALID_ARGUMENT, "the prepared cloud has another precision than the points");
        if (prepared->device != ws->device) return fail(PCU_B200_INVALID_ARGUMENT, "the prepared cloud lives on device %d, the workspace on %d", prepared->device, ws->device);
        b = (const T*)prepared->raw;
        m = prepared->n;
    }
    PCU_TRY(check_cloud_args<T>(a, n, b, m));
    if (!out_stats) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    const int ns = both ? 2 : 1;
    PlanSpec<T> spec;
    spec.a = a; spec.n = n; spec.b = b; spec.m = m;
    spec.nsweeps = ns; spec.k = 1; spec.want_stats = true;
    spec.occupancy = occupancy_for(ws, 1);
    spec.binning = ws->opts.binning;
    spec.stats = out_stats;
    spec.value_out = both ? out_value : nullptr;
    spec.prepared_second = prepared != nullptr;
    Plan<T> plan;
    PCU_TRY(prepare_plan(ws, plan, spec, stream));
    if (prepared != nullptr) plan.cv.v[1] = cloud_desc<T>(prepared);   // a single pair: descriptors travel by value
    mark(ws, 0, stream);
    PCU_TRY(upload_descriptors(plan, stream));
    mark(ws, 1, stream);
    PCU_TRY(enqueue_binning(ws, plan, stream, ready, prepared != nullptr, between));
    const unsigned qblocks = (unsigned)((std::max(n, m) + kThreads - 1) / kThreads);
    PCU_LAUNCH_CS(nn1_kernel, dim3(qblocks, ns), kThreads, false, true);
    mark(ws, 6, stream);
    PCU_LAUNCH_CS(nn1_far_kernel, dim3(plan.far_blocks, ns), kThreads, false, true);
    PCU_LAUNCH_CS(nn1_vfar_kernel, dim3(plan.far_blocks, ns), kThreads, false, true);
    mark(ws, 7, stream);
    mark(ws, 8, stream);
    return PCU_B200_OK;
}

// ---- Hausdorff witness under ties ---------------------------------------------------------------
template <typename T>
int resolve_witness_device(pcu_b200_workspace* ws, const T* query, long long n, const T* dataset, long long m,
                           pcu_b200_nn_stats* stats, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(check_cloud_args<T>(query, n, dataset, m));
    if (!stats) return fail(PCU_B200_INVALID_ARGUMENT, "null stats pointer");
    PCU_ON_DEVICE(ws);
    // the arena is re-carved in stream order: the sweep that produced `stats` has been enqueued before us
    KdReplayBuffers<T> rb;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { rb.carve(cv, m); }));
    const int leaf = ws->opts.max_points_per_leaf > 0 ? ws->opts.max_points_per_leaf : 10;
    const int rs = enqueue_witness_replay<T>(rb, query, n, dataset, m, leaf, stats, stream, g_launches);
    if (rs != PCU_B200_OK) return fail(rs, "witness replay failed: %s", cudaGetErrorString(cudaGetLastError()));
    return PCU_B200_OK;
}

// ---- normals from k nearest neighbours (SURVEY.md 8f N1) -------------------------------------------
// Self-query top-k (the point itself is its own first neighbour, as in the reference), plane fit, optional
// orientation / filtering by view directions, order-preserving compaction of the kept points.
template <typename T>
int normals_knn_device(pcu_b200_workspace* ws, const T* points, long long n, const T* view_dirs, int k,
                       double drop_angle_threshold, long long* out_idx, T* out_normals, long long* out_count,
                       cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid number of neighbors (%d) must be greater than 0.", k);
    if (!points || n <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid point set with zero elements: points must have shape (n, 3) (got %lld rows)", n);
    if (!out_idx || !out_normals || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    long long* nn_idx; T *nn_dist, *dense; unsigned char* keep; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        nn_idx = cv.take<long long>((size_t)n * k);
        nn_dist = cv.take<T>((size_t)n * k);
        dense = cv.take<T>((size_t)3 * n);
        keep = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_TRY(knn_device<T>(ws, points, n, points, n, k, 1, nn_dist, nn_idx, nullptr, stream));
    PCU_LAUNCH((normals_knn_kernel<T>), blocks_for(n), kThreads, stream, points, n, nn_idx, k, view_dirs, drop_angle_threshold, dense, keep);
    PCU_TRY(enqueue_keep_offsets(keep, n, counts, out_count, stream));
    PCU_LAUNCH((keep_scatter_kernel<T>), blocks_for(n), kThreads, stream, keep, n, counts, dense, out_idx, out_normals);
    return PCU_B200_OK;
}

// A call that bins one cloud: the plan of an ordinary pair whose second cloud is a one-point dummy that is never binned
// (prepared_second; it also keeps the dummy out of the one-CTA build).
template <typename T>
PlanSpec<T> one_cloud_spec(const T* points, long long n, float occupancy) {
    PlanSpec<T> spec;
    spec.a = points; spec.n = n; spec.b = points; spec.m = 1;
    spec.nsweeps = 1; spec.k = 1;
    spec.occupancy = occupancy;
    spec.prepared_second = true;
    return spec;
}

// The plan, carved from the arena, of a call that bins one cloud into cells no finer than `min_cell`.
template <typename T>
int single_cloud_plan(pcu_b200_workspace* ws, const T* points, long long n, double min_cell, Plan<T>& plan, cudaStream_t stream) {
    const PlanSpec<T> spec = one_cloud_spec(points, n, 0.125f);   // the cell budget; the cell size is held up by min_cell below
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { plan.layout(cv, spec); }));
    plan.cv.v[0].min_cell = (float)std::min(1e30, min_cell);
    plan.cv.v[0].hint_out = nullptr;
    return PCU_B200_OK;
}

// ---- normals from all points in a ball (SURVEY.md 8f N1, the radius variant) ---------------------------
// The cloud is binned once (cells no finer than half the reach of the search, at most 8 per point), one thread per
// point walks the cells its ball touches; the compaction is the k-NN variant's.
template <typename T>
int normals_ball_device(pcu_b200_workspace* ws, const T* points, long long n, const T* view_dirs, const pcu_b200_ball_options* o,
                        long long* out_idx, T* out_normals, long long* out_count, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!o) return fail(PCU_B200_INVALID_ARGUMENT, "null options");
    // the checks of the binding, src/point_cloud_normals.cpp:316-327
    if (!(o->radius > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid radius (%f) must be greater than 0.", o->radius);
    if (o->min_pts_per_ball < 3) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid min_pts_per_ball (%d) must be greater than 3.", o->min_pts_per_ball);
    if (o->max_pts_per_ball > 0 && o->max_pts_per_ball < 3)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid max_pts_per_ball (%d) must either be negative (no max) or a number greater than 3.", o->max_pts_per_ball);
    if (o->weight_function != 0 && o->weight_function != 1)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid weight_function, must be one of 'constant' or 'rbf'.");
    if (!points || n <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid point set with zero elements: points must have shape (n, 3) (got %lld rows)", n);
    PCU_TRY(check_cloud_args<T>(points, n, points, 1));
    if (!out_idx || !out_normals || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    const double reach = std::sqrt((double)(T)o->radius);     // the search radius is a squared distance (normals.cuh)
    Plan<T> plan;
    PCU_TRY(single_cloud_plan<T>(ws, points, n, 0.5 * reach, plan, stream));
    T* dense; unsigned char* keep; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        dense = cv.take<T>((size_t)3 * n);
        keep = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    mark(ws, 0, stream);
    mark(ws, 1, stream);
    PCU_TRY(enqueue_binning(ws, plan, stream, nullptr, true));
    BallParams bp;
    bp.radius = o->radius; bp.drop_angle_threshold = o->drop_angle_threshold;
    bp.min_pts = o->min_pts_per_ball; bp.max_pts = o->max_pts_per_ball;
    bp.weight_kind = o->weight_function; bp.seed = o->seed;
    PCU_LAUNCH((cell_order_kernel<T>), (unsigned)std::min<long long>(((long long)plan.cv.v[0].cell_cap + kThreads - 1) / kThreads, (long long)ws->sm_count * 64), kThreads, stream, plan.cv.v[0]);
    PCU_LAUNCH((normals_ball_kernel<T>), blocks_for(n), kThreads, stream, plan.cv.v[0], view_dirs, bp, dense, keep);
    mark(ws, 6, stream);
    PCU_TRY(enqueue_keep_offsets(keep, n, counts, out_count, stream));
    PCU_LAUNCH((keep_scatter_kernel<T>), blocks_for(n), kThreads, stream, keep, n, counts, dense, out_idx, out_normals);
    mark(ws, 7, stream);
    mark(ws, 8, stream);
    return PCU_B200_OK;
}

// ---- algebraic point set surfaces (pointcloud_apss_curvature, project_points_onto_apss) -----------------------------
// The points are binned as for the ball curvatures (cells no finer than r / 2, then row order within every cell), their
// unit fp64 normals are written in cell order into aux scratch, then one thread per query iterates its projection
// (apss.cuh).  Stream-ordered: no synchronisation.
template <typename T>
int apss_device(pcu_b200_workspace* ws, const T* p, const T* n, long long np, const T* q, long long nq, double r, T* out_x, T* out_n,
                T* out_kh, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!(r > 0.0) || !std::isfinite(r)) return fail(PCU_B200_INVALID_ARGUMENT, "apss: r must be finite and > 0, got %g", r);
    if (np < 0 || nq < 0) return fail(PCU_B200_INVALID_ARGUMENT, "apss: negative size (np = %lld, nq = %lld)", np, nq);
    if (!q && nq != np) return fail(PCU_B200_INVALID_ARGUMENT, "apss: without q the queries are the %lld points, got nq = %lld", np, nq);
    if (np > 0 && (!p || !n)) return fail(PCU_B200_INVALID_ARGUMENT, "null point or normal pointer");
    if (nq > 0 && !out_kh) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (nq == 0) return PCU_B200_OK;
    if (np == 0) {
        PCU_LAUNCH((apss_undetermined_kernel<T>), blocks_for(nq), kThreads, stream, nq, out_x, out_n, out_kh);
        return PCU_B200_OK;
    }
    PCU_TRY(check_cloud_args<T>(p, np, p, 1));
    Plan<T> plan;
    PCU_TRY(single_cloud_plan<T>(ws, p, np, 0.5 * r, plan, stream));
    double* nrm;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) { nrm = cv.take<double>(3 * (size_t)np); }));
    PCU_TRY(enqueue_binning(ws, plan, stream, nullptr, true));
    PCU_LAUNCH((cell_order_kernel<T>), (unsigned)std::min<long long>(((long long)plan.cv.v[0].cell_cap + kThreads - 1) / kThreads, (long long)ws->sm_count * 64), kThreads, stream, plan.cv.v[0]);
    PCU_LAUNCH((apss_normals_kernel<T>), blocks_for(np), kThreads, stream, plan.cv.v[0], n, nrm);
    PCU_LAUNCH((apss_kernel<T>), blocks_for(nq), kThreads, stream, plan.cv.v[0], (const double*)nrm, q, nq, r, out_x, out_n, out_kh);
    return PCU_B200_OK;
}

// ---- Poisson-disk downsampling (downsample_point_cloud_poisson_disk) --------------------------------------------
// The cloud is binned once (cells no finer than half the radius, as for the ball normals), then ONE cooperative launch
// runs every selection round of poisson.cuh with grid barriers between them -- the number of rounds depends on the
// data, and a barrier keeps that decision on the device without a launch per possible round -- and the kept rows are
// compacted in ascending order (compact.cuh).
template <typename T>
int poisson_grid_blocks(int device, int sm_count, long long n, unsigned* out_blocks) {
    constexpr int kMaxDevices = 64;   // co-residency limit of the cooperative launch, cached per device
    static std::atomic<int> cached[kMaxDevices];
    const int slot = device >= 0 && device < kMaxDevices ? device : 0;
    int per_sm = cached[slot].load(std::memory_order_acquire);
    if (per_sm == 0 || slot != device) {
        int fit = 0;
        PCU_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, poisson_rounds_kernel<T>, kThreads, 0));
        if (fit < 1) return fail(PCU_B200_CUDA_ERROR, "poisson_rounds_kernel cannot be resident on this device");
        per_sm = std::min(8, fit);
        cached[slot].store(per_sm, std::memory_order_release);
    }
    const long long want = (n + kThreads - 1) / kThreads;
    *out_blocks = (unsigned)std::max<long long>(1, std::min<long long>(want, (long long)per_sm * sm_count));
    return PCU_B200_OK;
}

// ---- prepared clouds ---------------------------------------------------------------------------------------
// Bins a copy of `points` once into a private block (the one-cloud plan of one_cloud_spec); the handle keeps that
// cloud's descriptor.
template <typename T>
int cloud_prepare_device(pcu_b200_workspace* ws, const T* points, long long n, pcu_b200_cloud** out, cudaStream_t stream,
                         int knn_k = 1, int leaf = 0) {
    if (!ws || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (knn_k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid value for k (%d) must be greater than 0.", knn_k);
    if (leaf < 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_points_per_leaf must be >= 0");
    PCU_TRY(check_cloud_args<T>(points, n, points, 1));
    PCU_ON_DEVICE(ws);
    pcu_b200_cloud* c = new (std::nothrow) pcu_b200_cloud();
    if (!c) return fail(PCU_B200_OUT_OF_MEMORY, "out of host memory");
    c->device = ws->device; c->is_f64 = sizeof(T) == 8 ? 1 : 0; c->n = n; c->knn_k = knn_k;
    // the block: the handle's own copy of the points, the plan that bins that copy (at the cell size the searches with
    // this k want), and with a leaf size the reference tree
    PlanSpec<T> spec = one_cloud_spec<T>(nullptr, n, occupancy_for(ws, knn_k));
    Plan<T> plan;
    T* raw_copy = nullptr;
    auto carve = [&](Carver& cv) {
        raw_copy = cv.take<T>((size_t)3 * n);
        spec.a = spec.b = raw_copy;
        plan.layout(cv, spec);
        if (leaf > 0) cloud_tree<T>(c).carve(cv, n);
    };
    const size_t bytes = carve_at(nullptr, carve);
    c->bytes = bytes;
    cudaError_t e = cudaMalloc((void**)&c->block, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        delete c;
        return fail(PCU_B200_OUT_OF_MEMORY, "cudaMalloc of %zu bytes for a prepared cloud failed: %s", bytes, cudaGetErrorString(e));
    }
    carve_at(c->block, carve);
    auto bail = [&](int status) { cudaFree(c->block); delete c; return status; };
    if (cudaMemcpyAsync(raw_copy, points, sizeof(T) * 3 * n, cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
        return bail(fail(PCU_B200_CUDA_ERROR, "copy of the points failed: %s", cudaGetErrorString(cudaGetLastError())));
    const int st = enqueue_binning(ws, plan, stream, nullptr, true);
    if (st != PCU_B200_OK) return bail(st);
    if (leaf > 0) {   // the full reference tree, once: k-NN calls against the handle only replay their tied rows on it
        KdReplayBuffers<T>& tree = cloud_tree<T>(c);
        const int ts = build_kd_replica<T>(tree, raw_copy, n, leaf, nullptr, KdPrune<T>{}, stream, g_launches);
        if (ts != PCU_B200_OK) return bail(fail(ts, "building the reference tree failed: %s", cudaGetErrorString(cudaGetLastError())));
        c->leaf = leaf;
    }
    Cloud<T> d = plan.cv.v[0];
    d.hint_out = nullptr;             // a prepared cloud takes no part in the grid-sizing feedback
    if (sizeof(T) == 8) std::memcpy(&c->desc64, &d, sizeof d); else std::memcpy(&c->desc32, &d, sizeof d);
    c->raw = raw_copy;
    *out = c;
    return PCU_B200_OK;
}

// ---- batched Chamfer ---------------------------------------------------------------------------
// out_stats (diagnostic, may be null): 2 * batch device records that receive every pair's two sweeps in place
// of the ones carved from the arena.
template <typename T>
int batched_chamfer_device(pcu_b200_workspace* ws, const T* x, const T* y, long long batch, long long n, long long m,
                           T* out_per_pair, double* out_sum, cudaStream_t stream, pcu_b200_nn_stats* out_stats = nullptr) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (batch <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "batch must be positive (got %lld)", batch);
    PCU_TRY(check_cloud_args<T>(x, n, y, m));
    if (!out_per_pair && !out_sum) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    // gridDim.y carries the cloud / sweep index: at most 65535, i.e. 32767 pairs per slice
    const long long slice = 16384;
    for (long long first = 0; first < batch; first += slice) {
        const long long B = std::min(slice, batch - first);
        PlanSpec<T> spec;
        spec.batch = B;
        spec.a = x + first * 3 * n; spec.n = n; spec.b = y + first * 3 * m; spec.m = m;
        spec.nsweeps = 2; spec.k = 1; spec.want_stats = true;
        spec.stats = out_stats ? out_stats + 2 * first : nullptr;
        spec.occupancy = occupancy_for(ws, 1);
        spec.binning = ws->opts.binning;
        Plan<T> plan;
        PCU_TRY(prepare_plan(ws, plan, spec, stream));
        mark(ws, 0, stream);
        PCU_TRY(upload_descriptors(plan, stream));
        mark(ws, 1, stream);
        PCU_TRY(enqueue_binning(ws, plan, stream));
        const unsigned qblocks = (unsigned)((std::max(n, m) + kThreads - 1) / kThreads);
        PCU_LAUNCH_CS(nn1_kernel, dim3(qblocks, plan.nsweeps_total), kThreads, false, true);
        mark(ws, 6, stream);
        PCU_LAUNCH_CS(nn1_far_kernel, dim3(plan.far_blocks, plan.nsweeps_total), kThreads, false, true);
        PCU_LAUNCH_CS(nn1_vfar_kernel, dim3(plan.far_blocks, plan.nsweeps_total), kThreads, false, true);
        mark(ws, 7, stream);
        PCU_LAUNCH(chamfer_value_kernel<T>, 1, kThreads, stream, plan.d_stats, B,
                   out_per_pair ? out_per_pair + first : (T*)nullptr, out_sum, first > 0 ? 1 : 0);
        mark(ws, 8, stream);
    }
    return PCU_B200_OK;
}

template <typename T>
int knn_host(pcu_b200_workspace* ws, const T* query, long long n, const T* dataset, long long m, int k, int squared,
             T* out_dist, long long* out_idx, long long* out_n_tied, pcu_b200_cloud* prepared = nullptr) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid value for k (%d) must be greater than 0.", k);
    if (prepared != nullptr) { dataset = query; m = 1; }   // placeholders for the checks and the staging layout: nothing of it is copied
    PCU_TRY(check_cloud_args<T>(query, n, dataset, m));
    if (!out_dist || !out_idx) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    T *dq, *dd, *od; long long *oi, *nt;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        dq = cv.take<T>((size_t)3 * n);
        dd = cv.take<T>((size_t)3 * m);
        od = cv.take<T>((size_t)n * k);
        oi = cv.take<long long>((size_t)n * k);
        nt = cv.take<long long>(1);
    }));
    mark(ws, 9, st);
    PCU_TRY(h2d(ws, dq, query, sizeof(T) * 3 * n, st));
    if (prepared == nullptr) PCU_TRY(h2d(ws, dd, dataset, sizeof(T) * 3 * m, st));
    PCU_TRY(knn_device<T>(ws, dq, n, dd, m, k, squared, od, oi, nt, st, prepared));
    PCU_CUDA(cudaMemcpyAsync(out_dist, od, sizeof(T) * n * k, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaMemcpyAsync(out_idx, oi, sizeof(long long) * n * k, cudaMemcpyDeviceToHost, st));
    long long tied = 0;
    unsigned overflows = 0;
    PCU_CUDA(cudaMemcpyAsync(&tied, nt, sizeof(long long), cudaMemcpyDeviceToHost, st));
    mark(ws, 10, st);
    if (ws->replay_overflows)
        PCU_CUDA(cudaMemcpyAsync(&overflows, ws->replay_overflows, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    if (out_n_tied) *out_n_tied = tied;
    if (tied > 0 && overflows > 0)
        return fail(PCU_B200_INTERNAL, "tie replay: the reference kd-tree of this dataset is deeper than the %d-frame walk "
                    "stack (%u walks affected); neighbour order among exactly equidistant points is not guaranteed", kKdStack, overflows);
    return PCU_B200_OK;
}

// Device-side results of one fused call, contiguous so that ONE copy brings them to the pinned slot.
template <typename T>
struct StatsResult {
    pcu_b200_nn_stats stats[2];
    T value;
};

template <typename T>
int stats_host(pcu_b200_workspace* ws, const T* a, long long n, const T* b, long long m, bool both,
               pcu_b200_nn_stats* out_stats, T* out_value, const pcu_b200_cloud* prepared = nullptr) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (prepared != nullptr) { b = a; m = 1; }   // placeholders for the checks and the staging layout: nothing of b is copied
    PCU_TRY(check_cloud_args<T>(a, n, b, m));
    if (!out_stats) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    T *da, *db; StatsResult<T>* dr;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        da = cv.take<T>((size_t)3 * n);
        db = cv.take<T>((size_t)3 * m);
        dr = cv.take<StatsResult<T>>(1);
    }));
    // the copies run on their own stream: the first cloud is binned while the second is still in flight.
    // (the staging block may have just been re-allocated in the order of `st`: the copies wait for that)
    PCU_CUDA(cudaEventRecord(ws->arrived[0], st));
    PCU_CUDA(cudaStreamWaitEvent(ws->copy_stream, ws->arrived[0], 0));
    mark(ws, 9, st);
    PCU_TRY(h2d(ws, da, a, sizeof(T) * 3 * n, ws->copy_stream));
    PCU_CUDA(cudaEventRecord(ws->arrived[0], ws->copy_stream));
    // the second cloud's copy is issued from inside the launch sequence, after the first cloud's passes have been
    // enqueued: a staged (pageable) copy keeps this thread busy while the GPU already bins the first cloud
    const std::function<int()> second_copy = [&]() -> int {
        if (prepared == nullptr) PCU_TRY(h2d(ws, db, b, sizeof(T) * 3 * m, ws->copy_stream));
        PCU_CUDA(cudaEventRecord(ws->arrived[1], ws->copy_stream));
        return PCU_B200_OK;
    };
    PCU_TRY(stats_device<T>(ws, da, n, db, m, both, dr->stats, both ? &dr->value : nullptr, st, ws->arrived, prepared, &second_copy));
    StatsResult<T>* hr = reinterpret_cast<StatsResult<T>*>(ws->host_slot);
    auto fetch = [&]() -> int {
        PCU_CUDA(cudaMemcpyAsync(hr, dr, sizeof(StatsResult<T>), cudaMemcpyDeviceToHost, st));
        mark(ws, 10, st);
        PCU_CUDA(cudaStreamSynchronize(st));
        return PCU_B200_OK;
    };
    PCU_TRY(fetch());
    // Hausdorff witnesses whose neighbour was decided by tie order: replay with the reference's tree
    if (ws->opts.disable_tie_replay != 1) {
        for (int s = 0; s < (both ? 2 : 1); ++s) {
            if (!hr->stats[s].witness_tied) continue;
            const T* second = prepared ? (const T*)prepared->raw : db;
            const long long msecond = prepared ? prepared->n : m;
            const T* qs = s == 0 ? da : second;
            const T* dsrc = s == 0 ? second : da;
            PCU_TRY(resolve_witness_device<T>(ws, qs, s == 0 ? n : msecond, dsrc, s == 0 ? msecond : n, dr->stats + s, st));
            PCU_TRY(fetch());
        }
    }
    for (int s = 0; s < (both ? 2 : 1); ++s) out_stats[s] = hr->stats[s];
    if (both && out_value) *out_value = hr->value;
    return PCU_B200_OK;
}

template <typename T>
int batched_chamfer_host(pcu_b200_workspace* ws, const T* x, const T* y, long long batch, long long n, long long m,
                         T* out_per_pair, double* out_sum) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (batch <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "batch must be positive (got %lld)", batch);
    PCU_TRY(check_cloud_args<T>(x, n, y, m));
    if (!out_per_pair) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    T *dx, *dy, *dv; double* dsum;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        dx = cv.take<T>((size_t)3 * n * batch);
        dy = cv.take<T>((size_t)3 * m * batch);
        dv = cv.take<T>((size_t)batch);
        dsum = cv.take<double>(1);
    }));
    PCU_TRY(h2d(ws, dx, x, sizeof(T) * 3 * n * batch, st));
    PCU_TRY(h2d(ws, dy, y, sizeof(T) * 3 * m * batch, st));
    PCU_TRY(batched_chamfer_device<T>(ws, dx, dy, batch, n, m, dv, out_sum ? dsum : nullptr, st));
    PCU_CUDA(cudaMemcpyAsync(out_per_pair, dv, sizeof(T) * batch, cudaMemcpyDeviceToHost, st));
    if (out_sum) PCU_CUDA(cudaMemcpyAsync(out_sum, dsum, sizeof(double), cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    return PCU_B200_OK;
}

// Host wrapper shared by the two normal estimators: stage points (and view directions), run `device_call` on the
// workspace's stream, fetch the count, then exactly the kept rows.
template <typename T, typename DeviceCall>
int normals_host(pcu_b200_workspace* ws, const T* points, long long n, const T* view_dirs, long long* out_idx, T* out_normals,
                 long long* out_count, DeviceCall&& device_call) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!points || n <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid point set with zero elements: points must have shape (n, 3) (got %lld rows)", n);
    if (!out_idx || !out_normals || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    T *dp, *dv, *dn; long long *di, *dc;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        dp = cv.take<T>((size_t)3 * n);
        dv = cv.take<T>(view_dirs ? (size_t)3 * n : 1);
        di = cv.take<long long>((size_t)n);
        dn = cv.take<T>((size_t)3 * n);
        dc = cv.take<long long>(1);
    }));
    PCU_TRY(h2d(ws, dp, points, sizeof(T) * 3 * n, st));
    if (view_dirs) PCU_TRY(h2d(ws, dv, view_dirs, sizeof(T) * 3 * n, st));
    PCU_TRY(device_call(dp, view_dirs ? dv : (const T*)nullptr, di, dn, dc, st));
    long long* hc = reinterpret_cast<long long*>(ws->host_slot);
    PCU_CUDA(cudaMemcpyAsync(hc, dc, sizeof(long long), cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    const long long kept = *hc;
    if (kept > 0) {
        PCU_CUDA(cudaMemcpyAsync(out_idx, di, sizeof(long long) * kept, cudaMemcpyDeviceToHost, st));
        PCU_CUDA(cudaMemcpyAsync(out_normals, dn, sizeof(T) * 3 * kept, cudaMemcpyDeviceToHost, st));
        PCU_CUDA(cudaStreamSynchronize(st));
    }
    *out_count = kept;
    return PCU_B200_OK;
}

template <typename T>
int normals_knn_host(pcu_b200_workspace* ws, const T* points, long long n, const T* view_dirs, int k,
                     double drop_angle_threshold, long long* out_idx, T* out_normals, long long* out_count) {
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid number of neighbors (%d) must be greater than 0.", k);
    return normals_host<T>(ws, points, n, view_dirs, out_idx, out_normals, out_count,
                           [&](const T* dp, const T* dv, long long* di, T* dn, long long* dc, cudaStream_t st) {
                               return normals_knn_device<T>(ws, dp, n, dv, k, drop_angle_threshold, di, dn, dc, st);
                           });
}

template <typename T>
int normals_ball_host(pcu_b200_workspace* ws, const T* points, long long n, const T* view_dirs, const pcu_b200_ball_options* o,
                      long long* out_idx, T* out_normals, long long* out_count) {
    return normals_host<T>(ws, points, n, view_dirs, out_idx, out_normals, out_count,
                           [&](const T* dp, const T* dv, long long* di, T* dn, long long* dc, cudaStream_t st) {
                               return normals_ball_device<T>(ws, dp, n, dv, o, di, dn, dc, st);
                           });
}

// Prepares a cloud from HOST points: staged through the workspace, binned into the handle's own block.
template <typename T>
int cloud_prepare_host(pcu_b200_workspace* ws, const T* points, long long n, pcu_b200_cloud** out, int knn_k = 1, int leaf = 0) {
    if (!ws || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_cloud_args<T>(points, n, points, 1));
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    T* dp;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) { dp = cv.take<T>((size_t)3 * n); }));
    PCU_TRY(h2d(ws, dp, points, sizeof(T) * 3 * n, st));
    PCU_TRY(cloud_prepare_device<T>(ws, dp, n, out, st, knn_k, leaf));
    PCU_CUDA(cudaStreamSynchronize(st));
    return PCU_B200_OK;
}

template <typename T>
int debug_kd_tree(pcu_b200_workspace* ws, const T* points, long long m, int leaf, int32_t* order, long long node_cap,
                  int32_t* feat, T* div_lo, T* div_hi, int32_t* first, int32_t* last, int32_t* kid0, int32_t* kid1,
                  int64_t* out_nodes) {
    if (!ws || !points || m <= 0 || leaf <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "bad argument");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    KdReplayBuffers<T> rb;
    T* dpts;
    PCU_TRY(carve_scratch(ws, kArena, st, [&](Carver& cv) {
        rb.carve(cv, m);
        dpts = cv.take<T>((size_t)3 * m);
    }));
    PCU_TRY(h2d(ws, dpts, points, sizeof(T) * 3 * m, st));
    const int rs = build_kd_replica<T>(rb, dpts, m, leaf, nullptr, KdPrune<T>{}, st, g_launches);
    if (rs != PCU_B200_OK) return fail(rs, "kd replica build failed: %s", cudaGetErrorString(cudaGetLastError()));
    KdCounters hc;
    PCU_CUDA(cudaMemcpyAsync(&hc, rb.counters, sizeof hc, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaMemcpyAsync(order, rb.order, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    std::vector<KdNode<T>> nodes((size_t)hc.n_nodes);
    PCU_CUDA(cudaMemcpy(nodes.data(), rb.nodes, sizeof(KdNode<T>) * nodes.size(), cudaMemcpyDeviceToHost));
    for (long long i = 0; i < hc.n_nodes && i < node_cap; ++i) {
        feat[i] = nodes[i].feat; div_lo[i] = nodes[i].div_lo; div_hi[i] = nodes[i].div_hi;
        first[i] = nodes[i].first; last[i] = nodes[i].last; kid0[i] = nodes[i].kid0; kid1[i] = nodes[i].kid1;
    }
    *out_nodes = hc.n_nodes;
    return PCU_B200_OK;
}

}  // namespace

namespace __attribute__((visibility("hidden"))) pcu_internal {

// ---- k nearest neighbours ---------------------------------------------------------------------
template <typename T>
int knn_device(pcu_b200_workspace* ws, const T* query, long long n, const T* dataset, long long m, int k, int squared,
               T* out_dist, long long* out_idx, long long* out_n_tied, cudaStream_t stream, pcu_b200_cloud* prepared,
               bool tie_replay) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid value for k (%d) must be greater than 0.", k);
    if (prepared != nullptr) {
        if (prepared->is_f64 != (sizeof(T) == 8 ? 1 : 0)) return fail(PCU_B200_INVALID_ARGUMENT, "the prepared cloud has another precision than the points");
        if (prepared->device != ws->device) return fail(PCU_B200_INVALID_ARGUMENT, "the prepared cloud lives on device %d, the workspace on %d", prepared->device, ws->device);
        dataset = (const T*)prepared->raw;
        m = prepared->n;
    }
    PCU_TRY(check_cloud_args<T>(query, n, dataset, m));
    if (!out_dist || !out_idx) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    if ((double)n * (double)k >= 9e18) return fail(PCU_B200_INVALID_ARGUMENT, "n * k overflows");
    PCU_ON_DEVICE(ws);

    PlanSpec<T> spec;
    spec.a = query; spec.n = n; spec.b = dataset; spec.m = m;
    spec.nsweeps = 1; spec.k = k; spec.squared = squared; spec.want_out = true;
    spec.occupancy = occupancy_for(ws, k);
    spec.binning = ws->opts.binning;
    spec.out_dist = out_dist; spec.out_idx = out_idx;
    const int leaf = ws->opts.max_points_per_leaf > 0 ? ws->opts.max_points_per_leaf : 10;
    // a prepared cloud that owns the reference tree (same leaf size) spares the call the build
    // tie_replay = false: callers to whom the order among equidistant neighbours does not matter (the Voronoi cells)
    // skip the replay without touching the workspace option
    const bool replay = tie_replay && ws->opts.disable_tie_replay != 1;
    const bool own_tree = replay && prepared != nullptr && prepared->leaf == leaf && ws->opts.disable_tie_replay == 0;
    spec.replay_points = (!replay || own_tree) ? 0 : m;
    spec.prepared_second = prepared != nullptr;
    Plan<T> plan;
    PCU_TRY(prepare_plan(ws, plan, spec, stream));
    if (prepared != nullptr) plan.cv.v[1] = cloud_desc<T>(prepared);   // a single pair: descriptors travel by value
    mark(ws, 0, stream);
    PCU_TRY(upload_descriptors(plan, stream));
    mark(ws, 1, stream);
    PCU_TRY(enqueue_binning(ws, plan, stream, nullptr, prepared != nullptr));
    const unsigned qblocks = (unsigned)((n + kThreads - 1) / kThreads);
    if (k == 1) {
        PCU_LAUNCH_CS(nn1_kernel, dim3(qblocks, 1), kThreads, true, false);
        mark(ws, 6, stream);
        PCU_LAUNCH_CS(nn1_far_kernel, dim3(plan.far_blocks, 1), kThreads, true, false);
        PCU_LAUNCH_CS(nn1_vfar_kernel, dim3(plan.far_blocks, 1), kThreads, true, false);
        mark(ws, 7, stream);
    } else if (k <= 32) {
        // thread-per-query lists in registers (capacity = next power of two), warp pass for the rest
        if (k <= 4)       PCU_LAUNCH_CS(knn_thread_kernel, dim3(qblocks, 1), kThreads, 4);
        else if (k <= 8)  PCU_LAUNCH_CS(knn_thread_kernel, dim3(qblocks, 1), kThreads, 8);
        else if (k <= 16) PCU_LAUNCH_CS(knn_thread_kernel, dim3(qblocks, 1), kThreads, 16);
        else              PCU_LAUNCH_CS(knn_thread_kernel, dim3(qblocks, 1), kThreads, 32);
        mark(ws, 6, stream);
        PCU_LAUNCH_CS(knn_warp_kernel, dim3(plan.far_blocks, 1), kThreads);
        PCU_LAUNCH_CS(knn_descend_kernel, dim3(plan.far_blocks, 1), kThreads, false);
        mark(ws, 7, stream);
    } else {
        // large k: generic path, every query descends the occupancy pyramid
        PCU_LAUNCH_CS(pyramid_build_kernel, dim3(1, 1), kThreads);
        PCU_LAUNCH_CS(knn_descend_kernel, dim3(std::min<unsigned>(qblocks, 2368u), 1), kThreads, true);
        mark(ws, 6, stream);
        mark(ws, 7, stream);
    }
    if (own_tree) {
        KdReplayBuffers<T>& tree = cloud_tree<T>(prepared);
        const int rs = enqueue_tie_replay_prebuilt<T>(tree, query, dataset, k, squared, plan.args.sweep[0].tie_list,
                                                      plan.args.sweep[0].counters + 1, n, out_dist, out_idx, stream, g_launches);
        if (rs != PCU_B200_OK) return fail(rs, "tie replay failed: %s", cudaGetErrorString(cudaGetLastError()));
        ws->replay_overflows = tree.overflows;
    } else if (replay) {
        const int rs = enqueue_tie_replay<T>(plan.replay, query, dataset, m, k, squared, leaf, plan.args.sweep[0].tie_list,
                                             plan.args.sweep[0].counters + 1, n, out_dist, out_idx, ws->opts.disable_tie_replay, stream, g_launches);
        if (rs != PCU_B200_OK) return fail(rs, "tie replay failed: %s", cudaGetErrorString(cudaGetLastError()));
        ws->replay_overflows = plan.replay.overflows;
    } else {
        ws->replay_overflows = nullptr;
    }
    if (out_n_tied) {
        PCU_LAUNCH(widen_counter_kernel, 1, 1, stream, plan.args.sweep[0].counters + 1, out_n_tied);
    }
    mark(ws, 8, stream);
    return PCU_B200_OK;
}

template <typename T>
int poisson_disk_device(pcu_b200_workspace* ws, const T* points, long long n, double radius, unsigned seed, int* out_idx,
                        long long* out_count, int* out_rounds, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!(radius > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid radius (%f) must be greater than 0.", radius);
    if (!points || n <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid point set with zero elements: points must have shape (n, 3) (got %lld rows)", n);
    if (n > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "poisson_disk: at most 2^31 - 1 points (the indices are int32), got %lld", n);
    PCU_TRY(check_cloud_args<T>(points, n, points, 1));
    if (!out_idx || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    const T r = (T)radius;        // blue_noise_downsample takes the radius as the cloud's scalar (:299, :328)
    const T rr = r * r;           // `const double rr = r*r;` with r of that type: the product is rounded in T (:72)
    Plan<T> plan;
    PCU_TRY(single_cloud_plan<T>(ws, points, n, 0.5 * (double)r, plan, stream));
    unsigned blocks = 1;
    PCU_TRY(poisson_grid_blocks<T>(ws->device, ws->sm_count, n, &blocks));
    PoissonScratch s; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        s.ring = cv.take<unsigned>(4);
        s.state = cv.take<unsigned char>((size_t)n);
        s.keep = cv.take<unsigned char>((size_t)n);
        s.list[0] = cv.take<unsigned>((size_t)n);
        s.list[1] = cv.take<unsigned>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_CUDA(cudaMemsetAsync(s.ring, 0, (size_t)((unsigned char*)s.list[0] - (unsigned char*)s.ring), stream));   // ring, state, keep
    mark(ws, 0, stream);
    mark(ws, 1, stream);
    PCU_TRY(enqueue_binning(ws, plan, stream, nullptr, true));
    Cloud<T> cl = plan.cv.v[0];
    T rr_arg = rr;
    void* args[] = {(void*)&cl, (void*)&rr_arg, (void*)&seed, (void*)&s, (void*)&out_rounds};
    PCU_CUDA(cudaLaunchCooperativeKernel((void*)poisson_rounds_kernel<T>, dim3(blocks), dim3(kThreads), args, 0, stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    mark(ws, 6, stream);
    PCU_TRY(enqueue_keep_offsets(s.keep, n, counts, out_count, stream));
    PCU_TRY(enqueue_keep_rows(s.keep, n, counts, out_idx, stream));
    mark(ws, 7, stream);
    mark(ws, 8, stream);
    return PCU_B200_OK;
}

// ---- principal curvatures from a quadric fit over a ball (mesh_principal_curvatures, r > 0) --------------------------
// The vertices are binned once (cells no finer than r / 2) and put in row order within every cell, then one thread per
// vertex walks its ball (curv_ball_kernel).
template <typename T>
int curvature_ball_device(pcu_b200_workspace* ws, const T* v, long long nv, const double* normal, double r, T* out_k1, T* out_k2,
                          T* out_d1, T* out_d2, cudaStream_t stream) {
    PCU_TRY(check_cloud_args<T>(v, nv, v, 1));
    Plan<T> plan;
    PCU_TRY(single_cloud_plan<T>(ws, v, nv, 0.5 * r, plan, stream));
    PCU_TRY(enqueue_binning(ws, plan, stream, nullptr, true));
    PCU_LAUNCH((cell_order_kernel<T>), (unsigned)std::min<long long>(((long long)plan.cv.v[0].cell_cap + kThreads - 1) / kThreads, (long long)ws->sm_count * 64), kThreads, stream, plan.cv.v[0]);
    PCU_LAUNCH((curv_ball_kernel<T>), blocks_for(nv), kThreads, stream, plan.cv.v[0], normal, r, out_k1, out_k2, out_d1, out_d2);
    return PCU_B200_OK;
}

template int curvature_ball_device<float>(pcu_b200_workspace*, const float*, long long, const double*, double, float*, float*, float*,
                                          float*, cudaStream_t);
template int curvature_ball_device<double>(pcu_b200_workspace*, const double*, long long, const double*, double, double*, double*,
                                           double*, double*, cudaStream_t);
template int knn_device<float>(pcu_b200_workspace*, const float*, long long, const float*, long long, int, int, float*, long long*,
                               long long*, cudaStream_t, pcu_b200_cloud*, bool);
template int knn_device<double>(pcu_b200_workspace*, const double*, long long, const double*, long long, int, int, double*, long long*,
                                long long*, cudaStream_t, pcu_b200_cloud*, bool);
template int poisson_disk_device<float>(pcu_b200_workspace*, const float*, long long, double, unsigned, int*, long long*, int*,
                                        cudaStream_t);
template int poisson_disk_device<double>(pcu_b200_workspace*, const double*, long long, double, unsigned, int*, long long*, int*,
                                         cudaStream_t);

}  // namespace pcu_internal

// =================================================================================================
extern "C" {

int pcu_b200_knn_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m, int k,
                     int squared, float* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream) {
    return knn_device<float>(ws, query, n, dataset, m, k, squared, out_dist, (long long*)out_idx,
                             (long long*)out_n_tied, (cudaStream_t)stream);
}
int pcu_b200_knn_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m, int k,
                     int squared, double* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream) {
    return knn_device<double>(ws, query, n, dataset, m, k, squared, out_dist, (long long*)out_idx,
                              (long long*)out_n_tied, (cudaStream_t)stream);
}
int pcu_b200_nn_stats_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m,
                          pcu_b200_nn_stats* out_stats, void* stream) {
    return stats_device<float>(ws, query, n, dataset, m, false, out_stats, nullptr, (cudaStream_t)stream);
}
int pcu_b200_nn_stats_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m,
                          pcu_b200_nn_stats* out_stats, void* stream) {
    return stats_device<double>(ws, query, n, dataset, m, false, out_stats, nullptr, (cudaStream_t)stream);
}
int pcu_b200_resolve_witness_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset,
                                 int64_t m, pcu_b200_nn_stats* stats, void* stream) {
    return resolve_witness_device<float>(ws, query, n, dataset, m, stats, (cudaStream_t)stream);
}
int pcu_b200_resolve_witness_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset,
                                 int64_t m, pcu_b200_nn_stats* stats, void* stream) {
    return resolve_witness_device<double>(ws, query, n, dataset, m, stats, (cudaStream_t)stream);
}
int pcu_b200_chamfer_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const float* y, int64_t m,
                         pcu_b200_nn_stats* out_stats, float* out_value, void* stream) {
    return stats_device<float>(ws, x, n, y, m, true, out_stats, out_value, (cudaStream_t)stream);
}
int pcu_b200_chamfer_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const double* y, int64_t m,
                         pcu_b200_nn_stats* out_stats, double* out_value, void* stream) {
    return stats_device<double>(ws, x, n, y, m, true, out_stats, out_value, (cudaStream_t)stream);
}

int pcu_b200_cloud_prepare_f32(pcu_b200_workspace* ws, const float* points, int64_t n, pcu_b200_cloud** out_cloud, void* stream) {
    return cloud_prepare_device<float>(ws, points, n, out_cloud, (cudaStream_t)stream);
}
int pcu_b200_cloud_prepare_f64(pcu_b200_workspace* ws, const double* points, int64_t n, pcu_b200_cloud** out_cloud, void* stream) {
    return cloud_prepare_device<double>(ws, points, n, out_cloud, (cudaStream_t)stream);
}
int pcu_b200_cloud_prepare_knn_f32(pcu_b200_workspace* ws, const float* points, int64_t n, int k, int max_points_per_leaf,
                                   pcu_b200_cloud** out_cloud, void* stream) {
    return cloud_prepare_device<float>(ws, points, n, out_cloud, (cudaStream_t)stream, k, max_points_per_leaf > 0 ? max_points_per_leaf : 10);
}
int pcu_b200_cloud_prepare_knn_f64(pcu_b200_workspace* ws, const double* points, int64_t n, int k, int max_points_per_leaf,
                                   pcu_b200_cloud** out_cloud, void* stream) {
    return cloud_prepare_device<double>(ws, points, n, out_cloud, (cudaStream_t)stream, k, max_points_per_leaf > 0 ? max_points_per_leaf : 10);
}
int pcu_b200_knn_prepared_f32(pcu_b200_workspace* ws, const float* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                              float* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return knn_device<float>(ws, query, n, nullptr, 0, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied,
                             (cudaStream_t)stream, dataset);
}
int pcu_b200_knn_prepared_f64(pcu_b200_workspace* ws, const double* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                              double* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return knn_device<double>(ws, query, n, nullptr, 0, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied,
                              (cudaStream_t)stream, dataset);
}
int pcu_b200_cloud_destroy(pcu_b200_cloud* cloud) {
    if (!cloud) return PCU_B200_OK;
    DeviceGuard guard(cloud->device);
    cudaDeviceSynchronize();          // calls that use the cloud may still be queued
    if (cloud->block) cudaFree(cloud->block);
    delete cloud;
    return PCU_B200_OK;
}
int64_t pcu_b200_cloud_size(const pcu_b200_cloud* cloud) { return cloud ? cloud->n : 0; }
const void* pcu_b200_cloud_points(const pcu_b200_cloud* cloud) { return cloud ? cloud->raw : nullptr; }
int pcu_b200_chamfer_prepared_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const pcu_b200_cloud* y,
                                  pcu_b200_nn_stats* out_stats, float* out_value, void* stream) {
    if (!y) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_device<float>(ws, x, n, nullptr, 0, true, out_stats, out_value, (cudaStream_t)stream, nullptr, y);
}
int pcu_b200_chamfer_prepared_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const pcu_b200_cloud* y,
                                  pcu_b200_nn_stats* out_stats, double* out_value, void* stream) {
    if (!y) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_device<double>(ws, x, n, nullptr, 0, true, out_stats, out_value, (cudaStream_t)stream, nullptr, y);
}
int pcu_b200_nn_stats_prepared_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const pcu_b200_cloud* dataset,
                                   pcu_b200_nn_stats* out_stats, void* stream) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_device<float>(ws, query, n, nullptr, 0, false, out_stats, nullptr, (cudaStream_t)stream, nullptr, dataset);
}
int pcu_b200_nn_stats_prepared_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const pcu_b200_cloud* dataset,
                                   pcu_b200_nn_stats* out_stats, void* stream) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_device<double>(ws, query, n, nullptr, 0, false, out_stats, nullptr, (cudaStream_t)stream, nullptr, dataset);
}

int pcu_b200_normals_knn_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs, int k,
                             double drop_angle_threshold, int64_t* out_idx, float* out_normals, int64_t* out_count, void* stream) {
    return normals_knn_device<float>(ws, points, n, view_dirs, k, drop_angle_threshold, (long long*)out_idx, out_normals,
                                     (long long*)out_count, (cudaStream_t)stream);
}
int pcu_b200_normals_knn_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs, int k,
                             double drop_angle_threshold, int64_t* out_idx, double* out_normals, int64_t* out_count, void* stream) {
    return normals_knn_device<double>(ws, points, n, view_dirs, k, drop_angle_threshold, (long long*)out_idx, out_normals,
                                      (long long*)out_count, (cudaStream_t)stream);
}

int pcu_b200_normals_ball_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs,
                              const pcu_b200_ball_options* options, int64_t* out_idx, float* out_normals, int64_t* out_count, void* stream) {
    return normals_ball_device<float>(ws, points, n, view_dirs, options, (long long*)out_idx, out_normals, (long long*)out_count, (cudaStream_t)stream);
}
int pcu_b200_normals_ball_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs,
                              const pcu_b200_ball_options* options, int64_t* out_idx, double* out_normals, int64_t* out_count, void* stream) {
    return normals_ball_device<double>(ws, points, n, view_dirs, options, (long long*)out_idx, out_normals, (long long*)out_count, (cudaStream_t)stream);
}

int pcu_b200_poisson_disk_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double radius, uint32_t seed,
                              int32_t* out_idx, int64_t* out_count, int32_t* out_rounds, void* stream) {
    return poisson_disk_device<float>(ws, points, n, radius, seed, out_idx, (long long*)out_count, out_rounds, (cudaStream_t)stream);
}
int pcu_b200_poisson_disk_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double radius, uint32_t seed,
                              int32_t* out_idx, int64_t* out_count, int32_t* out_rounds, void* stream) {
    return poisson_disk_device<double>(ws, points, n, radius, seed, out_idx, (long long*)out_count, out_rounds, (cudaStream_t)stream);
}

int pcu_b200_apss_project_f32(pcu_b200_workspace* ws, const float* p, const float* n, int64_t np, const float* q, int64_t nq, double r,
                              float* out_x, float* out_n, float* out_kh, void* stream) {
    return apss_device<float>(ws, p, n, np, q, nq, r, out_x, out_n, out_kh, (cudaStream_t)stream);
}
int pcu_b200_apss_project_f64(pcu_b200_workspace* ws, const double* p, const double* n, int64_t np, const double* q, int64_t nq, double r,
                              double* out_x, double* out_n, double* out_kh, void* stream) {
    return apss_device<double>(ws, p, n, np, q, nq, r, out_x, out_n, out_kh, (cudaStream_t)stream);
}

int pcu_b200_debug_kd_times(pcu_b200_workspace* ws, uint64_t* out40) {
    if (!ws || !out40) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    PCU_CUDA(cudaDeviceSynchronize());
    PCU_CUDA(cudaMemcpyFromSymbol(out40, g_kd_times, sizeof(unsigned long long) * 40));
    return PCU_B200_OK;
}

int pcu_b200_batched_chamfer_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch, int64_t n,
                                 int64_t m, float* out_per_pair, double* out_sum, void* stream) {
    return batched_chamfer_device<float>(ws, x, y, batch, n, m, out_per_pair, out_sum, (cudaStream_t)stream);
}

int pcu_b200_debug_batched_chamfer_stats_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch, int64_t n,
                                             int64_t m, pcu_b200_nn_stats* out_stats, float* out_per_pair, void* stream) {
    if (!out_stats) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    return batched_chamfer_device<float>(ws, x, y, batch, n, m, out_per_pair, nullptr, (cudaStream_t)stream, out_stats);
}

int pcu_b200_knn_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m,
                          int k, int squared, float* out_dist, int64_t* out_idx, int64_t* out_n_tied) {
    return knn_host<float>(ws, query, n, dataset, m, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied);
}
int pcu_b200_knn_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m,
                          int k, int squared, double* out_dist, int64_t* out_idx, int64_t* out_n_tied) {
    return knn_host<double>(ws, query, n, dataset, m, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied);
}
int pcu_b200_nn_stats_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset,
                               int64_t m, pcu_b200_nn_stats* out_stats) {
    return stats_host<float>(ws, query, n, dataset, m, false, out_stats, nullptr);
}
int pcu_b200_nn_stats_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset,
                               int64_t m, pcu_b200_nn_stats* out_stats) {
    return stats_host<double>(ws, query, n, dataset, m, false, out_stats, nullptr);
}
int pcu_b200_chamfer_host_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const float* y, int64_t m,
                              pcu_b200_nn_stats* out_stats, float* out_value) {
    return stats_host<float>(ws, x, n, y, m, true, out_stats, out_value);
}
int pcu_b200_chamfer_host_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const double* y, int64_t m,
                              pcu_b200_nn_stats* out_stats, double* out_value) {
    return stats_host<double>(ws, x, n, y, m, true, out_stats, out_value);
}

int pcu_b200_debug_kd_tree_f32(pcu_b200_workspace* ws, const float* points, int64_t m, int max_points_per_leaf,
                               int32_t* order, int64_t node_cap, int32_t* feat, float* div_lo, float* div_hi,
                               int32_t* first, int32_t* last, int32_t* kid0, int32_t* kid1, int64_t* out_nodes) {
    return debug_kd_tree<float>(ws, points, m, max_points_per_leaf, order, node_cap, feat, div_lo, div_hi, first, last,
                                kid0, kid1, out_nodes);
}
int pcu_b200_debug_kd_tree_f64(pcu_b200_workspace* ws, const double* points, int64_t m, int max_points_per_leaf,
                               int32_t* order, int64_t node_cap, int32_t* feat, double* div_lo, double* div_hi,
                               int32_t* first, int32_t* last, int32_t* kid0, int32_t* kid1, int64_t* out_nodes) {
    return debug_kd_tree<double>(ws, points, m, max_points_per_leaf, order, node_cap, feat, div_lo, div_hi, first, last,
                                 kid0, kid1, out_nodes);
}
int pcu_b200_cloud_prepare_knn_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, int k, int max_points_per_leaf,
                                        pcu_b200_cloud** out_cloud) {
    return cloud_prepare_host<float>(ws, points, n, out_cloud, k, max_points_per_leaf > 0 ? max_points_per_leaf : 10);
}
int pcu_b200_cloud_prepare_knn_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, int k, int max_points_per_leaf,
                                        pcu_b200_cloud** out_cloud) {
    return cloud_prepare_host<double>(ws, points, n, out_cloud, k, max_points_per_leaf > 0 ? max_points_per_leaf : 10);
}
int pcu_b200_knn_prepared_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                                   float* out_dist, int64_t* out_idx, int64_t* out_n_tied) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return knn_host<float>(ws, query, n, nullptr, 0, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied, dataset);
}
int pcu_b200_knn_prepared_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                                   double* out_dist, int64_t* out_idx, int64_t* out_n_tied) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return knn_host<double>(ws, query, n, nullptr, 0, k, squared, out_dist, (long long*)out_idx, (long long*)out_n_tied, dataset);
}
int pcu_b200_cloud_prepare_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, pcu_b200_cloud** out_cloud) {
    return cloud_prepare_host<float>(ws, points, n, out_cloud);
}
int pcu_b200_cloud_prepare_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, pcu_b200_cloud** out_cloud) {
    return cloud_prepare_host<double>(ws, points, n, out_cloud);
}
int pcu_b200_chamfer_prepared_host_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const pcu_b200_cloud* y,
                                       pcu_b200_nn_stats* out_stats, float* out_value) {
    if (!y) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_host<float>(ws, x, n, nullptr, 0, true, out_stats, out_value, y);
}
int pcu_b200_chamfer_prepared_host_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const pcu_b200_cloud* y,
                                       pcu_b200_nn_stats* out_stats, double* out_value) {
    if (!y) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_host<double>(ws, x, n, nullptr, 0, true, out_stats, out_value, y);
}
int pcu_b200_nn_stats_prepared_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const pcu_b200_cloud* dataset,
                                        pcu_b200_nn_stats* out_stats) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_host<float>(ws, query, n, nullptr, 0, false, out_stats, nullptr, dataset);
}
int pcu_b200_nn_stats_prepared_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const pcu_b200_cloud* dataset,
                                        pcu_b200_nn_stats* out_stats) {
    if (!dataset) return fail(PCU_B200_INVALID_ARGUMENT, "null prepared cloud");
    return stats_host<double>(ws, query, n, nullptr, 0, false, out_stats, nullptr, dataset);
}

int pcu_b200_normals_knn_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs, int k,
                                  double drop_angle_threshold, int64_t* out_idx, float* out_normals, int64_t* out_count) {
    return normals_knn_host<float>(ws, points, n, view_dirs, k, drop_angle_threshold, (long long*)out_idx, out_normals, (long long*)out_count);
}
int pcu_b200_normals_knn_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs, int k,
                                  double drop_angle_threshold, int64_t* out_idx, double* out_normals, int64_t* out_count) {
    return normals_knn_host<double>(ws, points, n, view_dirs, k, drop_angle_threshold, (long long*)out_idx, out_normals, (long long*)out_count);
}
int pcu_b200_normals_ball_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs,
                                   const pcu_b200_ball_options* options, int64_t* out_idx, float* out_normals, int64_t* out_count) {
    return normals_ball_host<float>(ws, points, n, view_dirs, options, (long long*)out_idx, out_normals, (long long*)out_count);
}
int pcu_b200_normals_ball_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs,
                                   const pcu_b200_ball_options* options, int64_t* out_idx, double* out_normals, int64_t* out_count) {
    return normals_ball_host<double>(ws, points, n, view_dirs, options, (long long*)out_idx, out_normals, (long long*)out_count);
}
int pcu_b200_batched_chamfer_host_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch,
                                      int64_t n, int64_t m, float* out_per_pair, double* out_sum) {
    return batched_chamfer_host<float>(ws, x, y, batch, n, m, out_per_pair, out_sum);
}

}  // extern "C"
