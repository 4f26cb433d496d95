// voronoi.cu -- Voronoi cells in the unit cube and square, Lloyd relaxation, Voronoi cells restricted to a triangle mesh
// and Lloyd sampling of its surface (voronoi.cuh, rvd.cuh): launch sequencing and C entry points.
#include "runtime.cuh"
#include "voronoi.cuh"
#include "rvd.cuh"

using namespace pcu;
using namespace pcu_internal;

namespace {

// ---- Voronoi cells in the unit cube / square and Lloyd relaxation (voronoi.cuh) ----------------------------------
// One evaluation of the cells of n seeds (fp64, (n, dim)):
//   pass 1  the seeds' self k-NN (k = 64 in 3-D, 24 in 2-D; no tie replay: the order among equidistant neighbours
//           cannot change a cell, and the certificate only reads the k-th distance), then every cell on the thread's
//           stack at 96 (3-D) / 48 (2-D) vertices;
//   pass 2  the cells pass 1 left uncertified, compacted in ascending order: their k-NN with k = 160 (3-D) / 64 (2-D),
//           at 252 / 250 vertices;
//   pass 3  what pass 2 left: its list, then every seed that can still cut the cell, with the cell in device memory at
//           2 048 (3-D) / 1 024 (2-D) vertices; the cells that outgrow it are compacted and redone at twice the
//           capacity, until every cell is certified.
// The host reads the count after pass 1 (one synchronisation), after pass 2 when it ran, and after every round of
// pass 3.  passes[p] += cells handled by pass p (pass 3: summed over its rounds).
constexpr int kVorK1[2] = {24, 64}, kVorK2[2] = {64, 160};   // by dim - 2
constexpr int kVorSmall[2] = {48, 96}, kVorLarge[2] = {250, 252};
constexpr int kVorWide[2] = {1024, 2048};
constexpr int kVorWideMax = 1 << 22;   // vertices of one cell: 150 MB of device memory in 3-D

// pass 0, 1: the small and the large capacity on the stack
template <int D>
int vor_pass_launch(const VorPass& p, int pass, cudaStream_t stream) {
    const unsigned blocks = (unsigned)((p.count + kVorThreads - 1) / kVorThreads);
    if (pass == 0) PCU_LAUNCH((vor_clip_kernel<D, kVorSmall[D - 2]>), blocks, kVorThreads, stream, p);
    else           PCU_LAUNCH((vor_clip_kernel<D, kVorLarge[D - 2]>), blocks, kVorThreads, stream, p);
    return PCU_B200_OK;
}

// How the passes clip one kind of entry: the cells in the unit cube / square, or the (face, seed) pairs of restricted
// cells (rvd.cuh).  k2: the longer lists of pass 2; wide: the first capacity of pass 3.
template <int D>
struct VorCube {
    static constexpr int k2 = kVorK2[D - 2], wide = kVorWide[D - 2];
    static int launch(const VorPass& p, int pass, cudaStream_t stream) { return vor_pass_launch<D>(p, pass, stream); }
    static size_t cell_bytes(int V) { return vor_cell_bytes<D>(V); }
    static int launch_wide(const VorPass& p, int V, cudaStream_t stream) {
        PCU_LAUNCH(vor_clip_wide_kernel<D>, (unsigned)((p.count + kVorThreads - 1) / kVorThreads), kVorThreads, stream, p, V);
        return PCU_B200_OK;
    }
};

// Restricted pairs: the k-NN lists of a 2-D cell (a restricted cell is a surface patch), polygons of 16 / 64 vertices on
// the stack, then 256 in device memory.
constexpr int kRvK1 = 24, kRvK2 = 64, kRvSmall = 16, kRvLarge = 64, kRvWide = 256;
struct VorRestricted {
    static constexpr int k2 = kRvK2, wide = kRvWide;
    static int launch(const VorPass& p, int pass, cudaStream_t stream) {
        const unsigned blocks = (unsigned)((p.count + kVorThreads - 1) / kVorThreads);
        if (pass == 0) PCU_LAUNCH(rv_clip_kernel<kRvSmall>, blocks, kVorThreads, stream, p);
        else           PCU_LAUNCH(rv_clip_kernel<kRvLarge>, blocks, kVorThreads, stream, p);
        return PCU_B200_OK;
    }
    static size_t cell_bytes(int V) { return poly_bytes(V); }
    static int launch_wide(const VorPass& p, int V, cudaStream_t stream) {
        PCU_LAUNCH(rv_clip_wide_kernel, (unsigned)((p.count + kVorThreads - 1) / kVorThreads), kVorThreads, stream, p, V);
        return PCU_B200_OK;
    }
};

// Passes 2 and 3 over the entries pass 1 (p, already enqueued over p.count entries) left uncertified in `flag`; `counts`
// holds keep_count_words(p.count) words.
template <class K>
int vor_fallback(pcu_b200_workspace* ws, VorPass p, unsigned char* flag, unsigned* counts, VorSync* sync, long long* passes,
                 VorSync* seen, cudaStream_t stream) {
    const long long n = p.n, entries = p.count;
    PCU_TRY(enqueue_keep_offsets(flag, entries, counts, &sync->count, stream));
    PCU_TRY(read_record(sync, seen, stream));
    const long long c1 = seen->count;
    if (c1 == 0) return PCU_B200_OK;
    const int k2 = (int)std::min<long long>(K::k2, n);
    int *rows, *sub[2]; double *q, *d2; long long* i2; unsigned char* flag2; unsigned* counts2;
    PCU_TRY(carve_scratch(ws, kVorList, stream, [&](Carver& cv) {
        rows = cv.take<int>((size_t)c1);
        sub[0] = cv.take<int>((size_t)c1);
        sub[1] = cv.take<int>((size_t)c1);
        q = cv.take<double>((size_t)3 * c1);
        d2 = cv.take<double>((size_t)k2 * c1);
        i2 = cv.take<long long>((size_t)k2 * c1);
        flag2 = cv.take<unsigned char>((size_t)c1);
        counts2 = cv.take<unsigned>(keep_count_words(c1));
    }));
    PCU_TRY(enqueue_keep_rows(flag, entries, counts, rows, stream));
    PCU_LAUNCH(vor_gather_kernel, blocks_for(c1), kThreads, stream, p.x3, (const int*)rows, c1, q, p.pair_seed);
    PCU_TRY(knn_device<double>(ws, q, c1, p.x3, n, k2, 1, d2, i2, nullptr, stream, nullptr, false));
    p.rows = rows; p.count = c1; p.nn_idx = i2; p.nn_d2 = d2; p.k = k2; p.list_is_all = k2 >= n; p.uncert = flag2;
    p.list_of_seed = 0;
    PCU_TRY(K::launch(p, 1, stream));
    passes[1] += c1;
    PCU_TRY(enqueue_keep_offsets(flag2, c1, counts2, &sync->count, stream));
    PCU_TRY(read_record(sync, seen, stream));
    long long cnt = seen->count;
    if (cnt == 0) return PCU_B200_OK;
    // the last resort; sub[r & 1]: the pass-2 entries of round r
    PCU_TRY(enqueue_keep_rows(flag2, c1, counts2, sub[0], stream));
    p.scan_all = 1; p.list_is_all = 0; p.uncert = flag2;
    for (int V = K::wide, r = 0;; V *= 2, ++r) {
        if (V > kVorWideMax)
            return fail(PCU_B200_OUT_OF_MEMORY, "voronoi: %lld cells have more than %d vertices", cnt, kVorWideMax);
        // the cells live in the arena: the k-NN searches, its only other users here, are enqueued already
        PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
            p.cells = cv.take<unsigned char>((size_t)cnt * K::cell_bytes(V));
        }));
        p.sub = sub[r & 1]; p.count = cnt;
        PCU_TRY(K::launch_wide(p, V, stream));
        passes[2] += cnt;
        PCU_TRY(enqueue_keep_offsets(flag2, cnt, counts2, &sync->count, stream));
        PCU_TRY(read_record(sync, seen, stream));
        if (seen->count == 0) break;
        PCU_LAUNCH(vor_keep_sub_kernel, blocks_for(cnt), kThreads, stream, (const unsigned char*)flag2, cnt, (const unsigned*)counts2,
                   (const int*)sub[r & 1], sub[(r + 1) & 1]);
        cnt = seen->count;
    }
    return PCU_B200_OK;
}

template <int D>
int vor_eval(pcu_b200_workspace* ws, const double* x, long long n, VorSync* sync, double** mom_out, long long* passes,
             VorSync* seen, cudaStream_t stream) {
    const int k1 = (int)std::min<long long>(kVorK1[D - 2], n);
    double *x3 = nullptr, *mom, *d1; long long* i1; unsigned char* flag; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        if (D == 2) x3 = cv.take<double>((size_t)3 * n);
        mom = cv.take<double>((size_t)kVorMoments * n);
        d1 = cv.take<double>((size_t)k1 * n);
        i1 = cv.take<long long>((size_t)k1 * n);
        flag = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    if (D == 3) x3 = (double*)x;
    else PCU_LAUNCH(vor_lift_kernel, blocks_for(n), kThreads, stream, x, n, x3);
    *mom_out = mom;
    PCU_TRY(knn_device<double>(ws, x3, n, x3, n, k1, 1, d1, i1, nullptr, stream, nullptr, false));
    VorPass p{};
    p.x = x; p.x3 = x3; p.n = n; p.count = n; p.nn_idx = i1; p.nn_d2 = d1; p.k = k1; p.list_is_all = k1 >= n;
    p.mom = mom; p.uncert = flag;
    PCU_TRY(vor_pass_launch<D>(p, 0, stream));
    passes[0] += n;
    return vor_fallback<VorCube<D>>(ws, p, flag, counts, sync, passes, seen, stream);
}

int vor_check(long long n, int dim) {
    if (dim != 2 && dim != 3) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: dim must be 2 or 3, got %d", dim);
    if (n > 0x7fffffffLL - 1) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: at most 2^31 - 2 seeds, got %lld", n);
    return PCU_B200_OK;
}

template <int D>
int voronoi_centroids_device(pcu_b200_workspace* ws, const double* x, long long n, double* out, double* out_moments,
                             long long* passes, cudaStream_t stream) {
    VorSync* sync;
    PCU_TRY(carve_scratch(ws, kLloyd, stream, [&](Carver& cv) { sync = cv.take<VorSync>(1); }));
    PCU_CUDA(cudaMemsetAsync(sync, 0, sizeof(VorSync), stream));
    double* mom; VorSync seen;
    PCU_TRY(vor_eval<D>(ws, x, n, sync, &mom, passes, &seen, stream));
    PCU_LAUNCH(vor_centroid_kernel<D>, blocks_for(n), kThreads, stream, x, n, (const double*)mom, out);
    if (out_moments)
        PCU_CUDA(cudaMemcpyAsync(out_moments, mom, (size_t)n * kVorMoments * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return PCU_B200_OK;
}

// Blocks of the cooperative L-BFGS step: at most 4 per SM, no more than the vectors need.
int lbfgs_grid_blocks(const pcu_b200_workspace* ws, long long N, unsigned* out_blocks) {
    int fit = 0;
    PCU_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, lbfgs_step_kernel, kThreads, 0));
    if (fit < 1) return fail(PCU_B200_CUDA_ERROR, "lbfgs_step_kernel cannot be resident on this device");
    const long long want = (N + kThreads - 1) / kThreads;
    *out_blocks = (unsigned)std::max<long long>(1, std::min<long long>(want, (long long)std::min(4, fit) * ws->sm_count));
    return PCU_B200_OK;
}

// The initial sample, num_lloyd Lloyd steps, then the Newton phase (L-BFGS, voronoi.cuh), for either kind of cell:
// init(x) writes the (n, D) initial sample; eval(x, sync, &mom, &seen) evaluates the cells of x (their (n, 5) moments
// into mom); cube: trial points must lie in the unit cube.  Synchronisations: those of init and of every cell evaluation,
// one for the initial L-BFGS state, one after every L-BFGS step (its verdict decides whether the trial point is
// evaluated), and one for the energies at the end.
template <int D, class Init, class Eval>
int lloyd_run(pcu_b200_workspace* ws, long long n, int cube, int num_lloyd, int num_newton, double* out, double* energy_host,
              int* iters_host, cudaStream_t stream, Init&& init, Eval&& eval) {
    const long long N = n * D;
    const bool newton = num_newton > 0;
    unsigned blocks = 1;
    if (newton) PCU_TRY(lbfgs_grid_blocks(ws, N, &blocks));
    double *x, *x_acc = nullptr, *g = nullptr, *p = nullptr, *S = nullptr, *Y = nullptr, *partial = nullptr, *energy = nullptr;
    LbState* st = nullptr; VorSync* sync;
    PCU_TRY(carve_scratch(ws, kLloyd, stream, [&](Carver& cv) {
        sync = cv.take<VorSync>(1);
        x = cv.take<double>((size_t)N);
        if (newton) {
            st = cv.take<LbState>(1);
            energy = cv.take<double>((size_t)num_newton + 1);
            partial = cv.take<double>((size_t)2 * blocks);
            x_acc = cv.take<double>((size_t)N);
            g = cv.take<double>((size_t)N);
            p = cv.take<double>((size_t)N);
            S = cv.take<double>((size_t)kLbSlots * N);
            Y = cv.take<double>((size_t)kLbSlots * N);
        }
    }));
    PCU_CUDA(cudaMemsetAsync(sync, 0, sizeof(VorSync), stream));
    PCU_TRY(init(x));
    double* mom; VorSync seen;
    for (int it = 0; it < num_lloyd; ++it) {
        PCU_TRY(eval((const double*)x, sync, &mom, &seen));
        PCU_LAUNCH(vor_centroid_kernel<D>, blocks_for(n), kThreads, stream, (const double*)x, n, (const double*)mom, x);
    }
    if (!newton) {
        PCU_CUDA(cudaMemcpyAsync(out, x, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, stream));
        if (iters_host) *iters_host = 0;
        return PCU_B200_OK;
    }
    LbState s0{};
    s0.t = 1.0; s0.gamma = 1.0; s0.init = 1;
    PCU_CUDA(cudaMemcpyAsync(st, &s0, sizeof(LbState), cudaMemcpyHostToDevice, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));   // s0 lives on this stack
    LbArgs a{};
    a.n = n; a.D = D; a.x_acc = x_acc; a.g = g; a.x_t = x; a.p = p; a.S = S; a.Y = Y; a.partial = partial;
    a.st = st; a.sync = sync; a.energy = energy; a.num_newton = num_newton; a.cube = cube;
    PCU_TRY(eval((const double*)x, sync, &mom, &seen));
    for (;;) {
        a.mom = mom;
        void* args[] = {(void*)&a};
        PCU_CUDA(cudaLaunchCooperativeKernel((void*)lbfgs_step_kernel, dim3(blocks), dim3(kThreads), args, 0, stream));
        g_launches.fetch_add(1, std::memory_order_relaxed);
        PCU_TRY(read_record(sync, &seen, stream));   // the step's verdict: evaluate its trial point, or stop
        if (seen.done) break;
        PCU_TRY(eval((const double*)x, sync, &mom, &seen));
    }
    PCU_CUDA(cudaMemcpyAsync(out, x_acc, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    if (energy_host) PCU_CUDA(cudaMemcpyAsync(energy_host, energy, ((size_t)seen.iter + 1) * sizeof(double), cudaMemcpyDeviceToHost, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));
    if (iters_host) *iters_host = seen.iter;
    return PCU_B200_OK;
}

// lloyd_3d / lloyd_2d: the counter-based initial sample of (n, D, seed) and the cube's cells.
template <int D>
int lloyd_device(pcu_b200_workspace* ws, long long n, unsigned seed, int num_lloyd, int num_newton, double* out,
                 double* energy_host, int* iters_host, long long* passes, cudaStream_t stream) {
    const long long N = n * D;
    return lloyd_run<D>(
        ws, n, 1, num_lloyd, num_newton, out, energy_host, iters_host, stream,
        [&](double* x) -> int {
            PCU_LAUNCH(lloyd_init_kernel, blocks_for(N), kThreads, stream, seed, N, x);
            return PCU_B200_OK;
        },
        [&](const double* x, VorSync* sync, double** mom, VorSync* seen) -> int {
            return vor_eval<D>(ws, x, n, sync, mom, passes, seen, stream);
        });
}

// ---- Voronoi cells restricted to a triangle mesh and Lloyd sampling of its surface (rvd.cuh) ---------------------
// One evaluation of the cells of n seeds x (fp64, (n, 3)) on the faces:
//   the faces' candidate balls (a k = 1 search of the face centroids among the seeds), their tree, the pair count
//   (one synchronisation sizes the pairs), the pairs, the seeds' self k-NN (k = 24, no tie replay), then pass 1 over
//   every pair with the polygon on the stack at 16 vertices, and the fallback passes of the cube's cells (vor_fallback:
//   k = 64 and 64 vertices, then every seed from 256 vertices in device memory up); finally each seed's pairs summed in
//   order.  Synchronisations: the pair count, the count pass 1 leaves, and one per fallback pass or round that runs.
//   passes[p] += pairs handled by pass p.
struct RvScratch {
    long long n = 0, m = 0;
    int k1 = 1;
    double *tri, *cen, *rad, *fd2, *balls, *sd2, *mom;
    long long *fidx, *sidx, *start;
    unsigned long long *local, *tiles, *bad;
    VorSync* sync;
    void carve(Carver& cv) {
        tri = cv.take<double>((size_t)9 * m);
        cen = cv.take<double>((size_t)3 * m);
        rad = cv.take<double>((size_t)m);
        fd2 = cv.take<double>((size_t)m);
        fidx = cv.take<long long>((size_t)m);
        balls = cv.take<double>((size_t)4 * m);
        sd2 = cv.take<double>((size_t)k1 * n);
        sidx = cv.take<long long>((size_t)k1 * n);
        mom = cv.take<double>((size_t)kVorMoments * n);
        start = cv.take<long long>((size_t)n);
        local = cv.take<unsigned long long>((size_t)n);
        tiles = cv.take<unsigned long long>((size_t)blocks_for(n));
        bad = cv.take<unsigned long long>(1);
        sync = cv.take<VorSync>(1);
    }
};

int rv_check(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind, long long n) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "num_samples must be > 0");
    if (n > 0x7fffffffLL - 1) return fail(PCU_B200_INVALID_ARGUMENT, "restricted Voronoi: at most 2^31 - 2 seeds, got %lld", n);
    return PCU_B200_OK;
}

// Carves the call's RvScratch and enqueues the per-face pass (corners, centroids, radii, faces out of range).
int rv_prepare(pcu_b200_workspace* ws, RvScratch& r, const double* v, long long nv, const void* f, long long m, int fkind,
               long long n, cudaStream_t stream) {
    r.n = n; r.m = m; r.k1 = (int)std::min<long long>(kRvK1, n);
    PCU_TRY(carve_scratch(ws, kRvd, stream, [&](Carver& cv) { r.carve(cv); }));
    PCU_CUDA(cudaMemsetAsync(r.bad, 0, sizeof(unsigned long long), stream));
    PCU_CUDA(cudaMemsetAsync(r.sync, 0, sizeof(VorSync), stream));
    PCU_LAUNCH(rv_face_kernel, blocks_for(m), kThreads, stream, v, nv, f, fkind, m, r.tri, r.cen, r.rad, r.bad);
    return PCU_B200_OK;
}

int rv_eval(pcu_b200_workspace* ws, const RvScratch& r, const double* x, VorSync* sync, double** mom_out, long long* passes,
            VorSync* seen, cudaStream_t stream) {
    const long long n = r.n, m = r.m;
    *mom_out = r.mom;
    PCU_TRY(knn_device<double>(ws, r.cen, m, x, n, 1, 1, r.fd2, r.fidx, nullptr, stream, nullptr, false));
    PCU_LAUNCH(rv_ball_kernel, blocks_for(m), kThreads, stream, (const double*)r.cen, (const double*)r.rad, (const double*)r.fd2,
               (const long long*)r.fidx, m, r.balls);
    PCU_TRY(knn_device<double>(ws, x, n, x, n, r.k1, 1, r.sd2, r.sidx, nullptr, stream, nullptr, false));
    MeshTree<RvBall> tree;   // in the arena, with its build's temporaries: nothing re-carves it before the pairs are out
    PCU_TRY(build_ball_tree(ws, r.balls, m, tree, stream));
    const unsigned sb = blocks_for(n);
    PCU_LAUNCH(rv_count_kernel, sb, kThreads, stream, x, n, m, (const MqScratch*)tree.sc, (const MqNode*)tree.nodes,
               (const RvBall*)tree.leaves, (const int*)tree.ids, r.local, r.tiles);
    PCU_LAUNCH(rv_tiles_kernel, 1, 1024, stream, r.tiles, (long long)sb, sync);
    PCU_TRY(read_record(sync, seen, stream));
    const long long P = seen->count;
    if (P == 0) {   // every face has zero area
        PCU_CUDA(cudaMemsetAsync(r.mom, 0, (size_t)n * kVorMoments * sizeof(double), stream));
        return PCU_B200_OK;
    }
    int *pseed, *pface; double* pmom; unsigned char* flag; unsigned* counts;
    const int rs = P > 0x7fffffffLL ? PCU_B200_OUT_OF_MEMORY : carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        pseed = cv.take<int>((size_t)P);
        pface = cv.take<int>((size_t)P);
        pmom = cv.take<double>((size_t)kVorMoments * P);
        flag = cv.take<unsigned char>((size_t)P);
        counts = cv.take<unsigned>(keep_count_words(P));
    });
    if (rs == PCU_B200_OUT_OF_MEMORY)
        return fail(PCU_B200_OUT_OF_MEMORY, "restricted Voronoi: %lld (face, seed) pairs do not fit (%zu bytes of scratch, at most "
                    "2^31 - 1 pairs)", P, (size_t)P * (8 + 8 * kVorMoments + 1));
    PCU_TRY(rs);
    PCU_LAUNCH(rv_emit_kernel, sb, kThreads, stream, x, n, m, (const MqScratch*)tree.sc, (const MqNode*)tree.nodes,
               (const RvBall*)tree.leaves, (const int*)tree.ids, (const unsigned long long*)r.local, (const unsigned long long*)r.tiles,
               r.start, pseed, pface);
    VorPass p{};
    p.x = x; p.x3 = x; p.n = n; p.count = P; p.nn_idx = r.sidx; p.nn_d2 = r.sd2; p.k = r.k1; p.list_is_all = r.k1 >= n;
    p.list_of_seed = 1; p.mom = pmom; p.uncert = flag; p.pair_seed = pseed; p.pair_face = pface; p.tri = r.tri;
    PCU_TRY(VorRestricted::launch(p, 0, stream));
    passes[0] += P;
    PCU_TRY(vor_fallback<VorRestricted>(ws, p, flag, counts, sync, passes, seen, stream));
    PCU_LAUNCH(rv_reduce_kernel, sb, kThreads, stream, (const long long*)r.start, n, P, (const double*)pmom, r.mom);
    return PCU_B200_OK;
}

int restricted_moments_device(pcu_b200_workspace* ws, const double* x, long long n, const double* v, long long nv, const void* f,
                              long long m, int fkind, double* out_moments, long long* passes, cudaStream_t stream) {
    RvScratch r;
    PCU_TRY(rv_prepare(ws, r, v, nv, f, m, fkind, n, stream));
    unsigned long long bad = 0;
    PCU_TRY(read_record(r.bad, &bad, stream));
    if (bad) return bad_corners(bad);
    double* mom; VorSync seen;
    PCU_TRY(rv_eval(ws, r, x, r.sync, &mom, passes, &seen, stream));
    PCU_CUDA(cudaMemcpyAsync(out_moments, mom, (size_t)n * kVorMoments * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return PCU_B200_OK;
}

// sample_mesh_lloyd: the first n samples of sample_mesh_random at `seed` (their fp64 positions) relaxed on the
// restricted cells, with no domain test for the Newton phase's trial points.  The initial sample reads the face CDF's
// record (one synchronisation) and fails as sample_mesh_random's caller does on faces out of range or a zero area.
int sample_mesh_lloyd_device(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind,
                             long long n, unsigned seed, int num_lloyd, int num_newton, double* out, double* energy_host,
                             int* iters_host, long long* passes, cudaStream_t stream) {
    RvScratch r;
    PCU_TRY(rv_prepare(ws, r, v, nv, f, m, fkind, n, stream));
    return lloyd_run<3>(
        ws, n, 0, num_lloyd, num_newton, out, energy_host, iters_host, stream,
        [&](double* x) -> int { return sample_mesh_positions(ws, v, nv, f, m, fkind, n, seed, x, stream); },
        [&](const double* x, VorSync* sync, double** mom, VorSync* seen) -> int {
            return rv_eval(ws, r, x, sync, mom, passes, seen, stream);
        });
}

}  // namespace

extern "C" {

int pcu_b200_voronoi_centroids(pcu_b200_workspace* ws, const double* centers, int64_t n, int dim, double* out_centroids,
                               double* out_moments, int64_t* out_passes, void* stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(vor_check(n, dim));
    if (n <= 0 || !centers || !out_centroids) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: n >= 1 seeds and non-null pointers required");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    const int rs = dim == 3 ? voronoi_centroids_device<3>(ws, centers, n, out_centroids, out_moments, passes, (cudaStream_t)stream)
                            : voronoi_centroids_device<2>(ws, centers, n, out_centroids, out_moments, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    return rs;
}
int pcu_b200_lloyd(pcu_b200_workspace* ws, int64_t n, int dim, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                   double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(vor_check(n, dim));
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "n must be a positive integer. Got n = %lld", (long long)n);
    if (!out_points) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    int steps = 0;
    const int rs = dim == 3 ? lloyd_device<3>(ws, n, seed, num_lloyd, num_newton, out_points, out_energy, &steps, passes, (cudaStream_t)stream)
                            : lloyd_device<2>(ws, n, seed, num_lloyd, num_newton, out_points, out_energy, &steps, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    if (out_newton_steps) *out_newton_steps = steps;
    return rs;
}

int pcu_b200_restricted_voronoi_moments(pcu_b200_workspace* ws, const double* seeds, int64_t n, const double* v, int64_t nv,
                                        const void* f, int64_t nf, int f_kind, double* out_moments, int64_t* out_passes, void* stream) {
    PCU_TRY(rv_check(ws, v, nv, f, nf, f_kind, n));
    if (!seeds || !out_moments) return fail(PCU_B200_INVALID_ARGUMENT, "null seeds or output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    const int rs = restricted_moments_device(ws, seeds, n, v, nv, f, nf, f_kind, out_moments, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    return rs;
}
int pcu_b200_sample_mesh_lloyd(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                               int64_t num_samples, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                               double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream) {
    PCU_TRY(rv_check(ws, v, nv, f, nf, f_kind, num_samples));
    if (!out_points) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    int steps = 0;
    const int rs = sample_mesh_lloyd_device(ws, v, nv, f, nf, f_kind, num_samples, seed, num_lloyd, num_newton, out_points, out_energy,
                                            &steps, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    if (out_newton_steps) *out_newton_steps = steps;
    return rs;
}

}  // extern "C"
