// pcu_b200.cu -- workspace, launch sequencing and the C ABI declared in include/pcu_b200.h.
//
// Host side of the H100 nearest-neighbour path.  It owns no algorithmic decisions that depend on
// the data: grid shapes, far-query lists and tie lists are produced and consumed on the device, so
// a device-pointer call enqueues a fixed sequence of launches and returns without synchronising.
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <functional>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/pcu_b200.h"
#include "host_util.h"
#include "staging.h"
#include "common.cuh"
#include "grid.cuh"
#include "search.cuh"
#include "nn1.cuh"
#include "topk.cuh"
#include "pyramid.cuh"
#include "kdreplay.cuh"
#include "compact.cuh"
#include "normals.cuh"
#include "morton.cuh"
#include "sinkhorn.cuh"
#include "voxel.cuh"
#include "dedup.cuh"
#include "poisson.cuh"
#include "meshsample.cuh"
#include "winding.cuh"
#include "raycast.cuh"
#include "sparse_voxels.cuh"
#include "voxelize.cuh"
#include "watertight.cuh"
#include "mesh_topology.cuh"
#include "orient.cuh"
#include "laplacian.cuh"
#include "voronoi.cuh"
#include "rvd.cuh"

using namespace pcu;

namespace {

thread_local std::string g_error;
std::atomic<long long> g_launches{0};

// Blocks of kThreads threads for one thread per row.
inline unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

int fail(int status, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_error = buf;
    return status;
}

// The library carries sm_90a code only, and architecture-specific code runs on compute capability 9.0 alone.
bool runs_this_build(int device) {
    int major = 0, minor = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device) != cudaSuccess ||
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return major == 9 && minor == 0;
}

#define PCU_CUDA(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess)                                                                          \
            return fail(e__ == cudaErrorMemoryAllocation ? PCU_B200_OUT_OF_MEMORY : PCU_B200_CUDA_ERROR, \
                        "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__);    \
    } while (0)

#define PCU_TRY(expr)                      \
    do {                                   \
        int s__ = (expr);                  \
        if (s__ != PCU_B200_OK) return s__; \
    } while (0)

#define PCU_LAUNCH(kernel, grid, block, stream, ...)                   \
    do {                                                               \
        kernel<<<grid, block, 0, stream>>>(__VA_ARGS__);               \
        g_launches.fetch_add(1, std::memory_order_relaxed);            \
        PCU_CUDA(cudaGetLastError());                                  \
    } while (0)

// Launch with programmatic stream serialisation: the kernel (which starts with grid_dependency_wait())
// may have its CTAs scheduled while its predecessor in the stream is still draining.
template <typename... Params, typename... Args>
int launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const Args&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    PCU_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return PCU_B200_OK;
}

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

// The workspace's device scratch blocks (carve_scratch).  Every call carves the blocks it uses afresh, so buffers that
// must outlive a nested call live in a block that the nested call does not carve.
enum Scratch {
    kArena,   // the device-pointer entry points' own scratch; any nested call may re-carve it
    kIo,      // device copies of a host entry point's inputs and outputs: outlive the device call they are passed to
    kAux,     // intermediate results (normals, Poisson disk) that outlive a nested call's re-carving of the arena
    kMesh,    // the face CDF and dense samples of mesh Poisson-disk sampling, which outlive the point-cloud Poisson-disk
              // call it makes (that one re-carves the arena and aux)
    kVorList, // the Voronoi cells' fallback passes (rows, queries, longer neighbour lists), sized once the first pass is done
    kLloyd,   // the points, L-BFGS history and sync record of a Lloyd relaxation, which outlive every cell evaluation
    kRvd,     // the faces and the per-seed buffers of restricted Voronoi cells, which outlive every cell evaluation of a call
    kScratchBlocks
};
static const char* const kScratchName[kScratchBlocks] = {"scratch", "staging", "intermediate scratch", "mesh-sampling scratch",
                                                         "Voronoi fallback scratch", "Lloyd scratch", "restricted Voronoi scratch"};

struct pcu_b200_workspace {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    unsigned char* block[kScratchBlocks] = {};   // indexed by Scratch
    size_t block_bytes[kScratchBlocks] = {};
    pcu_b200_options opts{};
    int sm_count = 132;                  // set from the device in pcu_b200_workspace_create
    // optional per-stage timing (bench.py's roofline pass): events recorded on the launching stream
    unsigned smem_raised = 0;            // kernel instantiations whose dynamic shared-memory limit has been raised (raise_smem_limit)
    // grid-sizing feedback: the kernels leave {cell_cap, non-empty cells, n, valid, unsettled queries, queries, valid, -}
    // per cloud in this
    // host-mapped buffer; the next call with the same shapes reads it (no synchronisation: a hint only)
    volatile unsigned* hint_host = nullptr;
    unsigned* hint_dev = nullptr;
    long long hint_key[5] = {0, 0, 0, 0, 0};   // n, m, k, sizeof(T), batch of the call the hints belong to
    float cell_mult[2] = {1.f, 1.f};           // current refinement of the two clouds' grids (cells per point x this)
    float cell_mult_ceiling[2] = {32.f, 32.f}; // lowered when a refinement left too many queries unsettled
    cudaStream_t copy_stream = nullptr;  // host entry points: the H2D copies run here, the kernels on own_stream
    cudaEvent_t arrived[2] = {};         // recorded on copy_stream behind each cloud's copy
    unsigned char* host_slot = nullptr;  // 4 KB of pinned host memory: small results land here, then in the caller's buffers
    const unsigned* replay_overflows = nullptr;   // device counter of the last KNN call's tie replay (null: none ran)
    cudaStream_t last_stream = nullptr;  // stream of the previous call (see adopt_stream)
    bool has_last_stream = false;
    cudaEvent_t handover = nullptr;
    bool profiling = false;
    cudaEvent_t marks[11] = {};   // 0 .. 8: stage boundaries of a device call; 9 / 10: before the H2D / after the D2H of a host call
    int marks_used = 0;
    bool host_marks = false;      // marks 9 and 10 belong to the last call
    HostStager* stager = nullptr; // pinned ring + copy threads for pageable inputs of the host entry points (created on first use)
};

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
// A mesh whose tree is built once (pcu_b200_mesh_prepare_*), or a point cloud's surfels (pcu_b200_surfel_prepare_*):
// the tree's header, nodes and leaves (carve_mesh_tree, no far-field data) live in one private device block.
struct pcu_b200_mesh {
    int device = 0;
    int is_f64 = 0;
    long long nf = 0;               // faces, or points
    int subdivs = 0;                // > 0: a surfel tree of fans of this many triangles (leaves SfWord, ids)
    unsigned char* block = nullptr;
    size_t bytes = 0;
    MqScratch* sc = nullptr;
    MqNode* nodes = nullptr;
    const void* leaves = nullptr;   // Pt<float> or Pt<double> by is_f64, or SfWord
    const int* ids = nullptr;       // surfels: the point id of each leaf
};
// What the stream-ordered handles below share: the device and stream they were prepared on.  Deleting a handle releases
// its blocks in the order of that stream.
struct StreamHandle {
    int device = 0;
    cudaStream_t stream = nullptr;
    void release(unsigned char* block) const { if (block) cudaFreeAsync(block, stream); }
};
// Marching cubes between pcu_b200_marching_cubes_prepare_* and _emit: the inputs, the cube block (case bytes, tile
// offsets, counts; sized by m) and the slot block (run of every slot, vertex id of every run, owner flags; sized by the
// slot count).
struct pcu_b200_marching_cubes : StreamHandle {
    int t_f64 = 0, s_f64 = 0, width = 4;   // coordinates, scalars, bytes per cube index
    const void* scalars = nullptr;
    const void* coords = nullptr;
    const void* idx = nullptr;
    long long n = 0, m = 0;
    double iso = 0.0;                       // T(S(isovalue)), exactly
    long long slots = 0, faces = 0, verts = 0;
    unsigned char* cube_block = nullptr;
    unsigned char* slot_block = nullptr;
    unsigned char* cases = nullptr;
    unsigned* tile_sum = nullptr;
    unsigned long long* tile_slot0 = nullptr;
    unsigned long long* tile_face0 = nullptr;
    McCounts* counts = nullptr;
    unsigned* slot_run = nullptr;
    unsigned* run_vid = nullptr;
    unsigned char* owner = nullptr;
    ~pcu_b200_marching_cubes() { release(cube_block); release(slot_block); }
};
// Voxelization between pcu_b200_voxelize_prepare_* and _emit: the sorted codes, their run heads and the heads' block
// offsets, in one block.
struct pcu_b200_voxelize : StreamHandle {
    long long recs = 0, n = 0;              // accepted (face, voxel) pairs; distinct voxels
    unsigned char* block = nullptr;
    const McRec* sorted = nullptr;
    unsigned char* head = nullptr;
    unsigned* offsets = nullptr;
    ~pcu_b200_voxelize() { release(block); }
};
// Watertight remeshing between pcu_b200_make_mesh_watertight_prepare_* and _emit: the result in one block, vertices in
// fp64 and faces in int32, which emit converts to the input's types.
struct pcu_b200_watertight : StreamHandle {
    int t_f64 = 0, fkind = 0, depth = 0;
    long long nv = 0, nf = 0;
    unsigned char* block = nullptr;
    const double* x = nullptr;
    const int* faces = nullptr;
    ~pcu_b200_watertight() { release(block); }
};
// Connected components between pcu_b200_connected_components_prepare and _emit: int32 labels and counts in one block
// (cv over n = max(f) + 1 vertices, cf over m faces, nv and nf over the k components, sized n).
struct pcu_b200_components : StreamHandle {
    int fkind = 0;
    long long n = 0, m = 0, k = 0;
    unsigned char* block = nullptr;
    const int* cv = nullptr;
    const int* cf = nullptr;
    const int* nv = nullptr;
    const int* nf = nullptr;
    ~pcu_b200_components() { release(block); }
};
// A sparse voxel grid's code set between pcu_b200_sparse_grid_*_prepare and pcu_b200_sparse_grid_emit: the sorted code
// records, their run heads, the heads' block offsets and the count record, in one block.  Prepared from points, by a
// dilation round or from a grid's cube corners; the mode says what emit writes.
struct SvgCounts { long long rows; unsigned long long bad; };
struct pcu_b200_sparse_grid : StreamHandle {
    int mode = 0;                           // SvgMode
    int out_kind = 0;                       // dilation: the grid's index kind; hex mesh: vertices in double (1) or float (0)
    const void* grid = nullptr;             // dilation: the input rows, which emit copies ahead of the new ones
    long long n = 0;                        // input rows (points or voxels)
    long long recs = 0;                     // sorted records
    long long rows = 0;                     // distinct codes: grid rows, new rows or vertices
    SvgPlace place{};
    unsigned char* block = nullptr;
    const McRec* sorted = nullptr;
    unsigned char* head = nullptr;          // nullptr: the records are distinct already (dilation)
    unsigned* offsets = nullptr;
    SvgCounts* counts = nullptr;
    ~pcu_b200_sparse_grid() { release(block); }
};
template <typename T> KdReplayBuffers<T>& cloud_tree(pcu_b200_cloud* c);
template <> KdReplayBuffers<float>& cloud_tree<float>(pcu_b200_cloud* c) { return c->kd32; }
template <> KdReplayBuffers<double>& cloud_tree<double>(pcu_b200_cloud* c) { return c->kd64; }

#define PCU_STAGE_NAMES "descriptors", "bbox+grid", "slab_count", "partition", "cell_sort", "search", "search_far", "finalize", "h2d", "d2h"

namespace {

// Makes ws->device current for the duration of an entry point and puts the caller's device back on every
// exit path (a torch program with cuda:0 current that passes cuda:1 tensors keeps cuda:0 current).
struct DeviceGuard {
    int previous = -1;
    bool switched = false;
    cudaError_t status = cudaSuccess;
    explicit DeviceGuard(int device) {
        status = cudaGetDevice(&previous);
        if (status == cudaSuccess && previous != device) {
            status = cudaSetDevice(device);
            switched = status == cudaSuccess;
        }
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(previous); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define PCU_ON_DEVICE(ws)                                                                              \
    DeviceGuard device_guard__((ws)->device);                                                          \
    if (device_guard__.status != cudaSuccess)                                                          \
        return fail(PCU_B200_CUDA_ERROR, "cudaSetDevice(%d) failed: %s", (ws)->device, cudaGetErrorString(device_guard__.status))

// A workspace serves one stream at a time.  When a call arrives on another stream than the previous one,
// the new stream is made to wait (on the device) for everything the previous call enqueued: the scratch is shared.
int adopt_stream(pcu_b200_workspace* ws, cudaStream_t stream) {
    if (ws->has_last_stream && ws->last_stream != stream) {
        if (!ws->handover) PCU_CUDA(cudaEventCreateWithFlags(&ws->handover, cudaEventDisableTiming));
        PCU_CUDA(cudaEventRecord(ws->handover, ws->last_stream));
        PCU_CUDA(cudaStreamWaitEvent(stream, ws->handover, 0));
    }
    ws->last_stream = stream;
    ws->has_last_stream = true;
    return PCU_B200_OK;
}

// Scratch grows with stream-ordered allocation: the old block is released and the new one obtained in the
// order of `stream`, so earlier calls still queued there keep their memory until they are done and neither
// the host nor the rest of the device is synchronised.
int grow_block(unsigned char*& block, size_t& have, size_t bytes, cudaStream_t stream, const char* what) {
    if (bytes <= have) return PCU_B200_OK;
    if (block) {
        PCU_CUDA(cudaFreeAsync(block, stream));
        block = nullptr;
        have = 0;
    }
    const size_t want = align_up(bytes + bytes / 8, 1 << 20);
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, want, stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PCU_B200_OUT_OF_MEMORY, "cudaMallocAsync of %zu bytes of %s failed: %s", want, what, cudaGetErrorString(e));
    }
    block = (unsigned char*)p;
    have = want;
    return PCU_B200_OK;
}

// Runs `carve(Carver&)` from `base` (a null base only measures) and returns the bytes it took.
template <class F>
size_t carve_at(unsigned char* base, F&& carve) {
    Carver cv(base);
    carve(cv);
    return cv.off;
}

// Carves a call's buffers out of scratch block `which`: measures them, hands the workspace over to `stream` (the block
// may still be in use by work queued on the previous stream), grows the block in the order of `stream`, then carves.
// `carve` assigns the buffers to the caller's variables; it runs twice, first from a null base.
template <class F>
int carve_scratch(pcu_b200_workspace* ws, Scratch which, cudaStream_t stream, F&& carve) {
    const size_t bytes = carve_at(nullptr, carve);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(grow_block(ws->block[which], ws->block_bytes[which], bytes, stream, kScratchName[which]));
    carve_at(ws->block[which], carve);
    return PCU_B200_OK;
}

void mark(pcu_b200_workspace* ws, int index, cudaStream_t stream) {
    if (!ws->profiling) return;
    cudaEventRecord(ws->marks[index], stream);
    if (index <= 8) ws->marks_used = index + 1;
    if (index == 0) ws->host_marks = false;
    if (index == 10) ws->host_marks = true;
}

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

// ---- k nearest neighbours ---------------------------------------------------------------------
template <typename T>
int knn_device(pcu_b200_workspace* ws, const T* query, long long n, const T* dataset, long long m, int k, int squared,
               T* out_dist, long long* out_idx, long long* out_n_tied, cudaStream_t stream, pcu_b200_cloud* prepared = nullptr,
               bool tie_replay = true) {
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

// ---- ordered compaction (compact.cuh) --------------------------------------------------------------
// Words of the block-count buffer that compacting n flags takes: one per block of keep_count_kernel.
inline size_t keep_count_words(long long n) { return blocks_for(n); }

// Enqueues the first two steps of compact.cuh over n flags: the kept rows of every block into `counts`
// (keep_count_words(n) words), scanned in place into the blocks' offsets, and the total into *out_count (device memory).
// The caller's emit kernel follows, with blocks_for(n) blocks of kThreads threads.
int enqueue_keep_offsets(const unsigned char* keep, long long n, unsigned* counts, long long* out_count, cudaStream_t stream) {
    const unsigned nblocks = blocks_for(n);
    PCU_LAUNCH(keep_count_kernel, nblocks, kThreads, stream, keep, n, counts);
    PCU_LAUNCH(keep_offsets_kernel, 1, 1024, stream, counts, (long long)nblocks, out_count);
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
    PCU_LAUNCH(keep_rows_kernel<int>, blocks_for(n), kThreads, stream, (const unsigned char*)s.keep, n, (const unsigned*)counts, out_idx);
    mark(ws, 7, stream);
    mark(ws, 8, stream);
    return PCU_B200_OK;
}

// ---- mesh sampling and barycentric interpolation (sample_mesh_random / sample_mesh_poisson_disk) -----------------
int mesh_check(const void* v, long long nv, const void* f, long long m, int fkind) {
    if (!v || !f || nv <= 0 || m <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements: v and f must have shape (n, 3) and (m, 3) (n, m > 0)");
    if (m > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "mesh sampling: at most 2^31 - 1 faces, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

inline long long mesh_tiles(long long m) { return (m + kMeshScanTile - 1) / kMeshScanTile; }

// The face CDF of meshsample.cuh: areas, then the three-launch scan.  `cdf` (m words), `tiles` (one word per scan
// tile) and `sc` are carved by the caller; {W, S, bad} land in *out.
template <typename T>
int enqueue_mesh_cdf(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, int fkind, long long m,
                     unsigned long long* cdf, unsigned long long* tiles, MeshScratch* sc, MeshArea* out, cudaStream_t stream) {
    PCU_CUDA(cudaMemsetAsync(sc, 0, sizeof(MeshScratch), stream));
    const unsigned blocks = (unsigned)std::min<long long>((m + kThreads - 1) / kThreads, (long long)ws->sm_count * 8);
    PCU_LAUNCH((mesh_area_kernel<T>), blocks, kThreads, stream, v, nv, f, fkind, m, cdf, sc);
    PCU_LAUNCH(mesh_cdf_reduce_kernel, (unsigned)mesh_tiles(m), kMeshScanThreads, stream, (const unsigned long long*)cdf, m,
               (const MeshScratch*)sc, tiles);
    PCU_LAUNCH(mesh_cdf_tiles_kernel, 1, 1024, stream, tiles, mesh_tiles(m), m, (const MeshScratch*)sc, out);
    PCU_LAUNCH(mesh_cdf_scan_kernel, (unsigned)mesh_tiles(m), kMeshScanThreads, stream, cdf, m, (const MeshScratch*)sc,
               (const unsigned long long*)tiles);
    return PCU_B200_OK;
}

struct MeshCdfScratch {
    unsigned long long* cdf;
    unsigned long long* tiles;
    MeshScratch* sc;
    MeshArea* area;       // the caller's, or this one when the caller passes none
    void carve(Carver& cv, long long m) {
        cdf = cv.take<unsigned long long>((size_t)m);
        tiles = cv.take<unsigned long long>((size_t)mesh_tiles(m));
        sc = cv.take<MeshScratch>(1);
        area = cv.take<MeshArea>(1);
    }
};

template <typename T>
int mesh_area_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, MeshArea* out,
                     cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (!out) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshCdfScratch ms;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { ms.carve(cv, m); }));
    return enqueue_mesh_cdf<T>(ws, v, nv, f, fkind, m, ms.cdf, ms.tiles, ms.sc, out, stream);
}

template <typename T>
int sample_mesh_random_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, long long n,
                              unsigned seed, void* out_fidx, T* out_bc, MeshArea* out_area, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "num_samples must be positive");
    if (!out_fidx || !out_bc) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshCdfScratch ms;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { ms.carve(cv, m); }));
    MeshArea* area = out_area ? out_area : ms.area;
    PCU_TRY(enqueue_mesh_cdf<T>(ws, v, nv, f, fkind, m, ms.cdf, ms.tiles, ms.sc, area, stream));
    const unsigned blocks = (unsigned)std::min<long long>((n + kThreads - 1) / kThreads, (long long)ws->sm_count * 16);
    PCU_LAUNCH((mesh_sample_kernel<T>), blocks, kThreads, stream, (const unsigned long long*)ms.cdf, m, (const MeshArea*)area,
               (unsigned long long)seed, n, (const int*)nullptr, (const long long*)nullptr, v, nv, f, fkind, out_fidx,
               (fkind & 1), out_bc, (T*)nullptr);
    return PCU_B200_OK;
}

// Dense samples (positions only) -> the point-cloud Poisson-disk selection of poisson.cuh at the same seed -> the
// kept rows' faces and coordinates, re-evaluated from their sample indices.  The CDF, the dense positions and the kept
// rows live in kMesh: poisson_disk_device carves the arena and aux for itself.
template <typename T>
int sample_mesh_poisson_disk_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind,
                                    double radius, long long n_dense, unsigned seed, void* out_fidx, T* out_bc, long long* out_count,
                                    cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (!(radius > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid radius (%f) must be greater than 0.", radius);
    if (n_dense <= 0 || n_dense > 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "the dense sample must have 1 .. 2^31 - 1 rows, got %lld", n_dense);
    if (!out_fidx || !out_bc || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshCdfScratch ms;
    T* pos;
    int* kept;
    PCU_TRY(carve_scratch(ws, kMesh, stream, [&](Carver& cv) {
        ms.carve(cv, m);
        pos = cv.take<T>((size_t)3 * n_dense);
        kept = cv.take<int>((size_t)n_dense);
    }));
    PCU_TRY(enqueue_mesh_cdf<T>(ws, v, nv, f, fkind, m, ms.cdf, ms.tiles, ms.sc, ms.area, stream));
    const unsigned blocks = (unsigned)std::min<long long>((n_dense + kThreads - 1) / kThreads, (long long)ws->sm_count * 16);
    PCU_LAUNCH((mesh_sample_kernel<T>), blocks, kThreads, stream, (const unsigned long long*)ms.cdf, m, (const MeshArea*)ms.area,
               (unsigned long long)seed, n_dense, (const int*)nullptr, (const long long*)nullptr, v, nv, f, fkind, (void*)nullptr, 0,
               (T*)nullptr, pos);
    PCU_TRY(poisson_disk_device<T>(ws, pos, n_dense, radius, seed, kept, out_count, nullptr, stream));
    PCU_LAUNCH((mesh_sample_kernel<T>), blocks, kThreads, stream, (const unsigned long long*)ms.cdf, m, (const MeshArea*)ms.area,
               (unsigned long long)seed, n_dense, (const int*)kept, (const long long*)out_count, v, nv, f, fkind, out_fidx,
               (fkind & 1), out_bc, (T*)nullptr);
    return PCU_B200_OK;
}

template <typename A, typename B, typename P>
int interpolate_launch(pcu_b200_workspace* ws, const void* f, long long m, int fkind, const void* fi, long long n, int fikind,
                       const void* bc, const void* attr, long long nv, long long dim, P* out, unsigned long long* out_bad,
                       cudaStream_t stream) {
    const long long work = n * dim;
    const unsigned blocks = (unsigned)std::min<long long>((work + kThreads - 1) / kThreads, (long long)ws->sm_count * 16);
    PCU_LAUNCH((interpolate_bary_kernel<A, B, P>), blocks, kThreads, stream, f, m, fkind, fi, n, fikind, (const B*)bc,
               (const A*)attr, nv, dim, out, out_bad);
    return PCU_B200_OK;
}

template <typename P>
int interpolate_device(pcu_b200_workspace* ws, const void* f, long long m, int fkind, const void* fi, long long n, int fikind,
                       const void* bc, int bc_is_f64, const void* attr, int attr_is_f64, long long nv, long long dim, P* out,
                       unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!f || !fi || !bc || !attr || !out || !out_bad) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (m <= 0 || nv <= 0 || n <= 0 || dim <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "interpolate_barycentric: empty input");
    if (fkind < kIdxI32 || fkind > kIdxU64 || fikind < kIdxI32 || fikind > kIdxU64)
        return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind");
    if (sizeof(P) == 4 && (bc_is_f64 || attr_is_f64))
        return fail(PCU_B200_INVALID_ARGUMENT, "a float64 input promotes the result to float64: use the _f64 entry point");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_CUDA(cudaMemsetAsync(out_bad, 0, sizeof(unsigned long long), stream));
    if constexpr (sizeof(P) == 4) {
        return interpolate_launch<float, float, float>(ws, f, m, fkind, fi, n, fikind, bc, attr, nv, dim, out, out_bad, stream);
    } else {
        if (attr_is_f64)
            return bc_is_f64 ? interpolate_launch<double, double, P>(ws, f, m, fkind, fi, n, fikind, bc, attr, nv, dim, out, out_bad, stream)
                             : interpolate_launch<double, float, P>(ws, f, m, fkind, fi, n, fikind, bc, attr, nv, dim, out, out_bad, stream);
        return bc_is_f64 ? interpolate_launch<float, double, P>(ws, f, m, fkind, fi, n, fikind, bc, attr, nv, dim, out, out_bad, stream)
                         : interpolate_launch<float, float, P>(ws, f, m, fkind, fi, n, fikind, bc, attr, nv, dim, out, out_bad, stream);
    }
}

// ---- radix sort of records (sort.cuh) ----------------------------------------------------------------------
// The buffers of one sort of n records.  The caller writes the records to `a`.
template <typename Rec>
struct SortScratch {
    Rec *a, *b;                    // the sort's two record buffers
    unsigned* hist;                // [bin][tile] digit counts
    unsigned long long* totals;    // per bin
    unsigned* base;                // per bin
    int* constant;                 // the pass's digit is the same in every record
    static unsigned tiles(long long n) { return (unsigned)((n + kSortTile - 1) / kSortTile); }
    void carve(Carver& cv, long long n) {
        a = cv.take<Rec>((size_t)n);
        b = cv.take<Rec>((size_t)n);
        hist = cv.take<unsigned>((size_t)kSortBins * tiles(n));
        totals = cv.take<unsigned long long>(kSortBins);
        base = cv.take<unsigned>(kSortBins);
        constant = cv.take<int>(1);
    }
};

// Stable LSD radix sort of the `n` records in s.a between the two buffers; returns the buffer holding the sorted records.
// key_bits > 0: only the low key_bits bits of each key word can be non-zero, and the passes over the bytes above them
// are skipped.
template <typename Rec>
int radix_sort_records(const SortScratch<Rec>& s, long long n, int words, cudaStream_t stream, Rec** sorted, int key_bits = 0) {
    const unsigned ntiles = SortScratch<Rec>::tiles(n);
    const int bits = key_bits > 0 ? key_bits : (int)sizeof(s.a->key[0]) * 8;
    Rec *in = s.a, *out = s.b;
    for (int w = words - 1; w >= 0; --w)          // least significant word first
        for (int shift = 0; shift < bits; shift += 8) {
            PCU_LAUNCH((sort_hist_kernel<Rec>), ntiles, kSortThreads, stream, (const Rec*)in, n, w, shift, s.hist, ntiles);
            PCU_LAUNCH(sort_scan_rows, kSortBins, kSortThreads, stream, s.hist, ntiles, s.totals);
            PCU_LAUNCH(sort_scan_bins, 1, kSortBins, stream, (const unsigned long long*)s.totals, n, s.base, s.constant);
            PCU_LAUNCH((sort_scatter_kernel<Rec>), ntiles, kSortThreads, stream, (const Rec*)in, out, n, w, shift, (const unsigned*)s.hist,
                       ntiles, (const unsigned*)s.base, (const int*)s.constant);
            std::swap(in, out);
        }
    *sorted = in;
    return PCU_B200_OK;
}

// ---- duplicate removal (SURVEY.md 8f N2, src/remove_duplicates.cpp) ----------------------------------------
// faces == nullptr: points only.  out_pts (n, 3), out_svi (n) and out_faces (nf, cols) are sized for the worst case;
// out_counts[0] = unique points, [1] = surviving faces, [2] = faces with a corner out of range (an error for the caller).
template <typename T, typename I>
int dedup_device(pcu_b200_workspace* ws, const T* pts, long long n, double epsilon, const I* faces, long long nf, int cols,
                 T* out_pts, int* out_svi, int* out_svj, I* out_faces, long long* out_counts, cudaStream_t stream) {
    using Rec = typename DedupRec<T>::type;
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld rows)", n);
    if (!out_pts || !out_svi || !out_svj || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    if (faces != nullptr && (nf < 0 || cols <= 0 || cols > 16 || (nf > 0 && !out_faces)))
        return fail(PCU_B200_INVALID_ARGUMENT, "faces must be an (m, c) array with 1 <= c <= 16");
    if (nf >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "too many faces (%lld)", nf);
    PCU_ON_DEVICE(ws);
    struct { SortScratch<Rec> sort; unsigned char* head; unsigned* counts; unsigned char* fkeep; unsigned* fcounts; unsigned* bad; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.head = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
        sc.fkeep = cv.take<unsigned char>((size_t)std::max<long long>(1, nf));
        sc.fcounts = cv.take<unsigned>(std::max<size_t>(1, faces ? keep_count_words(nf) : 0));
        sc.bad = cv.take<unsigned>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 3 * sizeof(long long), stream));
    PCU_LAUNCH((dedup_keys_kernel<T>), blocks_for(n), kThreads, stream, pts, n, (T)epsilon, sc.sort.a);
    Rec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 3, stream, &sorted));
    PCU_LAUNCH((dedup_heads_kernel<Rec>), blocks_for(n), kThreads, stream, (const Rec*)sorted, n, sc.head);
    PCU_TRY(enqueue_keep_offsets(sc.head, n, sc.counts, out_counts, stream));
    PCU_LAUNCH((dedup_emit_kernel<T, Rec>), blocks_for(n), kThreads, stream, (const Rec*)sorted, n, (const unsigned char*)sc.head,
               (const unsigned*)sc.counts, pts, out_pts, out_svi, out_svj);
    if (faces != nullptr && nf > 0) {
        PCU_CUDA(cudaMemsetAsync(sc.bad, 0, sizeof(unsigned), stream));
        PCU_LAUNCH((dedup_faces_flag_kernel<I>), blocks_for(nf), kThreads, stream, faces, nf, cols, n, (const int*)out_svj, sc.fkeep, sc.bad);
        PCU_TRY(enqueue_keep_offsets(sc.fkeep, nf, sc.fcounts, out_counts + 1, stream));
        PCU_LAUNCH((dedup_faces_emit_kernel<I>), blocks_for(nf), kThreads, stream, faces, nf, cols, (const int*)out_svj,
                   (const unsigned char*)sc.fkeep, (const unsigned*)sc.fcounts, out_faces);
        PCU_LAUNCH(widen_counter_kernel, 1, 1, stream, sc.bad, out_counts + 2);
    }
    return PCU_B200_OK;
}

template <typename T>
int dedup_dispatch(pcu_b200_workspace* ws, const T* pts, long long n, double epsilon, const void* faces, long long nf, int cols,
                   int faces_are_i64, T* out_pts, int* out_svi, int* out_svj, void* out_faces, long long* out_counts, cudaStream_t stream) {
    if (faces_are_i64)
        return dedup_device<T, long long>(ws, pts, n, epsilon, (const long long*)faces, nf, cols, out_pts, out_svi, out_svj,
                                          (long long*)out_faces, out_counts, stream);
    return dedup_device<T, int>(ws, pts, n, epsilon, (const int*)faces, nf, cols, out_pts, out_svi, out_svj, (int*)out_faces, out_counts, stream);
}

// ---- closest points, winding numbers and signed distances on a mesh or a point cloud (meshquery.cuh, winding.cuh) ----
// The tree over the valid faces, or over the points, built per call by the one builder below, then one traversal per
// query.  The count of faces with a corner out of range lands in *out_bad; the caller reads it (the call's one
// synchronisation) and raises when it is not zero.
template <typename L>
struct MeshTree {
    MqScratch* sc;
    MqNode* nodes;
    L* leaves;
    WnNode* wn;   // far-field data per node (with `moments` only)
    int* ids;     // surfel leaves: the point id of each leaf
};

// The arrays a built tree is queried through: the header, the nodes, the leaves, with `moments` the far-field data and
// for surfels (fans of `subdivs` triangles) the leaves' point ids.
template <typename L>
void carve_mesh_tree(Carver& cv, long long m, bool moments, MeshTree<L>& t, int subdivs = 0) {
    const long long inner = std::max<long long>(1, m - 1);
    t.sc = cv.take<MqScratch>(1);
    t.nodes = cv.take<MqNode>((size_t)inner);
    t.leaves = cv.take<L>((size_t)(kSurfelLeaf<L> ? sf_words(subdivs) : (kPointLeaf<L> || kBallLeaf<L> ? 1 : 3)) * m);
    t.wn = moments ? cv.take<WnNode>((size_t)inner) : nullptr;
    t.ids = kSurfelLeaf<L> || kBallLeaf<L> ? cv.take<int>((size_t)m) : nullptr;
}

// The surfel table of DESIGN.md §3: theta_j = ((float)j / ((float)(s + 1) - 1)) (float)pi 2 in fp32, as the reference
// computes it, then cs[2 j] = fl32(cos theta_j) and cs[2 j + 1] = fl32(sin theta_j) from the C library in fp64.
void surfel_table(int s, float* cs) {
    const float den = (float)(s + 1) - 1.0f;
    for (int j = 0; j < s; ++j) {
        const float theta = ((float)j / den) * (float)M_PI * 2.0f;
        cs[2 * j] = (float)std::cos((double)theta);
        cs[2 * j + 1] = (float)std::sin((double)theta);
    }
}

// Bytes of a surfel source record in device memory: the SfSrc, then its table.
size_t surfel_src_bytes(int s) { return align_up(sizeof(SfSrc)) + sizeof(float) * 2 * (size_t)s; }

// Writes the SfSrc of (n, r, s, boxes) and its table to `dev` (surfel_src_bytes(s) bytes of device memory) in the order
// of `stream`, through the parameters of sf_upload_kernel (no host buffer is copied, so nothing synchronises), and
// returns the record as the kernels take it by value.
int upload_surfel_src(unsigned char* dev, const void* n, const void* r, int s, MqBox* boxes, cudaStream_t stream, SfSrc& src) {
    std::vector<float> cs(2 * (size_t)s);
    surfel_table(s, cs.data());
    src.n = n; src.r = r; src.s = s; src.boxes = boxes;
    src.cs = reinterpret_cast<const float*>(dev + align_up(sizeof(SfSrc)));
    SfUpload u;
    u.src = src;
    for (size_t at = 0; at < cs.size(); at += kSfChunk) {
        u.dst_src = at == 0 ? reinterpret_cast<SfSrc*>(dev) : nullptr;
        u.dst = const_cast<float*>(src.cs) + at;
        u.count = (int)std::min<size_t>(kSfChunk, cs.size() - at);
        std::memcpy(u.v, cs.data() + at, sizeof(float) * u.count);
        PCU_LAUNCH(sf_upload_kernel, 1, kThreads, stream, u);
    }
    return PCU_B200_OK;
}

// Carves the build's temporaries from the arena, the tree itself (carve_mesh_tree) from `keep` or, when it is null, from
// the arena too, and enqueues the build over the leaf kind L (meshquery.cuh): bounds, codes, sort, leaves, nodes, for
// faces the refit and, with `moments`, the centre, radius and moment passes of winding.cuh.  Face leaves (L = Pt<T>)
// are built from the mesh (v, nv, f, fkind) and the count of invalid faces lands in *out_bad; point leaves (L = WnPoint)
// from the points v, normals n and areas a, always with moments; surfel leaves (L = SfWord) from the points v, normals
// n, radii a and `subdivs`, without moments, their non-finite fans counted in the header only; ball leaves (L = RvBall)
// from the (m, 4) balls v, without moments, the balls without a radius counted in the header only.  The caller has checked
// the input (m >= 1) and made the device current.
template <typename T, typename L>
int build_mesh_tree(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, bool moments,
                    unsigned long long* out_bad, cudaStream_t stream, MeshTree<L>& tree, unsigned char* keep = nullptr,
                    const T* n = nullptr, const T* a = nullptr, int subdivs = 0) {
    constexpr bool points = kPointLeaf<L>, surfels = kSurfelLeaf<L>;
    const long long inner = std::max<long long>(1, m - 1);
    struct { SortScratch<MqRec> sort; int* node_parent; int* leaf_parent; int* arrivals; MqBox* boxes; unsigned char* src; MqBox* in_boxes; } s;
    MeshTree<L> t;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        s.sort.carve(cv, m);
        s.node_parent = cv.take<int>((size_t)inner);
        s.leaf_parent = cv.take<int>((size_t)m);
        s.arrivals = cv.take<int>((size_t)inner);
        s.boxes = points ? nullptr : cv.take<MqBox>((size_t)m);
        s.src = surfels ? cv.take<unsigned char>(surfel_src_bytes(subdivs)) : nullptr;
        s.in_boxes = surfels ? cv.take<MqBox>((size_t)m) : nullptr;
        if (!keep) carve_mesh_tree<L>(cv, m, moments, t, subdivs);
    }));
    if (keep) carve_at(keep, [&](Carver& cv) { carve_mesh_tree<L>(cv, m, moments, t, subdivs); });
    SfSrc src{};
    if constexpr (surfels) {   // the bounds and codes passes find the surfels' normals, radii and table through f
        PCU_TRY(upload_surfel_src(s.src, n, a, subdivs, s.in_boxes, stream, src));
        f = s.src;
    }
    PCU_CUDA(cudaMemsetAsync(t.sc->scene, 0x7f, 3 * sizeof(int), stream));       // min: the image of a huge float
    PCU_CUDA(cudaMemsetAsync(t.sc->scene + 3, 0x80, 3 * sizeof(int), stream));   // max: the image of a huge negative one
    PCU_CUDA(cudaMemsetAsync(&t.sc->bad, 0, sizeof(unsigned long long), stream));
    const unsigned fblocks = blocks_for(m);
    PCU_LAUNCH((mq_bounds_kernel<L, T>), (unsigned)std::min<long long>(fblocks, (long long)ws->sm_count * 8), kThreads, stream,
               v, nv, f, fkind, m, t.sc);
    PCU_LAUNCH((mq_codes_kernel<L, T>), fblocks, kThreads, stream, v, nv, f, fkind, m, (const MqScratch*)t.sc, s.sort.a);
    MqRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(s.sort, m, 1, stream, &sorted));
    if constexpr (points)
        PCU_LAUNCH((wn_point_leaves_kernel<T>), fblocks, kThreads, stream, v, n, a, m, (const MqRec*)sorted, t.leaves);
    else if constexpr (surfels)
        PCU_LAUNCH((sf_leaves_kernel<T>), fblocks, kThreads, stream, v, src, m, (const MqScratch*)t.sc, (const MqRec*)sorted,
                   t.leaves, t.ids, s.boxes);
    else if constexpr (kBallLeaf<L>)
        PCU_LAUNCH(rv_ball_leaves_kernel, fblocks, kThreads, stream, (const double*)v, m, (const MqScratch*)t.sc, (const MqRec*)sorted,
                   t.leaves, t.ids, s.boxes);
    else
        PCU_LAUNCH((mq_leaves_kernel<T>), fblocks, kThreads, stream, v, nv, f, fkind, m, (const MqScratch*)t.sc, (const MqRec*)sorted,
                   t.leaves, s.boxes);
    PCU_LAUNCH(mq_nodes_kernel, fblocks, kThreads, stream, (const MqRec*)sorted, m, (const MqScratch*)t.sc, t.nodes, s.node_parent,
               s.leaf_parent);
    if constexpr (!points) {
        PCU_CUDA(cudaMemsetAsync(s.arrivals, 0, (size_t)inner * sizeof(int), stream));
        PCU_LAUNCH(mq_refit_kernel, fblocks, kThreads, stream, m, (const MqScratch*)t.sc, t.nodes, (const int*)s.node_parent,
                   (const int*)s.leaf_parent, (const MqBox*)s.boxes, s.arrivals);
    }
    if constexpr (!surfels && !kBallLeaf<L>) if (moments) {   // surfel and ball trees carry no far field
        PCU_CUDA(cudaMemsetAsync(s.arrivals, 0, (size_t)inner * sizeof(int), stream));
        PCU_LAUNCH((wn_centres_kernel<L>), fblocks, kThreads, stream, m, (const MqScratch*)t.sc, (const MqNode*)t.nodes,
                   (const int*)s.node_parent, (const int*)s.leaf_parent, (const L*)t.leaves, t.wn, s.arrivals);
        PCU_LAUNCH((wn_radius_kernel<L>), fblocks, kThreads, stream, m, (const MqScratch*)t.sc, (const int*)s.node_parent,
                   (const int*)s.leaf_parent, (const L*)t.leaves, t.wn);
        PCU_CUDA(cudaMemsetAsync(s.arrivals, 0, (size_t)inner * sizeof(int), stream));
        PCU_LAUNCH((wn_moments_kernel<L>), fblocks, kThreads, stream, m, (const MqScratch*)t.sc, (const MqNode*)t.nodes,
                   (const int*)s.node_parent, (const int*)s.leaf_parent, (const L*)t.leaves, t.wn, s.arrivals);
    }
    if constexpr (!points && !surfels && !kBallLeaf<L>)
        PCU_CUDA(cudaMemcpyAsync(out_bad, &t.sc->bad, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, stream));
    tree = t;
    return PCU_B200_OK;
}

inline unsigned query_blocks(pcu_b200_workspace* ws, long long nq) {
    return (unsigned)std::min<long long>((nq + kThreads - 1) / kThreads, (long long)ws->sm_count * 64);
}

template <typename T>
int closest_points_device(pcu_b200_workspace* ws, const T* p, long long np, const T* v, long long nv, const void* f, long long m,
                          int fkind, T* out_d, void* out_fidx, T* out_bc, unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (np < 0 || (np > 0 && !p)) return fail(PCU_B200_INVALID_ARGUMENT, "p must be an (n, 3) array");
    if (!out_bad || (np > 0 && (!out_d || !out_fidx || !out_bc))) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshTree<Pt<T>> t;
    PCU_TRY(build_mesh_tree<T>(ws, v, nv, f, m, fkind, false, out_bad, stream, t));
    if (np == 0) return PCU_B200_OK;
    PCU_LAUNCH((mq_query_kernel<T>), query_blocks(ws, np), kThreads, stream, p, np, m, (const MqScratch*)t.sc, (const MqNode*)t.nodes,
               (const Pt<T>*)t.leaves, out_d, out_fidx, (fkind & 1), out_bc);
    return PCU_B200_OK;
}

// Winding numbers at q with far-field threshold beta (DESIGN.md §3; beta = inf: every face exactly).
template <typename T>
int winding_number_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, const T* q,
                          long long nq, double beta, T* out_w, unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (nq < 0 || (nq > 0 && !q)) return fail(PCU_B200_INVALID_ARGUMENT, "q must be an (n, 3) array");
    if (!(beta > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "accuracy_scale must be positive (got %g)", beta);
    if (!out_bad || (nq > 0 && !out_w)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshTree<Pt<T>> t;
    PCU_TRY(build_mesh_tree<T>(ws, v, nv, f, m, fkind, true, out_bad, stream, t));
    if (nq == 0) return PCU_B200_OK;
    PCU_LAUNCH((wn_query_kernel<T, Pt<T>>), query_blocks(ws, nq), kThreads, stream, q, nq, m, (const MqScratch*)t.sc, (const MqNode*)t.nodes,
               (const WnNode*)t.wn, (const Pt<T>*)t.leaves, (float)beta, out_w);
    return PCU_B200_OK;
}

// Winding numbers of the oriented cloud (p, n, a) at q with far-field threshold beta (DESIGN.md §3, point clouds): the
// tree over the points (build_mesh_tree with point leaves), built per call from the arena, then one thread per query.
// No points: w = 0.
template <typename T>
int point_winding_number_device(pcu_b200_workspace* ws, const T* p, const T* n, const T* a, long long m, const T* q, long long nq,
                                double beta, T* out_w, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (m < 0 || (m > 0 && (!p || !n || !a))) return fail(PCU_B200_INVALID_ARGUMENT, "p, n and a must be (n, 3), (n, 3) and (n,) arrays");
    if (m >= INT_MAX) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud winding numbers: at most 2^31 - 2 points, got %lld", m);
    if (nq < 0 || (nq > 0 && !q)) return fail(PCU_B200_INVALID_ARGUMENT, "q must be an (n, 3) array");
    if (nq >= INT_MAX) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud winding numbers: at most 2^31 - 2 queries, got %lld", nq);
    if (!(beta > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "accuracy_scale must be positive (got %g)", beta);
    if (nq > 0 && !out_w) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (nq == 0) return PCU_B200_OK;
    if (m == 0) {
        PCU_TRY(adopt_stream(ws, stream));
        PCU_CUDA(cudaMemsetAsync(out_w, 0, (size_t)nq * sizeof(T), stream));   // +0.0 in either precision
        return PCU_B200_OK;
    }
    MeshTree<WnPoint> t;
    PCU_TRY(build_mesh_tree<T>(ws, p, 0, nullptr, m, 0, true, nullptr, stream, t, nullptr, n, a));
    PCU_LAUNCH((wn_query_kernel<T, WnPoint>), query_blocks(ws, nq), kThreads, stream, q, nq, m, (const MqScratch*)t.sc,
               (const MqNode*)t.nodes, (const WnNode*)t.wn, (const WnPoint*)t.leaves, (float)beta, out_w);
    return PCU_B200_OK;
}

// Signed distances (libigl's fast-winding-number sign): the closest-point walk, then sd_sign_kernel on the same tree.
// The band is libigl's, computed in T from the fp32 bounds; max(a, b) is a < b ? b : a, so NaN (the defaults give
// inf - inf) disables the lower limit.
template <typename T>
int signed_distance_device(pcu_b200_workspace* ws, const T* p, long long np, const T* v, long long nv, const void* f, long long m,
                           int fkind, float lower_bound, float upper_bound, T* out_s, int* out_fidx, T* out_bc,
                           unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (np < 0 || (np > 0 && !p)) return fail(PCU_B200_INVALID_ARGUMENT, "p must be an (n, 3) array");
    if (!out_bad || (np > 0 && (!out_s || !out_fidx || !out_bc))) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    if (m >= INT_MAX) return fail(PCU_B200_INVALID_ARGUMENT, "signed distance returns int32 face indices: at most 2^31 - 2 faces");
    PCU_ON_DEVICE(ws);
    const auto larger = [](T a, T b) { return a < b ? b : a; };
    const T lo = (T)lower_bound, hi = (T)upper_bound;
    const T max_abs = larger(-lo, hi);
    const T up = max_abs * max_abs;
    const T low_root = larger(max_abs - (hi - lo), (T)0);
    const T low = low_root * low_root;
    MeshTree<Pt<T>> t;
    PCU_TRY(build_mesh_tree<T>(ws, v, nv, f, m, fkind, true, out_bad, stream, t));
    if (np == 0) return PCU_B200_OK;
    PCU_LAUNCH((mq_query_kernel<T>), query_blocks(ws, np), kThreads, stream, p, np, m, (const MqScratch*)t.sc, (const MqNode*)t.nodes,
               (const Pt<T>*)t.leaves, out_s, (void*)out_fidx, 0, out_bc);
    PCU_LAUNCH((sd_sign_kernel<T>), query_blocks(ws, np), kThreads, stream, p, np, v, nv, f, fkind, m, (const MqScratch*)t.sc,
               (const MqNode*)t.nodes, (const WnNode*)t.wn, (const Pt<T>*)t.leaves, 2.f, up, low, out_s, out_fidx, out_bc);
    return PCU_B200_OK;
}

// ---- rays against a mesh (raycast.cuh) --------------------------------------------------------------------------------
// One launch over the rays of a built tree.  o_stride: 0 (one origin for every ray) or 3.  near and far are fp32
// (DESIGN.md §3); out_fidx holds 8-byte indices when fidx_wide, else 4-byte ones.
template <typename TR, typename TM>
int cast_rays(pcu_b200_workspace* ws, const MqScratch* sc, const MqNode* nodes, const Pt<TM>* leaves, long long m, const TR* o,
              int o_stride, const TR* d, long long n, float near, float far, void* out_fidx, int fidx_wide, TR* out_bc, TR* out_t,
              cudaStream_t stream) {
    if (n == 0) return PCU_B200_OK;
    PCU_LAUNCH((rc_query_kernel<TR, TM>), query_blocks(ws, n), kThreads, stream, o, o_stride, d, n, near, far, m, sc, nodes, leaves,
               out_fidx, fidx_wide, out_bc, out_t);
    return PCU_B200_OK;
}

int check_rays(const void* o, int o_stride, const void* d, long long n) {
    if (o_stride != 0 && o_stride != 3) return fail(PCU_B200_INVALID_ARGUMENT, "o_stride must be 0 (one origin) or 3 (got %d)", o_stride);
    if (n < 0 || (n > 0 && (!o || !d))) return fail(PCU_B200_INVALID_ARGUMENT, "ray_o and ray_d must be (n, 3) arrays");
    return PCU_B200_OK;
}

// What every cast against a handle checks first: the handle is there, lives on the workspace's device and holds the
// kind of tree the caller casts against, and the rays are well formed.
int check_cast(pcu_b200_workspace* ws, const pcu_b200_mesh* h, bool want_surfels, const void* o, int o_stride, const void* d,
               long long n) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (h->device != ws->device)
        return fail(PCU_B200_INVALID_ARGUMENT, "the %s on device %d, the workspace on device %d", want_surfels ? "surfels live" : "mesh lives",
                    h->device, ws->device);
    if ((h->subdivs != 0) != want_surfels)
        return fail(PCU_B200_INVALID_ARGUMENT, "the handle holds %s", want_surfels ? "a mesh, not surfels" : "surfels, not a mesh");
    return check_rays(o, o_stride, d, n);
}

// A new handle for a tree of m leaves L (fans of `subdivs` triangles for surfels, else 0) over coordinates T, built once
// into a private block: sizes the block, allocates handle and block, runs build(block, tree) and frees both if that
// fails.  m = 0 (surfels only): a handle without a block, which every ray misses.  `what` names the block when
// cudaMalloc fails.
template <typename T, typename L, typename Build>
int prepare_tree(pcu_b200_workspace* ws, const char* what, long long m, int subdivs, pcu_b200_mesh** out, Build&& build) {
    MeshTree<L> t{};
    const size_t bytes = m > 0 ? carve_at(nullptr, [&](Carver& cv) { carve_mesh_tree(cv, m, false, t, subdivs); }) : 0;
    pcu_b200_mesh* h = new (std::nothrow) pcu_b200_mesh();
    if (!h) return fail(PCU_B200_OUT_OF_MEMORY, "out of host memory");
    h->device = ws->device; h->is_f64 = sizeof(T) == 8 ? 1 : 0; h->nf = m; h->subdivs = subdivs; h->bytes = bytes;
    if (m > 0) {
        cudaError_t e = cudaMalloc((void**)&h->block, bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            delete h;
            return fail(PCU_B200_OUT_OF_MEMORY, "cudaMalloc of %zu bytes for %s failed: %s", bytes, what, cudaGetErrorString(e));
        }
        const int st = build(h->block, t);
        if (st != PCU_B200_OK) { cudaFree(h->block); delete h; return st; }
        h->sc = t.sc; h->nodes = t.nodes; h->leaves = t.leaves; h->ids = t.ids;
    }
    *out = h;
    return PCU_B200_OK;
}

// The tree of the closest-point query, built for this call, then one thread per ray.
template <typename T>
int ray_mesh_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, const T* o, int o_stride,
                    const T* d, long long n, float near, float far, void* out_fidx, T* out_bc, T* out_t, unsigned long long* out_bad,
                    cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    PCU_TRY(check_rays(o, o_stride, d, n));
    if (!out_bad || (n > 0 && (!out_fidx || !out_bc || !out_t))) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    MeshTree<Pt<T>> t;
    PCU_TRY(build_mesh_tree<T>(ws, v, nv, f, m, fkind, false, out_bad, stream, t));
    return cast_rays<T, T>(ws, t.sc, t.nodes, t.leaves, m, o, o_stride, d, n, near, far, out_fidx, fkind & 1, out_bc, out_t, stream);
}

// Builds the tree once into a private block; *out_bad gets the count of faces with a corner out of range.
template <typename T>
int mesh_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, pcu_b200_mesh** out,
                        unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws || !out || !out_bad) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    PCU_ON_DEVICE(ws);
    return prepare_tree<T, Pt<T>>(ws, "a prepared mesh", m, 0, out, [&](unsigned char* block, MeshTree<Pt<T>>& t) {
        return build_mesh_tree<T>(ws, v, nv, f, m, fkind, false, out_bad, stream, t, block);
    });
}

// Rays of precision TR against a prepared mesh of either precision; face indices as int32.
template <typename TR>
int ray_mesh_prepared_device(pcu_b200_workspace* ws, const pcu_b200_mesh* mesh, const TR* o, int o_stride, const TR* d, long long n,
                             float near, float far, int* out_fidx, TR* out_bc, TR* out_t, cudaStream_t stream) {
    PCU_TRY(check_cast(ws, mesh, false, o, o_stride, d, n));
    if (n > 0 && (!out_fidx || !out_bc || !out_t)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (mesh->is_f64)
        return cast_rays<TR, double>(ws, mesh->sc, mesh->nodes, (const Pt<double>*)mesh->leaves, mesh->nf, o, o_stride, d, n, near, far,
                                     out_fidx, 0, out_bc, out_t, stream);
    return cast_rays<TR, float>(ws, mesh->sc, mesh->nodes, (const Pt<float>*)mesh->leaves, mesh->nf, o, o_stride, d, n, near, far,
                                out_fidx, 0, out_bc, out_t, stream);
}

// ---- rays against surfels (raycast.cuh) ------------------------------------------------------------------------------
// The largest subdivs: theta_j's fp32 quotient j / s is then exact in its numerator and denominator.
constexpr int kMaxSubdivs = 1 << 24;

int check_surfels(const void* p, const void* n, const void* r, long long m, int subdivs) {
    if (m < 0 || (m > 0 && (!p || !n || !r))) return fail(PCU_B200_INVALID_ARGUMENT, "p, n and r must be (n, 3), (n, 3) and (n,) arrays");
    if (m >= INT_MAX) return fail(PCU_B200_INVALID_ARGUMENT, "surfels: at most 2^31 - 2 points, got %lld", m);
    if (subdivs < 4 || subdivs > kMaxSubdivs)
        return fail(PCU_B200_INVALID_ARGUMENT, "subdivs must be in [4, 2^24] (got %d)", subdivs);
    return PCU_B200_OK;
}

// The surfel tree of (p, n, r, subdivs), built for this call, then one thread per ray (m = 0: no tree, every ray misses).
template <typename T>
int ray_surfel_device(pcu_b200_workspace* ws, const T* p, const T* nrm, const T* r, long long m, int subdivs, const T* o, int o_stride,
                      const T* d, long long n, float near, float far, int* out_pid, T* out_t, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(check_surfels(p, nrm, r, m, subdivs));
    PCU_TRY(check_rays(o, o_stride, d, n));
    if (n > 0 && (!out_pid || !out_t)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (n == 0) return PCU_B200_OK;
    MeshTree<SfWord> t{};
    if (m > 0) PCU_TRY(build_mesh_tree<T>(ws, p, 0, nullptr, m, 0, false, nullptr, stream, t, nullptr, nrm, r, subdivs));
    PCU_LAUNCH((rs_query_kernel<T>), query_blocks(ws, n), kThreads, stream, o, o_stride, d, n, near, far, m, subdivs,
               (const MqScratch*)t.sc, (const MqNode*)t.nodes, (const SfWord*)t.leaves, (const int*)t.ids, out_pid, out_t);
    return PCU_B200_OK;
}

// Builds the surfel tree once into a private block (no block for m = 0).
template <typename T>
int surfel_prepare_device(pcu_b200_workspace* ws, const T* p, const T* nrm, const T* r, long long m, int subdivs, pcu_b200_mesh** out,
                          cudaStream_t stream) {
    if (!ws || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(check_surfels(p, nrm, r, m, subdivs));
    PCU_ON_DEVICE(ws);
    return prepare_tree<T, SfWord>(ws, "prepared surfels", m, subdivs, out, [&](unsigned char* block, MeshTree<SfWord>& t) {
        return build_mesh_tree<T>(ws, p, 0, nullptr, m, 0, false, nullptr, stream, t, block, nrm, r, subdivs);
    });
}

// Rays of precision TR against prepared surfels of either precision (the leaves are fp32 either way).
template <typename TR>
int ray_surfel_prepared_device(pcu_b200_workspace* ws, const pcu_b200_mesh* h, const TR* o, int o_stride, const TR* d, long long n,
                               float near, float far, int* out_pid, TR* out_t, cudaStream_t stream) {
    PCU_TRY(check_cast(ws, h, true, o, o_stride, d, n));
    if (n > 0 && (!out_pid || !out_t)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (n == 0) return PCU_B200_OK;
    PCU_LAUNCH((rs_query_kernel<TR>), query_blocks(ws, n), kThreads, stream, o, o_stride, d, n, near, far, h->nf, h->subdivs,
               (const MqScratch*)h->sc, (const MqNode*)h->nodes, (const SfWord*)h->leaves, h->ids, out_pid, out_t);
    return PCU_B200_OK;
}

// pointcloud_surfel_geometry: (s + 1) m vertices in T and s m int32 faces.
template <typename T>
int surfel_geometry_device(pcu_b200_workspace* ws, const T* p, const T* nrm, const T* r, long long m, int subdivs, T* out_v,
                           int* out_f, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(check_surfels(p, nrm, r, m, subdivs));
    if (m * (long long)(subdivs + 1) >= INT_MAX)
        return fail(PCU_B200_INVALID_ARGUMENT, "surfel geometry: int32 faces index at most 2^31 - 2 vertices, got %lld points of %d",
                    m, subdivs + 1);
    if (m > 0 && (!out_v || !out_f)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    if (m == 0) return PCU_B200_OK;
    unsigned char* dev = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { dev = cv.take<unsigned char>(surfel_src_bytes(subdivs)); }));
    SfSrc src{};
    PCU_TRY(upload_surfel_src(dev, nrm, r, subdivs, nullptr, stream, src));
    PCU_LAUNCH((sf_geometry_kernel<T>), (unsigned)((m + kThreads - 1) / kThreads), kThreads, stream, p, src, m, out_v, out_f);
    return PCU_B200_OK;
}

// ---- marching cubes and the boundary of a sparse voxel grid (sparse_voxels.cuh) ------------------------------------
// Copies a count record to the host and waits for it: one synchronisation of `stream`.
template <class R>
int read_record(const R* dev, R* host, cudaStream_t stream) {
    PCU_CUDA(cudaMemcpyAsync(host, dev, sizeof(R), cudaMemcpyDeviceToHost, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));
    return PCU_B200_OK;
}

// The failure of a call that found `bad` faces with a corner outside [0, #v).
int bad_corners(unsigned long long bad) {
    return fail(PCU_B200_INVALID_ARGUMENT, "Invalid face indices: %llu faces have a corner outside [0, #v)", bad);
}

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
    PCU_LAUNCH(keep_rows_kernel<int>, blocks_for(entries), kThreads, stream, (const unsigned char*)flag, entries, (const unsigned*)counts, rows);
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
    PCU_LAUNCH(keep_rows_kernel<int>, blocks_for(c1), kThreads, stream, (const unsigned char*)flag2, c1, (const unsigned*)counts2, sub[0]);
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
    PCU_TRY((build_mesh_tree<double, RvBall>)(ws, r.balls, m, nullptr, m, 0, false, nullptr, stream, tree));
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
        [&](double* x) -> int {
            MeshCdfScratch ms;
            PCU_TRY(carve_scratch(ws, kMesh, stream, [&](Carver& cv) { ms.carve(cv, m); }));
            PCU_TRY(enqueue_mesh_cdf<double>(ws, v, nv, f, fkind, m, ms.cdf, ms.tiles, ms.sc, ms.area, stream));
            MeshArea area;
            PCU_TRY(read_record(ms.area, &area, stream));
            if (area.bad) return bad_corners(area.bad);
            if (area.total == 0) return fail(PCU_B200_INVALID_ARGUMENT, "Mesh has zero area");
            const unsigned blocks = (unsigned)std::min<long long>((n + kThreads - 1) / kThreads, (long long)ws->sm_count * 16);
            PCU_LAUNCH((mesh_sample_kernel<double>), blocks, kThreads, stream, (const unsigned long long*)ms.cdf, m,
                       (const MeshArea*)ms.area, (unsigned long long)seed, n, (const int*)nullptr, (const long long*)nullptr, v, nv, f,
                       fkind, (void*)nullptr, 0, (double*)nullptr, x);
            return PCU_B200_OK;
        },
        [&](const double* x, VorSync* sync, double** mom, VorSync* seen) -> int {
            return rv_eval(ws, r, x, sync, mom, passes, seen, stream);
        });
}

// Whether face indices of this kind are 64 bits wide.
inline bool wide_index(int kind) { return kind & 1; }

// A handle's block, allocated in the order of `stream`; `what` names the handle's feature when that fails.
int alloc_block(unsigned char*& block, size_t bytes, cudaStream_t stream, const char* what) {
    const cudaError_t e = cudaMallocAsync((void**)&block, bytes, stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        block = nullptr;
        return fail(PCU_B200_OUT_OF_MEMORY, "cudaMallocAsync of %zu bytes for %s failed: %s", bytes, what, cudaGetErrorString(e));
    }
    return PCU_B200_OK;
}

// A new handle H on the workspace's device and `stream`: runs build(h), deletes the handle if that fails and
// publishes it in *out if it succeeds.
template <class H, class Build>
int prepare_handle(pcu_b200_workspace* ws, cudaStream_t stream, H** out, Build&& build) {
    H* h = new (std::nothrow) H();
    if (!h) return fail(PCU_B200_OUT_OF_MEMORY, "out of host memory");
    h->device = ws->device;
    h->stream = stream;
    const int st = build(h);
    if (st != PCU_B200_OK) { delete h; return st; }
    *out = h;
    return PCU_B200_OK;
}

// An emit runs on the device its handle was prepared on; `what` names the handle.
int check_handle_device(const pcu_b200_workspace* ws, const StreamHandle* h, const char* what) {
    if (h->device != ws->device)
        return fail(PCU_B200_INVALID_ARGUMENT, "the %s handle lives on device %d, the workspace on %d", what, h->device, ws->device);
    return PCU_B200_OK;
}

// Classify + scan, read the counts (first synchronisation), then the slot records, their sort, the runs and the owners'
// vertex ids, and read the vertex count (second synchronisation).
template <typename T, typename S, int W>
int mc_build(pcu_b200_workspace* ws, pcu_b200_marching_cubes* h, cudaStream_t stream) {
    const long long m = h->m;
    const unsigned tiles = blocks_for(m);
    PCU_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(McCounts), stream));
    PCU_LAUNCH((mc_classify_kernel<T, S, W>), tiles, kThreads, stream, (const S*)h->scalars, h->n, h->idx, m, (T)h->iso,
               h->cases, h->tile_sum, h->counts);
    PCU_LAUNCH(mc_tiles_kernel, 1, 1024, stream, (const unsigned*)h->tile_sum, (long long)tiles, h->tile_slot0, h->tile_face0, h->counts);
    McCounts c;
    PCU_TRY(read_record(h->counts, &c, stream));
    if (c.bad) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid cube_indices: %llu cubes have a corner outside [0, %lld)", c.bad, h->n);
    if (c.slots >= (1ull << 32))
        return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: at most 2^32 - 1 crossing edges are supported, got %llu", c.slots);
    h->slots = (long long)c.slots;
    h->faces = (long long)c.faces;
    const long long ns = h->slots;
    if (ns == 0) return PCU_B200_OK;
    PCU_TRY(alloc_block(h->slot_block, carve_at(nullptr, [&](Carver& cv) {
        cv.take<unsigned>((size_t)ns); cv.take<unsigned>((size_t)ns); cv.take<unsigned char>((size_t)ns); }), stream, "marching cubes"));
    carve_at(h->slot_block, [&](Carver& cv) {
        h->slot_run = cv.take<unsigned>((size_t)ns);
        h->run_vid = cv.take<unsigned>((size_t)ns);
        h->owner = cv.take<unsigned char>((size_t)ns);
    });
    struct { SortScratch<McRec> sort; unsigned char* head; unsigned* counts; unsigned* ocounts; long long* owners; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, ns);
        sc.head = cv.take<unsigned char>((size_t)ns);
        sc.counts = cv.take<unsigned>(keep_count_words(ns));
        sc.ocounts = cv.take<unsigned>(keep_count_words(ns));
        sc.owners = cv.take<long long>(1);
    }));
    int b = 1;                                       // bits of the largest corner index, n - 1
    while (b < 31 && ((h->n - 1) >> b) != 0) ++b;
    PCU_LAUNCH((mc_slots_kernel<W>), tiles, kThreads, stream, h->idx, (const unsigned char*)h->cases, m,
               (const unsigned long long*)h->tile_slot0, (const unsigned long long*)h->tile_face0, b, sc.sort.a);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, ns, 1, stream, &sorted, 2 * b));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(ns), kThreads, stream, (const McRec*)sorted, ns, sc.head);
    PCU_TRY(enqueue_keep_offsets(sc.head, ns, sc.counts, &h->counts->verts, stream));
    PCU_LAUNCH(mc_runs_kernel, blocks_for(ns), kThreads, stream, (const McRec*)sorted, ns, (const unsigned char*)sc.head,
               (const unsigned*)sc.counts, h->slot_run, h->owner);
    PCU_TRY(enqueue_keep_offsets(h->owner, ns, sc.ocounts, sc.owners, stream));
    PCU_LAUNCH(mc_owner_kernel, blocks_for(ns), kThreads, stream, (const unsigned char*)h->owner, ns, (const unsigned*)sc.ocounts,
               (const unsigned*)h->slot_run, h->run_vid);
    PCU_TRY(read_record(h->counts, &c, stream));
    h->verts = c.verts;
    return PCU_B200_OK;
}

template <typename T, typename S>
int mc_build_width(pcu_b200_workspace* ws, pcu_b200_marching_cubes* h, cudaStream_t stream) {
    return h->width == 8 ? mc_build<T, S, 8>(ws, h, stream) : mc_build<T, S, 4>(ws, h, stream);
}

template <typename T>
int marching_cubes_prepare_device(pcu_b200_workspace* ws, const void* scalars, int s_f64, const T* coords, long long n, const void* idx,
                                  long long m, int kind, double isovalue, pcu_b200_marching_cubes** out, long long* out_counts,
                                  cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!scalars || !coords || !idx) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (n <= 0 || n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: n must be in [1, 2^31 - 2], got %lld", n);
    if (m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid cube_indices has zero rows!");
    if (kind < kIdxI32 || kind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind %d", kind);
    if ((uintptr_t)idx % 16 != 0) return fail(PCU_B200_INVALID_ARGUMENT, "cube_idx must be 16-byte aligned");
    if ((m + kThreads - 1) / kThreads > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "too many cubes (%lld)", m);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_marching_cubes* h) -> int {
        h->t_f64 = sizeof(T) == 8; h->s_f64 = s_f64 != 0; h->width = wide_index(kind) ? 8 : 4;
        h->scalars = scalars; h->coords = coords; h->idx = idx; h->n = n; h->m = m;
        h->iso = s_f64 ? (double)(T)isovalue : (double)(T)(float)isovalue;
        const long long tiles = (m + kThreads - 1) / kThreads;
        const auto carve = [&](Carver& cv) {
            h->cases = cv.take<unsigned char>((size_t)m);
            h->tile_sum = cv.take<unsigned>((size_t)tiles);
            h->tile_slot0 = cv.take<unsigned long long>((size_t)tiles);
            h->tile_face0 = cv.take<unsigned long long>((size_t)tiles);
            h->counts = cv.take<McCounts>(1);
        };
        PCU_TRY(alloc_block(h->cube_block, carve_at(nullptr, carve), stream, "marching cubes"));
        carve_at(h->cube_block, carve);
        PCU_TRY((h->s_f64 ? mc_build_width<T, double>(ws, h, stream) : mc_build_width<T, float>(ws, h, stream)));
        const long long most = kind == kIdxI32 ? (1ll << 31) : kind == kIdxU32 ? (1ll << 32) : LLONG_MAX;
        if (h->verts > most)
            return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: %lld vertices cannot be indexed by cube_indices' dtype", h->verts);
        return PCU_B200_OK;
    }));
    out_counts[0] = (*out)->verts;
    out_counts[1] = (*out)->faces;
    return PCU_B200_OK;
}

template <typename T, typename S, int W>
int mc_emit_launch(const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    PCU_LAUNCH((mc_emit_kernel<T, S, W>), blocks_for(h->m), kThreads, stream, (const S*)h->scalars, (const T*)h->coords, h->idx,
               (const unsigned char*)h->cases, h->m, (const unsigned long long*)h->tile_slot0,
               (const unsigned long long*)h->tile_face0, (T)h->iso, (const unsigned*)h->slot_run, (const unsigned*)h->run_vid,
               (const unsigned char*)h->owner, (T*)out_v, out_f);
    return PCU_B200_OK;
}

template <typename T, typename S>
int mc_emit_width(const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    return h->width == 8 ? mc_emit_launch<T, S, 8>(h, out_v, out_f, stream) : mc_emit_launch<T, S, 4>(h, out_v, out_f, stream);
}

int marching_cubes_emit_device(pcu_b200_workspace* ws, const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "marching-cubes"));
    if (h->slots == 0) return PCU_B200_OK;
    if (!out_v || (h->faces > 0 && !out_f)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    if (h->t_f64) return h->s_f64 ? mc_emit_width<double, double>(h, out_v, out_f, stream) : mc_emit_width<double, float>(h, out_v, out_f, stream);
    return h->s_f64 ? mc_emit_width<float, double>(h, out_v, out_f, stream) : mc_emit_width<float, float>(h, out_v, out_f, stream);
}

// Codes, their sort, the six-neighbour lookups, the ordered compaction.  out_counts (device): {boundary rows, bad rows}.
template <typename I>
int svb_device(pcu_b200_workspace* ws, const I* g, long long n, long long* out_idx, long long* out_counts, cudaStream_t stream) {
    struct { SortScratch<McRec> sort; unsigned char* keep; unsigned* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.keep = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 2 * sizeof(long long), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, (unsigned long long*)(out_counts + 1));
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH((svb_flag_kernel<I>), blocks_for(n), kThreads, stream, g, n, (const McRec*)sorted, sc.keep);
    PCU_TRY(enqueue_keep_offsets(sc.keep, n, sc.counts, out_counts, stream));
    PCU_LAUNCH(keep_rows_kernel<long long>, blocks_for(n), kThreads, stream, (const unsigned char*)sc.keep, n, (const unsigned*)sc.counts, out_idx);
    return PCU_B200_OK;
}

int sparse_voxel_grid_boundary_device(pcu_b200_workspace* ws, const void* g, long long n, int kind, long long* out_idx,
                                      long long* out_counts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!g || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid grid_coordinates has zero rows!");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "sparse_voxel_grid_boundary: at most 2^31 - 2 voxels, got %lld", n);
    if (kind != kIdxI32 && kind != kIdxI64)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small.");
    if (!out_idx || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    return kind == kIdxI64 ? svb_device<long long>(ws, (const long long*)g, n, out_idx, out_counts, stream)
                           : svb_device<int>(ws, (const int*)g, n, out_idx, out_counts, stream);
}

// ---- sparse voxel grids and voxel cube meshes (sparse_voxels.cuh) -------------------------------------------------
enum SvgMode { kSvgPoints = 0, kSvgDilate = 1, kSvgHex = 2 };
// Dilation ranks 26 flags per voxel, the hex mesh 8 corners per voxel, in 32 bits (compact.cuh: fewer than 2^31 rows);
// voxel_grid_geometry's int32 faces index 8 n vertices.
constexpr long long kSvgMaxDilate = (0x7ffffffeLL) / 26;   // 82 595 524
constexpr long long kSvgMaxHex = (0x7ffffffeLL) / 8;       // 2^28 - 1
constexpr long long kVgMaxVoxels = 1LL << 28;

int svg_overflow() {
    return fail(PCU_B200_INVALID_ARGUMENT, "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small.");
}

// The handle's block for `recs` records: sort scratch, run heads (unless the records are distinct), block offsets, the
// count record.  The caller writes the records into sort.a.
int svg_alloc(pcu_b200_sparse_grid* h, long long recs, bool heads, SortScratch<McRec>& sort, cudaStream_t stream) {
    h->recs = recs;
    const auto carve = [&](Carver& cv) {
        sort.carve(cv, recs);
        h->head = heads ? cv.take<unsigned char>((size_t)recs) : nullptr;
        h->offsets = cv.take<unsigned>(keep_count_words(recs));
        h->counts = cv.take<SvgCounts>(1);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "sparse voxel grid"));
    carve_at(h->block, carve);
    PCU_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(SvgCounts), stream));
    return PCU_B200_OK;
}

// Sorts the records, numbers their runs (the count of distinct codes into h->counts->rows) and, when read, reads the
// count record: one synchronisation of `stream`.
int svg_sort_runs(pcu_b200_sparse_grid* h, const SortScratch<McRec>& sort, bool read, cudaStream_t stream) {
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sort, h->recs, 1, stream, &sorted));
    h->sorted = sorted;
    if (h->head) {
        PCU_LAUNCH(mc_heads_kernel, blocks_for(h->recs), kThreads, stream, (const McRec*)sorted, h->recs, h->head);
        PCU_TRY(enqueue_keep_offsets(h->head, h->recs, h->offsets, &h->counts->rows, stream));
    }
    if (!read) return PCU_B200_OK;
    SvgCounts c;
    PCU_TRY(read_record(h->counts, &c, stream));
    if (c.bad) return svg_overflow();
    h->rows = c.rows;
    return PCU_B200_OK;
}

// A grid argument of the sparse-grid entry points: int32 or int64 (unsigned grids fail the reference's range check).
int svg_check_grid(const void* g, long long n, int kind, long long most, const char* what) {
    if (!g || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid grid_coordinates has zero rows!");
    if (n > most) return fail(PCU_B200_INVALID_ARGUMENT, "%s: at most %lld voxels are supported, got %lld", what, most, n);
    if (kind != kIdxI32 && kind != kIdxI64) return svg_overflow();
    return PCU_B200_OK;
}

template <typename T>
int svg_points_prepare(pcu_b200_workspace* ws, const T* p, long long n, const double size[3], const double origin[3],
                       pcu_b200_sparse_grid** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!p || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid points has zero rows!");
    if (n >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "sparse_voxel_grid_from_pointcloud: at most 2^31 - 2 points are supported, got %lld", n);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgPoints; h->n = n;
        for (int a = 0; a < 3; ++a) { h->place.g[a] = size[a]; h->place.o[a] = origin[a]; }
        SortScratch<McRec> sort;
        PCU_TRY(svg_alloc(h, n, true, sort, stream));
        PCU_LAUNCH((svg_point_codes_kernel<T>), blocks_for(n), kThreads, stream, p, n, h->place, sort.a, &h->counts->bad);
        return svg_sort_runs(h, sort, true, stream);
    }));
    out_counts[0] = (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

// One dilation round: the input's codes and their sort, the owned missing neighbours' flags and their count (read:
// one synchronisation), then the owned codes, compacted and sorted.
template <typename I>
int svg_dilate_build(pcu_b200_workspace* ws, pcu_b200_sparse_grid* h, const I* g, long long n, cudaStream_t stream) {
    const long long slots = 26 * n;
    struct { SortScratch<McRec> sort; unsigned char* flag; unsigned* counts; SvgCounts* rec; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.flag = cv.take<unsigned char>((size_t)slots);
        sc.counts = cv.take<unsigned>(keep_count_words(slots));
        sc.rec = cv.take<SvgCounts>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(SvgCounts), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, &sc.rec->bad);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH(svg_dilate_flag_kernel, blocks_for(n), kThreads, stream, (const McRec*)sorted, n, sc.flag);
    PCU_TRY(enqueue_keep_offsets(sc.flag, slots, sc.counts, &sc.rec->rows, stream));
    SvgCounts c;
    PCU_TRY(read_record(sc.rec, &c, stream));
    if (c.bad) return svg_overflow();
    h->rows = c.rows;
    if (c.rows == 0) return PCU_B200_OK;
    SortScratch<McRec> sort;
    PCU_TRY(svg_alloc(h, c.rows, false, sort, stream));
    PCU_LAUNCH(svg_dilate_write_kernel, blocks_for(slots), kThreads, stream, (const McRec*)sorted, n, (const unsigned char*)sc.flag,
               (const unsigned*)sc.counts, sort.a);
    return svg_sort_runs(h, sort, false, stream);
}

int svg_dilate_prepare(pcu_b200_workspace* ws, const void* g, long long n, int kind, pcu_b200_sparse_grid** out, long long* out_counts,
                       cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(svg_check_grid(g, n, kind, kSvgMaxDilate, "dilate_sparse_voxel_grid"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgDilate; h->n = n; h->grid = g; h->out_kind = kind;
        return kind == kIdxI64 ? svg_dilate_build<long long>(ws, h, (const long long*)g, n, stream)
                               : svg_dilate_build<int>(ws, h, (const int*)g, n, stream);
    }));
    out_counts[0] = n + (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

int svg_hex_prepare(pcu_b200_workspace* ws, const void* g, long long n, int kind, const double size[3], const double origin[3], int v_f64,
                    pcu_b200_sparse_grid** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(svg_check_grid(g, n, kind, kSvgMaxHex, "sparse_voxel_grid_to_hex_mesh"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgHex; h->n = n; h->out_kind = v_f64 != 0;
        for (int a = 0; a < 3; ++a) { h->place.g[a] = size[a]; h->place.o[a] = origin[a]; }
        SortScratch<McRec> sort;
        PCU_TRY(svg_alloc(h, 8 * n, true, sort, stream));
        if (kind == kIdxI64) PCU_LAUNCH((svg_corners_kernel<long long>), blocks_for(n), kThreads, stream, (const long long*)g, n, sort.a, &h->counts->bad);
        else PCU_LAUNCH((svg_corners_kernel<int>), blocks_for(n), kThreads, stream, (const int*)g, n, sort.a, &h->counts->bad);
        return svg_sort_runs(h, sort, true, stream);
    }));
    out_counts[0] = (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

template <typename O>
int svg_decode_launch(const pcu_b200_sparse_grid* h, void* out, cudaStream_t stream) {
    PCU_LAUNCH(svg_decode_kernel<O>, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, h->place, (O*)out);
    return PCU_B200_OK;
}

// From points: out_rows (rows, 3) int32, out_index (n) int64 point_to_vox.  Dilation: out_rows (n + rows, 3) of the
// grid's kind, the input rows then the new ones.  Hex mesh: out_rows (rows, 3) vertices, out_index (n, 8) int64 cubes.
int svg_emit(pcu_b200_workspace* ws, const pcu_b200_sparse_grid* h, void* out_rows, int64_t* out_index, cudaStream_t stream) {
    if (!ws || !h || !out_rows || (h->mode != kSvgDilate && !out_index)) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "sparse voxel grid"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    if (h->mode == kSvgDilate) {
        const size_t width = h->out_kind == kIdxI64 ? 8 : 4;
        PCU_CUDA(cudaMemcpyAsync(out_rows, h->grid, (size_t)h->n * 3 * width, cudaMemcpyDeviceToDevice, stream));
        if (h->rows == 0) return PCU_B200_OK;
        unsigned char* tail = (unsigned char*)out_rows + (size_t)h->n * 3 * width;
        return h->out_kind == kIdxI64 ? svg_decode_launch<long long>(h, tail, stream) : svg_decode_launch<int>(h, tail, stream);
    }
    if (h->mode == kSvgPoints) PCU_TRY(svg_decode_launch<int>(h, out_rows, stream));
    else PCU_TRY(h->out_kind ? svg_decode_launch<double>(h, out_rows, stream) : svg_decode_launch<float>(h, out_rows, stream));
    PCU_LAUNCH(svg_rank_kernel, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, (long long*)out_index);
    return PCU_B200_OK;
}

// Erosion: codes, their sort, the 26-neighbour test, the ordered copy of the kept rows.  out_counts (device):
// {kept rows, rows out of range}.
template <typename I>
int svg_erode_device(pcu_b200_workspace* ws, const I* g, long long n, I* out, long long* out_counts, cudaStream_t stream) {
    struct { SortScratch<McRec> sort; unsigned char* keep; unsigned* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.keep = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 2 * sizeof(long long), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, (unsigned long long*)(out_counts + 1));
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH((svg_erode_flag_kernel<I>), blocks_for(n), kThreads, stream, g, n, (const McRec*)sorted, sc.keep);
    PCU_TRY(enqueue_keep_offsets(sc.keep, n, sc.counts, out_counts, stream));
    PCU_LAUNCH((svg_keep_voxels_kernel<I>), blocks_for(n), kThreads, stream, g, (const unsigned char*)sc.keep, n, (const unsigned*)sc.counts, out);
    return PCU_B200_OK;
}

int svg_erode(pcu_b200_workspace* ws, const void* g, long long n, int kind, void* out, long long* out_counts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(svg_check_grid(g, n, kind, 0x7ffffffeLL, "erode_sparse_voxel_grid"));
    if (!out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    return kind == kIdxI64 ? svg_erode_device<long long>(ws, (const long long*)g, n, (long long*)out, out_counts, stream)
                           : svg_erode_device<int>(ws, (const int*)g, n, (int*)out, out_counts, stream);
}

int voxel_grid_geometry_device(pcu_b200_workspace* ws, const void* ijk, long long n, int kind, const double size[3], const double origin[3],
                               double gap, float* out_v, int32_t* out_f, cudaStream_t stream) {
    if (!ws || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (!ijk || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input point cloud with zero points");
    if (n > kVgMaxVoxels) return fail(PCU_B200_INVALID_ARGUMENT, "voxel_grid_geometry: at most 2^28 voxels are supported, got %lld", n);
    if (kind < kIdxI32 || kind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind %d", kind);
    // as in the reference, a NaN size passes here
    if (size[0] <= 0.0 || size[1] <= 0.0 || size[2] <= 0.0) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size must be positive");
    if (!out_v || !out_f) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    VgGeom g;
    for (int k = 0; k < 3; ++k) { g.s[k] = size[k]; g.o[k] = origin[k]; }
    g.keep = 1.0 - gap;
    g.shift = 0.5 * gap;
    const unsigned blocks = blocks_for(12 * n);
    switch (kind) {
        case kIdxI32: PCU_LAUNCH(vg_geometry_kernel<int>, blocks, kThreads, stream, (const int*)ijk, n, g, out_v, out_f); break;
        case kIdxI64: PCU_LAUNCH(vg_geometry_kernel<long long>, blocks, kThreads, stream, (const long long*)ijk, n, g, out_v, out_f); break;
        case kIdxU32: PCU_LAUNCH(vg_geometry_kernel<unsigned>, blocks, kThreads, stream, (const unsigned*)ijk, n, g, out_v, out_f); break;
        default: PCU_LAUNCH(vg_geometry_kernel<unsigned long long>, blocks, kThreads, stream, (const unsigned long long*)ijk, n, g, out_v, out_f);
    }
    return PCU_B200_OK;
}

// ---- triangle-mesh voxelization and 3-D flood fill (voxelize.cuh) ------------------------------------------------
// Persistent CTAs of vx_test_kernel: enough to fill every SM (the kernel holds 16-32 KB of shared memory per CTA).
inline unsigned vx_test_blocks(const pcu_b200_workspace* ws) { return (unsigned)ws->sm_count * 6u; }

// Bounds, scan and the counting pass; read the counts (first synchronisation); the code records, sized by the accepted
// count, their sort and run heads; read the number of distinct codes (second synchronisation).
template <typename T>
int vx_build(pcu_b200_workspace* ws, pcu_b200_voxelize* h, const T* v, long long nv, const void* f, long long m, int fkind,
             const VxGeom& g, cudaStream_t stream) {
    const long long tiles = (m + kThreads - 1) / kThreads;
    struct { VxFace* faces; unsigned long long* local; unsigned long long* tile; VxCounts* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.faces = cv.take<VxFace>((size_t)m);
        sc.local = cv.take<unsigned long long>((size_t)m);
        sc.tile = cv.take<unsigned long long>((size_t)tiles);
        sc.counts = cv.take<VxCounts>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.counts, 0, sizeof(VxCounts), stream));
    PCU_LAUNCH((vx_bounds_kernel<T>), (unsigned)tiles, kThreads, stream, v, nv, f, fkind, m, g, sc.faces, sc.local, sc.tile, sc.counts);
    PCU_LAUNCH(vx_tiles_kernel, 1, 1024, stream, sc.tile, tiles, sc.counts);
    PCU_LAUNCH((vx_test_kernel<T, kVxCount>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
               (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr);
    VxCounts c;
    PCU_TRY(read_record(sc.counts, &c, stream));
    if (c.bad_corner) return bad_corners(c.bad_corner);
    if (c.bad_bounds)
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: %llu faces have a non-finite vertex or voxel index bounds outside "
                    "[-2^31, 2^31 - 2]", c.bad_bounds);
    if (!(c.cand_d < kVxMaxCandidates))
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: %.6g candidate voxels overflow a 64-bit count", c.cand_d);
    if (c.accepted >= 0x7fffffffull)
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: at most 2^31 - 2 (face, voxel) overlaps are supported, got %llu",
                    c.accepted);
    const long long na = (long long)c.accepted;
    h->recs = na;
    if (na == 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    struct { SortScratch<McRec> sort; unsigned char* head; unsigned* counts; } hb;
    const auto carve = [&](Carver& cv) {
        hb.sort.carve(cv, na);
        hb.head = cv.take<unsigned char>((size_t)na);
        hb.counts = cv.take<unsigned>(keep_count_words(na));
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "voxelization"));
    carve_at(h->block, carve);
    PCU_LAUNCH((vx_test_kernel<T, kVxCodes>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
               (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, hb.sort.a);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(hb.sort, na, 1, stream, &sorted));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(na), kThreads, stream, (const McRec*)sorted, na, hb.head);
    PCU_TRY(enqueue_keep_offsets(hb.head, na, hb.counts, &sc.counts->unique, stream));
    PCU_TRY(read_record(sc.counts, &c, stream));
    h->n = c.unique;
    h->sorted = sorted;
    h->head = hb.head;
    h->offsets = hb.counts;
    return PCU_B200_OK;
}

template <typename T>
int voxelize_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, const double size[3],
                            const double origin[3], pcu_b200_voxelize** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (m >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: at most 2^31 - 2 faces are supported, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    // as in the reference, a NaN size passes here (it makes every face's bounds non-finite)
    if (size[0] <= 0.0 || size[1] <= 0.0 || size[2] <= 0.0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid voxel size");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    VxGeom g;
    for (int k = 0; k < 3; ++k) { g.o[k] = origin[k]; g.s[k] = size[k]; g.h[k] = size[k] / 2; }
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_voxelize* h) { return vx_build<T>(ws, h, v, nv, f, m, fkind, g, stream); }));
    out_counts[0] = (*out)->n;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

int voxelize_emit_device(pcu_b200_workspace* ws, const pcu_b200_voxelize* h, int32_t* out_ijk, cudaStream_t stream) {
    if (!ws || !h || !out_ijk) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "voxelization"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_LAUNCH(vx_decode_kernel, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, (int*)out_ijk);
    return PCU_B200_OK;
}

// (T)fill_value as the reference's x86 build converts a double: cvttsd2si for the integers (truncation toward zero; NaN
// and values whose truncation is out of range give the "integer indefinite" INT_MIN), round to nearest for float.
template <typename T>
T ff_cast(double x) {
    if constexpr (std::is_same<T, int>::value) return (x > -2147483649.0 && x < 2147483648.0) ? (int)x : INT32_MIN;
    else if constexpr (std::is_same<T, long long>::value) return (x >= -0x1p63 && x < 0x1p63) ? (long long)x : LLONG_MIN;
    else return (T)x;
}

// Tiles of at most kFfTileMax voxels, sides powers of two: up to 32 along z, then up to 256 / tz along y, the rest along
// x, each no larger than the grid needs.
inline int ff_log2_cover(long long n, int cap_log2) {
    int l = 0;
    while (l < cap_log2 && (1ll << l) < n) ++l;
    return l;
}

template <typename T>
int ff_device(pcu_b200_workspace* ws, const T* grid, long long w, long long h, long long d, long long seed, double fill, T* out,
              cudaStream_t stream) {
    FfShape s;
    s.w = w; s.h = h; s.d = d; s.n = w * h * d; s.seed = seed;
    s.lz = ff_log2_cover(d, 5);
    s.ly = ff_log2_cover(h, 8 - s.lz);
    s.lx = ff_log2_cover(w, 10 - s.lz - s.ly);
    s.tz_n = (unsigned)((d + (1ll << s.lz) - 1) >> s.lz);
    s.ty_n = (unsigned)((h + (1ll << s.ly) - 1) >> s.ly);
    const long long tx_n = (w + (1ll << s.lx) - 1) >> s.lx;
    const long long tiles = tx_n * s.ty_n * s.tz_n;
    int* P = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { P = cv.take<int>((size_t)s.n); }));
    PCU_LAUNCH((ff_tile_kernel<T>), (unsigned)tiles, kThreads, stream, grid, s, P);
    PCU_LAUNCH((ff_cross_kernel<T>), (unsigned)tiles, kThreads, stream, grid, s, P);
    PCU_LAUNCH((ff_out_kernel<T>), blocks_for(s.n), kThreads, stream, grid, s.n, seed, ff_cast<T>(fill), P, out);
    return PCU_B200_OK;
}

int flood_fill_3d_device(pcu_b200_workspace* ws, const void* grid, int kind, long long w, long long h, long long d, long long sx,
                         long long sy, long long sz, double fill, void* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!grid || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (sx < 0 || sx >= w || sy < 0 || sy >= h || sz < 0 || sz >= d) return fail(PCU_B200_INVALID_ARGUMENT, "seed point must be inside grid");
    if (w > 0x7fffffffLL || h > 0x7fffffffLL || d > 0x7fffffffLL || w * h > 0x7fffffffLL || w * h * d > 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "flood_fill_3d: grids of at most 2^31 - 1 voxels are supported, got %lld x %lld x %lld", w, h, d);
    PCU_ON_DEVICE(ws);
    const long long seed = (sx * h + sy) * d + sz;
    switch (kind) {
        case PCU_B200_GRID_I32: return ff_device<int>(ws, (const int*)grid, w, h, d, seed, fill, (int*)out, stream);
        case PCU_B200_GRID_I64: return ff_device<long long>(ws, (const long long*)grid, w, h, d, seed, fill, (long long*)out, stream);
        case PCU_B200_GRID_F32: return ff_device<float>(ws, (const float*)grid, w, h, d, seed, fill, (float*)out, stream);
        case PCU_B200_GRID_F64: return ff_device<double>(ws, (const double*)grid, w, h, d, seed, fill, (double*)out, stream);
        default: return fail(PCU_B200_INVALID_ARGUMENT, "unknown grid kind %d", kind);
    }
}

// ---- watertight manifold remeshing (watertight.cuh) ---------------------------------------------------------------
// A block of device memory that lives for one call, freed in the order of its stream.
struct CallBlock {
    unsigned char* p = nullptr;
    cudaStream_t stream = nullptr;
    explicit CallBlock(cudaStream_t s) : stream(s) {}
    ~CallBlock() { reset(); }
    void reset() { if (p) cudaFreeAsync(p, stream); p = nullptr; }
};

// The grid of DESIGN.md §3: c = (lo + hi) / 2, L = 1.4 max_a (hi_a - lo_a), o = c - L / 2, every operation rounded.
struct WtFrame { double o[3], L; };

// Bounds of v (first synchronisation), then per depth the counting pass (one synchronisation) and, where its pair
// count reaches the resolution, the grid pass (one more): the depth, the occupancy bytes of its grid in *grid.
template <typename T>
int wt_depth_search(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, double resolution,
                    CallBlock& grid, WtFrame& fr, int& depth, cudaStream_t stream) {
    const long long tiles = (m + kThreads - 1) / kThreads;
    struct { VxFace* faces; unsigned long long* local; unsigned long long* tile; VxCounts* counts; WtBounds* bounds; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.faces = cv.take<VxFace>((size_t)m);
        sc.local = cv.take<unsigned long long>((size_t)m);
        sc.tile = cv.take<unsigned long long>((size_t)tiles);
        sc.counts = cv.take<VxCounts>(1);
        sc.bounds = cv.take<WtBounds>(1);
    }));
    WtBounds b;
    for (int k = 0; k < 3; ++k) { b.lo[k] = LLONG_MAX; b.hi[k] = LLONG_MIN; }
    b.bad = 0;
    PCU_CUDA(cudaMemcpyAsync(sc.bounds, &b, sizeof b, cudaMemcpyHostToDevice, stream));
    PCU_LAUNCH((wt_bounds_kernel<T>), (unsigned)std::min<long long>(blocks_for(nv), (long long)ws->sm_count * 8), kThreads, stream, v, nv,
               sc.bounds);
    PCU_TRY(read_record(sc.bounds, &b, stream));
    if (b.bad) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: v has %llu non-finite coordinates", b.bad);
    double ext = 0.0, c[3];
    for (int k = 0; k < 3; ++k) {
        const auto unord = [](long long x) { x = x >= 0 ? x : x ^ 0x7fffffffffffffffll; double d; std::memcpy(&d, &x, 8); return d; };
        const double lo = unord(b.lo[k]), hi = unord(b.hi[k]);
        const volatile double sum = lo + hi, width = hi - lo;
        c[k] = sum / 2.0;
        ext = std::max(ext, (double)width);
    }
    if (!(ext > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: the mesh has zero extent (every vertex is the same point)");
    const volatile double L = 1.4 * ext;
    fr.L = L;
    if (!std::isfinite(fr.L)) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: the mesh's extent %g overflows fp64", ext);
    for (int k = 0; k < 3; ++k) { const volatile double h = fr.L / 2.0; fr.o[k] = c[k] - h; }
    for (depth = kWtMinDepth;; ++depth) {
        const double s = std::ldexp(fr.L, -depth);
        VxGeom g;
        for (int k = 0; k < 3; ++k) { const volatile double hs = s / 2.0, ok = fr.o[k] + hs; g.o[k] = ok; g.s[k] = s; g.h[k] = hs; }
        PCU_CUDA(cudaMemsetAsync(sc.counts, 0, sizeof(VxCounts), stream));
        PCU_LAUNCH((vx_bounds_kernel<T>), (unsigned)tiles, kThreads, stream, v, nv, f, fkind, m, g, sc.faces, sc.local, sc.tile, sc.counts);
        PCU_LAUNCH(vx_tiles_kernel, 1, 1024, stream, sc.tile, tiles, sc.counts);
        PCU_LAUNCH((vx_test_kernel<T, kVxCount>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
                   (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr, (unsigned*)nullptr, 0);
        VxCounts cnt;
        PCU_TRY(read_record(sc.counts, &cnt, stream));
        if (cnt.bad_corner) return bad_corners(cnt.bad_corner);
        if (cnt.bad_bounds || !(cnt.cand_d < kVxMaxCandidates))   // not reached: the mesh lies inside the grid
            return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: voxel bounds out of range at depth %d", depth);
        if ((double)cnt.accepted < resolution && depth < kWtMaxDepth) continue;   // occupied <= accepted pairs
        const size_t bytes = (size_t)1 << (3 * depth);
        grid.reset();
        PCU_TRY(alloc_block(grid.p, bytes, stream, "make_mesh_watertight's occupancy grid"));
        PCU_CUDA(cudaMemsetAsync(grid.p, 0, bytes, stream));
        PCU_LAUNCH((vx_test_kernel<T, kVxGrid>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
                   (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr, (unsigned*)grid.p, depth);
        PCU_TRY(read_record(sc.counts, &cnt, stream));
        if ((double)cnt.occupied >= resolution || depth == kWtMaxDepth) return PCU_B200_OK;
    }
}

// The exterior and the surface of the occupancy grid (two synchronisations: the counts, then nothing until the
// projection), into the handle's block: x (nv, 3) fp64 pre-projection vertices, faces (nf, 3) int32.
int wt_surface(pcu_b200_workspace* ws, pcu_b200_watertight* h, unsigned char* grid, int lg, const WtFrame& fr, CallBlock& dense,
               cudaStream_t stream) {
    const long long N = 1ll << lg, n = N * N * N;
    PCU_TRY(alloc_block(dense.p, sizeof(int) * (size_t)n, stream, "make_mesh_watertight's voxel labels"));
    int* P = (int*)dense.p;
    FfShape sh;
    sh.w = sh.h = sh.d = N; sh.n = n; sh.seed = 0;
    sh.lz = ff_log2_cover(N, 5);
    sh.ly = ff_log2_cover(N, 8 - sh.lz);
    sh.lx = ff_log2_cover(N, 10 - sh.lz - sh.ly);
    sh.tz_n = (unsigned)((N + (1ll << sh.lz) - 1) >> sh.lz);
    sh.ty_n = (unsigned)((N + (1ll << sh.ly) - 1) >> sh.ly);
    const long long ftiles = ((N + (1ll << sh.lx) - 1) >> sh.lx) * sh.ty_n * sh.tz_n;
    PCU_LAUNCH((ff_tile_kernel<unsigned char>), (unsigned)ftiles, kThreads, stream, (const unsigned char*)grid, sh, P);
    PCU_LAUNCH((ff_cross_kernel<unsigned char>), (unsigned)ftiles, kThreads, stream, (const unsigned char*)grid, sh, P);
    PCU_LAUNCH(wt_exterior_kernel, blocks_for(n), kThreads, stream, grid, n, P);
    const unsigned tiles = blocks_for(n);
    struct { unsigned* sum; unsigned long long* v0; unsigned long long* f0; McCounts* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sum = cv.take<unsigned>(tiles);
        sc.v0 = cv.take<unsigned long long>(tiles);
        sc.f0 = cv.take<unsigned long long>(tiles);
        sc.counts = cv.take<McCounts>(1);
    }));
    PCU_LAUNCH(wt_count_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, sc.sum);
    PCU_LAUNCH(mc_tiles_kernel, 1, 1024, stream, (const unsigned*)sc.sum, (long long)tiles, sc.v0, sc.f0, sc.counts);
    McCounts c;
    PCU_TRY(read_record(sc.counts, &c, stream));
    if (c.slots >= 0x7fffffffull || c.faces >= 0x7fffffffull)
        return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: at most 2^31 - 2 vertices and faces are supported, got %llu and %llu",
                    c.slots, c.faces);
    h->nv = (long long)c.slots;
    h->nf = (long long)c.faces;
    const auto carve = [&](Carver& cv) {
        h->x = cv.take<double>(3 * (size_t)h->nv);
        h->faces = cv.take<int>(3 * (size_t)h->nf);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "make_mesh_watertight"));
    carve_at(h->block, carve);
    WtPlace pl;
    for (int k = 0; k < 3; ++k) pl.o[k] = fr.o[k];
    pl.s = std::ldexp(fr.L, -lg);
    PCU_LAUNCH(wt_verts_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, (const unsigned long long*)sc.v0,
               (const unsigned long long*)sc.f0, pl, P, const_cast<double*>(h->x));
    PCU_LAUNCH(wt_faces_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, (const unsigned long long*)sc.v0,
               (const unsigned long long*)sc.f0, (const int*)P, const_cast<int*>(h->faces));
    return PCU_B200_OK;
}

constexpr int kWtRounds = 10;

// The projection rounds of DESIGN.md §3 on h->x: the input's fp64 tree once, then per round the closest points, the
// proposals, flip passes until none is flipped (one synchronisation each) and the commit.
template <typename T>
int wt_project(pcu_b200_workspace* ws, pcu_b200_watertight* h, const T* v, long long nv, const void* f, long long m, int fkind,
               cudaStream_t stream) {
    const long long n = h->nv, nf = h->nf;
    if (n == 0) return PCU_B200_OK;
    struct { unsigned char* tree; double* v64; double* x0; double* y; double* alpha; int* rev; double* d; long long* fidx; double* bc;
             unsigned long long* flipped; } sc;
    MeshTree<Pt<double>> t;
    const auto carve = [&](Carver& cv) {
        sc.tree = cv.take<unsigned char>(carve_at(nullptr, [&](Carver& c2) { carve_mesh_tree<Pt<double>>(c2, m, false, t); }));
        sc.v64 = sizeof(T) == 8 ? nullptr : cv.take<double>(3 * (size_t)nv);
        sc.x0 = cv.take<double>(3 * (size_t)n);
        sc.y = cv.take<double>(3 * (size_t)n);
        sc.alpha = cv.take<double>((size_t)n);
        sc.rev = cv.take<int>((size_t)n);
        sc.d = cv.take<double>((size_t)n);
        sc.fidx = cv.take<long long>((size_t)n);
        sc.bc = cv.take<double>(3 * (size_t)n);
        sc.flipped = cv.take<unsigned long long>(2);
    };
    CallBlock blk(stream);
    PCU_TRY(alloc_block(blk.p, carve_at(nullptr, carve), stream, "make_mesh_watertight's projection"));
    carve_at(blk.p, carve);
    const double* v64 = (const double*)v;
    if (sizeof(T) != 8) {
        PCU_LAUNCH((wt_widen_kernel<T>), blocks_for(3 * nv), kThreads, stream, v, 3 * nv, sc.v64);
        v64 = sc.v64;
    }
    PCU_TRY(build_mesh_tree<double>(ws, v64, nv, f, m, fkind, false, sc.flipped + 1, stream, t, sc.tree));
    double* x = const_cast<double*>(h->x);
    const unsigned vb = blocks_for(n), fb = blocks_for(nf);
    PCU_LAUNCH(wt_start_kernel, vb, kThreads, stream, (const double*)x, n, sc.x0, sc.alpha);
    for (int round = 0; round < kWtRounds; ++round) {
        PCU_LAUNCH((mq_query_kernel<double>), query_blocks(ws, n), kThreads, stream, (const double*)x, n, m, (const MqScratch*)t.sc,
                   (const MqNode*)t.nodes, (const Pt<double>*)t.leaves, sc.d, (void*)sc.fidx, 1, sc.bc);
        PCU_LAUNCH(wt_propose_kernel, vb, kThreads, stream, v64, nv, f, fkind, (const long long*)sc.fidx, (const double*)sc.bc,
                   (const double*)x, (const double*)sc.alpha, n, sc.y);
        PCU_CUDA(cudaMemsetAsync(sc.rev, 0, sizeof(int) * (size_t)n, stream));
        for (int pass = 1;; ++pass) {
            PCU_CUDA(cudaMemsetAsync(sc.flipped, 0, sizeof(unsigned long long), stream));
            PCU_LAUNCH(wt_flip_kernel, fb, kThreads, stream, h->faces, nf, (const double*)sc.x0, (const double*)x, (const double*)sc.y,
                       sc.rev, pass, sc.flipped);
            unsigned long long flipped = 0;
            PCU_TRY(read_record(sc.flipped, &flipped, stream));
            if (flipped == 0) break;
        }
        PCU_LAUNCH(wt_commit_kernel, vb, kThreads, stream, (const double*)sc.y, (const int*)sc.rev, n, x, sc.alpha);
    }
    return PCU_B200_OK;
}

template <typename T>
int make_mesh_watertight_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind,
                                        double resolution, pcu_b200_watertight** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: at most 2^31 - 2 vertices and faces are supported");
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_watertight* h) -> int {
        h->t_f64 = sizeof(T) == 8;
        h->fkind = fkind;
        CallBlock grid(stream), dense(stream);
        WtFrame fr;
        PCU_TRY(wt_depth_search<T>(ws, v, nv, f, m, fkind, resolution, grid, fr, h->depth, stream));
        PCU_TRY(wt_surface(ws, h, grid.p, h->depth, fr, dense, stream));
        grid.reset();
        dense.reset();
        const long long most = fkind == kIdxI32 ? (1ll << 31) : fkind == kIdxU32 ? (1ll << 32) : LLONG_MAX;
        if (h->nv > most) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: %lld vertices cannot be indexed by f's dtype", h->nv);
        return wt_project<T>(ws, h, v, nv, f, m, fkind, stream);
    }));
    out_counts[0] = (*out)->nv;
    out_counts[1] = (*out)->nf;
    out_counts[2] = (*out)->depth;
    return PCU_B200_OK;
}

int make_mesh_watertight_emit_device(pcu_b200_workspace* ws, const pcu_b200_watertight* h, void* out_v, void* out_f, cudaStream_t stream) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "watertight"));
    if (h->nv == 0 && h->nf == 0) return PCU_B200_OK;
    if (!out_v || !out_f) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(3 * std::max(h->nv, h->nf));
    if (h->t_f64) PCU_LAUNCH(wt_emit_kernel<double>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->nf, (int)wide_index(h->fkind), (double*)out_v, out_f);
    else PCU_LAUNCH(wt_emit_kernel<float>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->nf, (int)wide_index(h->fkind), (float*)out_v, out_f);
    return PCU_B200_OK;
}

// ---- mesh connected components and vertex removal (mesh_topology.cuh) ----------------------------------------------
// Persistent CTAs of cc_validate_kernel.
inline unsigned cc_validate_blocks(const pcu_b200_workspace* ws, long long total) {
    return (unsigned)std::max(1ll, std::min((long long)ws->sm_count * 8, (total + kThreads - 1) / kThreads));
}

// Validate f and read max(f) (first synchronisation); the labels and counts in the handle's block; read the component
// count (second synchronisation).
int cc_build(pcu_b200_workspace* ws, pcu_b200_components* h, const void* f, long long m, int c, int fkind, cudaStream_t stream) {
    CcCounts* rec = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { rec = cv.take<CcCounts>(1); }));
    PCU_CUDA(cudaMemsetAsync(rec, 0, sizeof(CcCounts), stream));
    const long long total = m * c;
    PCU_LAUNCH(cc_validate_kernel, cc_validate_blocks(ws, total), kThreads, stream, f, fkind, total, rec);
    CcCounts hc;
    PCU_TRY(read_record(rec, &hc, stream));
    if (hc.bad)
        return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: %llu face indices are negative or above 2^31 - 2", hc.bad);
    const long long n = (long long)hc.max_index + 1;
    struct { int *P, *root, *rank, *nv, *nf, *cf; unsigned char* is_root; unsigned* counts; } b;
    const auto carve = [&](Carver& cv) {
        b.P = cv.take<int>((size_t)n);
        b.root = cv.take<int>((size_t)n);
        b.rank = cv.take<int>((size_t)n);
        b.nv = cv.take<int>((size_t)n);
        b.nf = cv.take<int>((size_t)n);
        b.cf = cv.take<int>((size_t)m);
        b.is_root = cv.take<unsigned char>((size_t)n);
        b.counts = cv.take<unsigned>(keep_count_words(n));
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "connected components"));
    carve_at(h->block, carve);
    PCU_CUDA(cudaMemsetAsync(b.nv, 0, sizeof(int) * (size_t)n, stream));
    PCU_CUDA(cudaMemsetAsync(b.nf, 0, sizeof(int) * (size_t)n, stream));
    PCU_LAUNCH(cc_init_kernel, blocks_for(n), kThreads, stream, b.P, n);
    PCU_LAUNCH(cc_hook_kernel, blocks_for(m), kThreads, stream, f, fkind, m, c, b.P);
    PCU_LAUNCH(cc_flatten_kernel, blocks_for(n), kThreads, stream, b.P, n, b.root, b.is_root);
    PCU_TRY(enqueue_keep_offsets(b.is_root, n, b.counts, &rec->ncomp, stream));
    PCU_LAUNCH(cc_rank_kernel, blocks_for(n), kThreads, stream, (const unsigned char*)b.is_root, n, (const unsigned*)b.counts, b.rank);
    PCU_LAUNCH(cc_label_kernel, blocks_for(n), kThreads, stream, b.root, n, (const int*)b.rank, b.nv);
    PCU_LAUNCH(cc_face_kernel, blocks_for(m), kThreads, stream, f, fkind, m, c, (const int*)b.root, b.cf, b.nf);
    PCU_TRY(read_record(rec, &hc, stream));
    h->n = n;
    h->m = m;
    h->k = hc.ncomp;
    h->cv = b.root;
    h->cf = b.cf;
    h->nv = b.nv;
    h->nf = b.nf;
    return PCU_B200_OK;
}

int connected_components_prepare_device(pcu_b200_workspace* ws, const void* f, long long m, int c, int fkind, pcu_b200_components** out,
                                        long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (m <= 0 || c <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: f must have at least one row and one column");
    if (m >= 0x7fffffffLL || m * c >= (1ll << 40))
        return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: at most 2^31 - 2 faces are supported, got %lld x %d", m, c);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_components* h) {
        h->fkind = fkind;
        return cc_build(ws, h, f, m, c, fkind, stream);
    }));
    out_counts[0] = (*out)->n;
    out_counts[1] = (*out)->k;
    return PCU_B200_OK;
}

int connected_components_emit_device(pcu_b200_workspace* ws, const pcu_b200_components* h, void* out_cv, void* out_nv, void* out_cf,
                                     void* out_nf, cudaStream_t stream) {
    if (!ws || !h || !out_cv || !out_nv || !out_cf || !out_nf) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "components"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(std::max(h->n, h->m));
    if (wide_index(h->fkind))
        PCU_LAUNCH(cc_emit_kernel<long long>, blocks, kThreads, stream, h->cv, h->n, h->cf, h->m, h->nv, h->nf, h->k, (long long*)out_cv,
                   (long long*)out_cf, (long long*)out_nv, (long long*)out_nf);
    else
        PCU_LAUNCH(cc_emit_kernel<int>, blocks, kThreads, stream, h->cv, h->n, h->cf, h->m, h->nv, h->nf, h->k, (int*)out_cv, (int*)out_cf,
                   (int*)out_nv, (int*)out_nf);
    return PCU_B200_OK;
}

// Arguments shared by the two removals.
int mt_check(const pcu_b200_workspace* ws, const void* v, long long nv, const void* f, long long m, int fkind) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "at most 2^31 - 2 vertices and faces are supported, got %lld and %lld", nv, m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

template <typename T>
int remove_mesh_vertices_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind,
                                const unsigned char* mask, T* out_v, void* out_f, long long* out_counts, cudaStream_t stream) {
    PCU_TRY(mt_check(ws, v, nv, f, m, fkind));
    if (fkind != kIdxI32 && fkind != kIdxI64) return fail(PCU_B200_INVALID_ARGUMENT, "remove_mesh_vertices: f must be int32 or int64");
    if (!mask || !out_v || !out_f || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    struct { MtCounts* rec; int* remap; unsigned* vcounts; unsigned char* keep; unsigned* fcounts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MtCounts>(1);
        sc.remap = cv.take<int>((size_t)nv);
        sc.vcounts = cv.take<unsigned>(keep_count_words(nv));
        sc.keep = cv.take<unsigned char>((size_t)m);
        sc.fcounts = cv.take<unsigned>(keep_count_words(m));
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MtCounts), stream));
    PCU_TRY(enqueue_keep_offsets(mask, nv, sc.vcounts, &sc.rec->kept_v, stream));
    PCU_LAUNCH(rmv_vertex_kernel<T>, blocks_for(nv), kThreads, stream, v, nv, mask, (const unsigned*)sc.vcounts, out_v, sc.remap);
    PCU_LAUNCH(rmv_face_flag_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const int*)sc.remap, sc.keep, sc.rec);
    PCU_TRY(enqueue_keep_offsets(sc.keep, m, sc.fcounts, &sc.rec->kept_f, stream));
    if (wide_index(fkind))
        PCU_LAUNCH(rmv_face_emit_kernel<long long>, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const unsigned char*)sc.keep,
                   (const unsigned*)sc.fcounts, (const int*)sc.remap, (long long*)out_f);
    else
        PCU_LAUNCH(rmv_face_emit_kernel<int>, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const unsigned char*)sc.keep,
                   (const unsigned*)sc.fcounts, (const int*)sc.remap, (int*)out_f);
    MtCounts hc;
    PCU_TRY(read_record(sc.rec, &hc, stream));
    if (hc.bad) return bad_corners(hc.bad);
    out_counts[0] = hc.kept_v;
    out_counts[1] = hc.kept_f;
    return PCU_B200_OK;
}

template <typename T, typename I>
int rur_launch(const T* v, long long nv, const void* f, long long m, int fkind, const unsigned char* used, const unsigned* vcounts,
               T* out_v, void* out_f, void* out_j, void* out_i, cudaStream_t stream) {
    PCU_LAUNCH((rur_vertex_kernel<T, I>), blocks_for(nv), kThreads, stream, v, nv, used, vcounts, out_v, (I*)out_j, (I*)out_i);
    PCU_LAUNCH(rur_face_kernel<I>, blocks_for(3 * m), kThreads, stream, f, fkind, 3 * m, nv, (const I*)out_i, (I*)out_f);
    return PCU_B200_OK;
}

template <typename T>
int remove_unreferenced_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, T* out_v,
                               void* out_f, void* out_j, void* out_i, long long* out_count, cudaStream_t stream) {
    PCU_TRY(mt_check(ws, v, nv, f, m, fkind));
    if (!out_v || !out_f || !out_j || !out_i || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    struct { MtCounts* rec; unsigned char* used; unsigned* vcounts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MtCounts>(1);
        sc.used = cv.take<unsigned char>((size_t)nv);
        sc.vcounts = cv.take<unsigned>(keep_count_words(nv));
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MtCounts), stream));
    PCU_CUDA(cudaMemsetAsync(sc.used, 0, (size_t)nv, stream));
    PCU_LAUNCH(rur_mark_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, sc.used, sc.rec);
    PCU_TRY(enqueue_keep_offsets(sc.used, nv, sc.vcounts, &sc.rec->kept_v, stream));
    if (wide_index(fkind))
        PCU_TRY((rur_launch<T, long long>(v, nv, f, m, fkind, sc.used, sc.vcounts, out_v, out_f, out_j, out_i, stream)));
    else
        PCU_TRY((rur_launch<T, int>(v, nv, f, m, fkind, sc.used, sc.vcounts, out_v, out_f, out_j, out_i, stream)));
    MtCounts hc;
    PCU_TRY(read_record(sc.rec, &hc, stream));
    if (hc.bad) return bad_corners(hc.bad);
    *out_count = hc.kept_v;
    return PCU_B200_OK;
}

// ---- consistent face orientation (orient.cuh) ----------------------------------------------------------------------
// K = the half-edge records' word, I = f's width.  Every buffer is sized by m: no synchronisation.
template <typename K, typename I>
int orient_launch(pcu_b200_workspace* ws, const void* f, long long m, int fkind, I* out_f, I* out_c, cudaStream_t stream) {
    using Rec = OmRec<K>;
    const long long n = 3 * m;
    struct { SortScratch<Rec> sort; int *P, *nb, *root, *rank, *next; unsigned char *flag, *enq; unsigned* counts; long long* seeds; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.P = cv.take<int>(2 * (size_t)m);
        sc.nb = cv.take<int>((size_t)n);
        sc.root = cv.take<int>((size_t)m);
        sc.rank = cv.take<int>((size_t)m);
        sc.next = cv.take<int>((size_t)m);
        sc.flag = cv.take<unsigned char>((size_t)m);
        sc.enq = cv.take<unsigned char>((size_t)m);
        sc.counts = cv.take<unsigned>(keep_count_words(m));
        sc.seeds = cv.take<long long>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.nb, 0xff, sizeof(int) * (size_t)n, stream));
    PCU_CUDA(cudaMemsetAsync(sc.enq, 0, (size_t)m, stream));
    PCU_LAUNCH(om_records_kernel<K>, blocks_for(m), kThreads, stream, f, fkind, m, sc.sort.a, sc.P);
    Rec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 2, stream, &sorted));
    PCU_LAUNCH(om_runs_kernel<K>, blocks_for(n), kThreads, stream, (const Rec*)sorted, n, m, f, fkind, sc.nb, sc.P);
    PCU_LAUNCH(om_flatten_kernel, blocks_for(m), kThreads, stream, sc.P, m, sc.root, sc.flag);
    PCU_TRY(enqueue_keep_offsets(sc.flag, m, sc.counts, sc.seeds, stream));
    PCU_LAUNCH(cc_rank_kernel, blocks_for(m), kThreads, stream, (const unsigned char*)sc.flag, m, (const unsigned*)sc.counts, sc.rank);
    PCU_LAUNCH(om_emit_kernel<I>, blocks_for(m), kThreads, stream, (const I*)f, m, (const int*)sc.root, (const int*)sc.rank, out_f, out_c);
    PCU_LAUNCH(om_replay_kernel<I>, blocks_for(m), kThreads, stream, (const unsigned char*)sc.flag, m, (const int*)sc.nb, sc.enq, sc.next,
               out_f);
    return PCU_B200_OK;
}

int orient_mesh_faces_device(pcu_b200_workspace* ws, const void* f, long long m, int fkind, void* out_f, void* out_c, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!f || !out_f || !out_c) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (m <= 0 || m > kOmMaxFaces)
        return fail(PCU_B200_INVALID_ARGUMENT, "orient_mesh_faces: between 1 and 2^30 - 1 faces are supported, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    return wide_index(fkind) ? orient_launch<unsigned long long, long long>(ws, f, m, fkind, (long long*)out_f, (long long*)out_c, stream)
                             : orient_launch<unsigned, int>(ws, f, m, fkind, (int*)out_f, (int*)out_c, stream);
}

// ---- mesh normals, face areas and Laplacian smoothing (mesh_geometry.cuh, laplacian.cuh) ---------------------------
// Arguments shared by the four entry points.  6 m records must fit int32 positions.
int mg_check(const pcu_b200_workspace* ws, const void* v, long long nv, const void* f, long long m, int fkind, const void* out) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!v || !f || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m > 0x7fffffffLL / 6)
        return fail(PCU_B200_INVALID_ARGUMENT, "at most 2^31 - 2 vertices and 357913941 faces are supported, got %lld and %lld", nv, m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

// CTAs of the kernels that reduce (reduce_grid): a function of the row count alone, so the sums' order is too.
inline unsigned mg_blocks(long long n) { return std::min<unsigned>(kMgBlocks, blocks_for(n)); }

// Bits of the largest vertex index n - 1 (at least 1).
inline int mg_index_bits(long long n) {
    int b = 1;
    while (b < 31 && ((n - 1) >> b) != 0) ++b;
    return b;
}

// One face pass over v (T = the type of v; double for the smoothing's fp64 iterate).
template <typename T>
int mg_face_pass(const T* v, long long nv, const void* f, int fkind, long long m, const FaceOut<T>& out, MgRecord* rec, cudaStream_t stream) {
    PCU_LAUNCH(mg_face_kernel<T>, mg_blocks(m), kThreads, stream, v, nv, f, fkind, m, out, rec);
    return PCU_B200_OK;
}

// The corner CSR of the nv vertices: first (nv + 1) and corner (3 m), through the stable sort of the corner records
// (sort: scratch for at least 3 m records).
int enqueue_incidence(const SortScratch<MgRec>& sort, const void* f, int fkind, long long m, long long nv, int* first, int* corner,
                      cudaStream_t stream) {
    const long long n = 3 * m;
    PCU_LAUNCH(mg_corner_kernel, blocks_for(n), kThreads, stream, f, fkind, n, nv, sort.a);
    MgRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sort, n, 1, stream, &sorted, mg_index_bits(nv)));
    PCU_LAUNCH(mg_rows_kernel, blocks_for(n + 1), kThreads, stream, (const MgRec*)sorted, n, nv, first, corner, 0);
    return PCU_B200_OK;
}

// mesh_face_areas (normal == false) or estimate_mesh_face_normals (normal == true): one face pass, one synchronisation.
template <typename T>
int mesh_face_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, bool normal, T* out,
                     cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    PCU_ON_DEVICE(ws);
    MgRecord* rec = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { rec = cv.take<MgRecord>(1); }));
    PCU_CUDA(cudaMemsetAsync(rec, 0, sizeof(MgRecord), stream));
    FaceOut<T> o = {};
    if (normal) o.normal = out; else o.area = out;
    PCU_TRY(mg_face_pass<T>(v, nv, f, fkind, m, o, rec, stream));
    MgRecord host;
    PCU_TRY(read_record(rec, &host, stream));
    return host.bad ? bad_corners(host.bad) : PCU_B200_OK;
}

// estimate_mesh_vertex_normals, weighting 0 uniform, 1 area, 2 angle: face pass, corner CSR, vertex pass; one
// synchronisation.
template <typename T>
int vertex_normals_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, int weighting, T* out,
                          cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    if (weighting < 0 || weighting > 2) return fail(PCU_B200_INVALID_ARGUMENT, "unknown weighting %d", weighting);
    PCU_ON_DEVICE(ws);
    struct { MgRecord* rec; double *unit, *weight; SortScratch<MgRec> sort; int *first, *corner; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MgRecord>(1);
        sc.unit = cv.take<double>(3 * (size_t)m);
        sc.weight = weighting ? cv.take<double>(3 * (size_t)m) : nullptr;
        sc.sort.carve(cv, 3 * m);
        sc.first = cv.take<int>((size_t)nv + 1);
        sc.corner = cv.take<int>(3 * (size_t)m);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MgRecord), stream));
    FaceOut<T> o = {};
    o.unit = sc.unit;
    o.weight = sc.weight;
    o.weighting = weighting;
    PCU_TRY(mg_face_pass<T>(v, nv, f, fkind, m, o, sc.rec, stream));
    PCU_TRY(enqueue_incidence(sc.sort, f, fkind, m, nv, sc.first, sc.corner, stream));
    PCU_LAUNCH(mg_vertex_normal_kernel<T>, blocks_for(nv), kThreads, stream, (const int*)sc.first, (const int*)sc.corner, nv,
               (const double*)sc.unit, (const double*)sc.weight, out);
    MgRecord host;
    PCU_TRY(read_record(sc.rec, &host, stream));
    return host.bad ? bad_corners(host.bad) : PCU_B200_OK;
}

constexpr int kCgWindow = 16;   // CG iterations enqueued between two reads of the solver's record

// The buffers of one smoothing call.
struct LapScratch {
    LapRecord* rec;
    double *u, *r, *z, *p, *q, *mass, *halfcot, *dbla, *partial, *val, *diag;
    SortScratch<MgRec> sort;
    MgRec* rows;
    unsigned char *head, *lone;
    unsigned* counts;
    int *col, *rowptr, *first, *corner;
    void carve(Carver& cv, long long nv, long long m, bool cotan) {
        const size_t n3 = 3 * (size_t)nv, e = 6 * (size_t)m;
        rec = cv.take<LapRecord>(1);
        u = cv.take<double>(n3); r = cv.take<double>(n3); z = cv.take<double>(n3); p = cv.take<double>(n3); q = cv.take<double>(n3);
        mass = cotan ? cv.take<double>((size_t)nv) : nullptr;
        halfcot = cv.take<double>(3 * (size_t)m);
        dbla = cotan ? cv.take<double>((size_t)m) : nullptr;
        partial = cv.take<double>((size_t)kMgBlocks * 9);
        sort.carve(cv, (long long)e);
        rows = cv.take<MgRec>(e);
        head = cv.take<unsigned char>(e);
        counts = cv.take<unsigned>(keep_count_words((long long)e));
        col = cv.take<int>(e);
        val = cv.take<double>(e);
        rowptr = cv.take<int>((size_t)nv + 1);
        diag = cv.take<double>((size_t)nv);
        lone = cv.take<unsigned char>((size_t)nv);
        first = cotan ? cv.take<int>((size_t)nv + 1) : nullptr;
        corner = cotan ? cv.take<int>(3 * (size_t)m) : nullptr;
    }
};

// Reads the record (one synchronisation) and fails on a mesh of zero total area.
int lap_read(const LapRecord* rec, LapRecord* host, cudaStream_t stream) {
    PCU_TRY(read_record(rec, host, stream));
    if (host->mesh.zero_area) return fail(PCU_B200_INVALID_ARGUMENT, "laplacian_smooth_mesh: the mesh has zero total area");
    return PCU_B200_OK;
}

// The cotangent Laplacian of u in the scratch's CSR; reads the record once (corners, finiteness, entries).
int lap_assemble(LapScratch& s, const void* f, int fkind, long long m, long long nv, bool cotan, cudaStream_t stream) {
    const long long e = 6 * m;
    const int bits = mg_index_bits(nv);
    FaceOut<double> o = {};
    o.halfcot = s.halfcot;
    PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
    PCU_LAUNCH(lap_edge_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, bits, s.sort.a);
    MgRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(s.sort, e, 1, stream, &sorted, 2 * bits));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(e), kThreads, stream, (const McRec*)sorted, e, s.head);
    PCU_TRY(enqueue_keep_offsets(s.head, e, s.counts, &s.rec->mesh.nnz, stream));
    PCU_LAUNCH(lap_entries_kernel, blocks_for(e), kThreads, stream, (const MgRec*)sorted, e, (const unsigned char*)s.head,
               (const unsigned*)s.counts, (const double*)s.halfcot, bits, s.rows, s.col, s.val);
    if (cotan) PCU_TRY(enqueue_incidence(s.sort, f, fkind, m, nv, s.first, s.corner, stream));
    LapRecord host;
    PCU_TRY(lap_read(s.rec, &host, stream));
    if (host.mesh.bad) return bad_corners(host.mesh.bad);
    if (host.mesh.nonfinite)
        return fail(PCU_B200_INVALID_ARGUMENT, "laplacian_smooth_mesh: v has %llu coordinates that are not finite", host.mesh.nonfinite);
    PCU_LAUNCH(mg_rows_kernel, blocks_for(host.mesh.nnz + 1), kThreads, stream, (const MgRec*)s.rows, host.mesh.nnz, nv, s.rowptr,
               (int*)nullptr, 0);
    PCU_LAUNCH(lap_diag_kernel, blocks_for(nv), kThreads, stream, (const int*)s.rowptr, (const double*)s.val, nv, s.diag, s.lone);
    return PCU_B200_OK;
}

// One CG solve of S u' = M u in place; reads the record once per window of kCgWindow iterations.  Returns the
// iterations and the largest |r| / |b| of the three columns at exit.
int lap_solve(const LapScratch& s, const LapSystem& sys, int max_iters, int* out_iters, double* out_residual, cudaStream_t stream) {
    const long long n = sys.n;
    const unsigned blocks = mg_blocks(n);
    PCU_CUDA(cudaMemsetAsync(&s.rec->cg, 0, sizeof(CgState), stream));
    PCU_LAUNCH(lap_cg_init_kernel, blocks, kThreads, stream, sys, (const double*)s.u, s.r, s.z, s.p, s.partial, s.rec);
    LapRecord host;
    for (;;) {
        for (int k = 0; k < kCgWindow; ++k) {
            PCU_LAUNCH(lap_cg_spmv_kernel, blocks, kThreads, stream, sys, (const double*)s.p, s.q, s.partial, s.rec);
            PCU_LAUNCH(lap_cg_update_kernel, blocks, kThreads, stream, sys, s.u, s.r, s.z, (const double*)s.p, (const double*)s.q, s.partial,
                       max_iters, s.rec);
            PCU_LAUNCH(lap_cg_direction_kernel, blocks_for(3 * n), kThreads, stream, n, (const double*)s.z, s.p, (const LapRecord*)s.rec);
        }
        PCU_TRY(lap_read(s.rec, &host, stream));
        if (host.cg.done) break;
    }
    double worst = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double rr = host.cg.rr[c], bb = host.cg.bb[c];
        const double rel = bb > 0.0 ? std::sqrt(rr / bb) : (rr > 0.0 ? HUGE_VAL : 0.0);
        worst = std::max(worst, rel);
    }
    *out_iters = host.cg.iters;
    *out_residual = worst;
    return PCU_B200_OK;
}

// laplacian_smooth_mesh (src/smooth.cpp): out_iters / out_residual (host, num_iters entries) receive every step's CG
// iterations and its largest relative residual at exit.
template <typename T>
int laplacian_smooth_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, int num_iters,
                            double step_size, bool cotan, int max_cg_iters, T* out, int* out_iters, double* out_residual, cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    if (num_iters < 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid value for argument num_iters in smooth_mesh_laplacian. Must be a positive integer or 0.");
    if (max_cg_iters <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_cg_iters must be positive, got %d", max_cg_iters);
    if (num_iters > 0 && (!out_iters || !out_residual)) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    if (num_iters == 0) {
        PCU_TRY(adopt_stream(ws, stream));
        PCU_CUDA(cudaMemcpyAsync(out, v, 3 * (size_t)nv * sizeof(T), cudaMemcpyDeviceToDevice, stream));
        return PCU_B200_OK;
    }
    LapScratch s;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { s.carve(cv, nv, m, cotan); }));
    PCU_CUDA(cudaMemsetAsync(s.rec, 0, sizeof(LapRecord), stream));
    PCU_LAUNCH(lap_load_kernel<T>, blocks_for(3 * nv), kThreads, stream, v, 3 * nv, s.u, &s.rec->mesh);
    PCU_TRY(lap_assemble(s, f, fkind, m, nv, cotan, stream));
    const LapSystem sys = {s.rowptr, s.col, s.val, s.diag, s.mass, cotan ? step_size * 1e-3 : step_size, nv};
    for (int it = 0; it < num_iters; ++it) {
        if (cotan) {
            FaceOut<double> o = {};
            o.dbla = s.dbla;
            o.partial = s.partial;
            PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
            PCU_LAUNCH(lap_mass_kernel, blocks_for(nv), kThreads, stream, (const int*)s.first, (const int*)s.corner, nv, (const double*)s.dbla,
                       (const unsigned char*)s.lone, s.mass);
        }
        PCU_TRY(lap_solve(s, sys, max_cg_iters, out_iters + it, out_residual + it, stream));
        if (cotan) {
            FaceOut<double> o = {};
            o.partial = s.partial;
            PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
            PCU_LAUNCH(lap_rescale_kernel, blocks_for(3 * nv), kThreads, stream, s.u, nv, (const MgRecord*)&s.rec->mesh);
        }
    }
    PCU_LAUNCH(lap_store_kernel<T>, blocks_for(3 * nv), kThreads, stream, (const double*)s.u, 3 * nv, out);
    if (cotan) {
        LapRecord host;
        PCU_TRY(lap_read(s.rec, &host, stream));
    }
    return PCU_B200_OK;
}

// ---- Morton codes (SURVEY.md 8f N3) -------------------------------------------------------------------

template <typename I>
int morton_encode_device(pcu_b200_workspace* ws, const I* pts, long long n, unsigned long long* out_codes, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    if (!out_codes) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH((morton_encode_kernel<I>), blocks_for(n), kThreads, stream, pts, n, out_codes);
    return PCU_B200_OK;
}

int morton_decode_device(pcu_b200_workspace* ws, const unsigned long long* codes, long long n, int* out_pts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!codes || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    if (!out_pts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_decode_kernel, blocks_for(n), kThreads, stream, codes, n, out_pts);
    return PCU_B200_OK;
}

int morton_addsub_device(pcu_b200_workspace* ws, const unsigned long long* a, const unsigned long long* b, long long n, int op,
                         unsigned long long* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes_1 and codes_2 must be arrays of shape [n,] but got an empty array");
    if (!out) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_addsub_kernel, blocks_for(n), kThreads, stream, a, b, n, op, out);
    return PCU_B200_OK;
}

int morton_knn_device(pcu_b200_workspace* ws, const unsigned long long* codes, long long n, const unsigned long long* qcodes,
                      long long m, int k, int sort_dist, long long* out_idx, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "k must be greater than 0");
    if (!codes || n <= 0 || !qcodes || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    if ((long long)k > n) return fail(PCU_B200_INVALID_ARGUMENT, "k (%d) exceeds the number of codes (%lld): clamp it first (morton.cpp:351)", k, n);
    if (!out_idx) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_knn_kernel, blocks_for(m), kThreads, stream, codes, n, qcodes, m, k, sort_dist, out_idx);
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

// ---- voxel-grid down-sampling (SURVEY.md 8f N2) -----------------------------------------------------------
template <typename T, typename A>
int voxel_downsample_device(pcu_b200_workspace* ws, const T* pts, long long n, const A* attr, int attr_cols, const double size[3],
                            const double min_bound[3], const double max_bound[3], int min_points, T* out_pts, A* out_attr,
                            int* out_counts, long long* out_rows, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld rows)", n);
    if (!out_pts || !out_rows || attr_cols < 0 || (attr_cols > 0 && (!attr || !out_attr)))
        return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    VoxelGrid<T> g;
    for (int a = 0; a < 3; ++a) {   // src/sample_point_cloud.cpp:175-182, in the cloud's precision like the reference's casts (:346-354)
        g.size[a] = (T)size[a];
        g.min_bound[a] = (T)min_bound[a];
        if (g.size[a] <= (T)0) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size is negative");
        if (g.size[a] * (T)2147483647 < (T)max_bound[a] - g.min_bound[a]) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size is too small");
    }
    PCU_ON_DEVICE(ws);
    unsigned slots = 64;
    while ((long long)slots < 2 * n) slots <<= 1;     // load factor <= 1/2
    int *table, *slot_of; VoxelAcc* acc; double* attr_sum; unsigned char* keep; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        table = cv.take<int>(slots);
        acc = cv.take<VoxelAcc>(slots);
        slot_of = cv.take<int>((size_t)n);
        attr_sum = cv.take<double>((size_t)slots * (attr_cols > 0 ? attr_cols : 0) + 1);
        keep = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_LAUNCH(voxel_init_kernel, blocks_for(slots), kThreads, stream, table, acc, slots);
    if (attr_cols > 0) PCU_CUDA(cudaMemsetAsync(attr_sum, 0, sizeof(double) * (size_t)slots * attr_cols, stream));
    PCU_LAUNCH((voxel_insert_kernel<T, A>), blocks_for(n), kThreads, stream, pts, n, g, table, slots, acc, slot_of, attr, attr_cols, attr_sum);
    PCU_LAUNCH(voxel_flag_kernel, blocks_for(n), kThreads, stream, slot_of, acc, n, min_points, keep);
    PCU_TRY(enqueue_keep_offsets(keep, n, counts, out_rows, stream));
    PCU_LAUNCH((voxel_emit_kernel<T, A>), blocks_for(n), kThreads, stream, keep, n, counts, slot_of, acc, attr_sum, attr_cols, out_pts, out_attr, out_counts);
    return PCU_B200_OK;
}

template <typename T>
int voxel_downsample_dispatch(pcu_b200_workspace* ws, const T* pts, long long n, const void* attr, int attr_cols, int attr_is_f64,
                              const double size[3], const double min_bound[3], const double max_bound[3], int min_points, T* out_pts,
                              void* out_attr, int* out_counts, long long* out_rows, cudaStream_t stream) {
    if (attr_is_f64)
        return voxel_downsample_device<T, double>(ws, pts, n, (const double*)attr, attr_cols, size, min_bound, max_bound, min_points,
                                                  out_pts, (double*)out_attr, out_counts, out_rows, stream);
    return voxel_downsample_device<T, float>(ws, pts, n, (const float*)attr, attr_cols, size, min_bound, max_bound, min_points, out_pts,
                                             (float*)out_attr, out_counts, out_rows, stream);
}

// ---- dense pairwise distances, Sinkhorn (SURVEY.md 8f N4) ------------------------------------------------
// gridDim.y and gridDim.z stop at 65535: the dense kernels take rows and batches there, so larger problems are
// launched in chunks of that many, the pointers offset to each chunk's first row or batch.
constexpr long long kMaxGridYZ = 65535;

template <typename T>
int pairwise_device(pcu_b200_workspace* ws, const T* a, const T* b, long long nb, long long n, long long m, int d, int norm_kind,
                    double p, T* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (nb <= 0 || n <= 0 || m <= 0 || d <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid shape: a and b must be [m, n, d] or [n, d] with positive sizes");
    if (norm_kind < kNorm2 || norm_kind > kNormP) return fail(PCU_B200_INVALID_ARGUMENT, "unknown norm");
    PCU_ON_DEVICE(ws);
    for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ)
        for (long long i0 = 0; i0 < n; i0 += kMaxGridYZ) {
            const dim3 grid(blocks_for(m), (unsigned)std::min(n - i0, kMaxGridYZ), (unsigned)std::min(nb - b0, kMaxGridYZ));
            PCU_LAUNCH((pairwise_kernel<T>), grid, kThreads, stream, a + (b0 * n + i0) * d, b + b0 * m * d, n, m, d, norm_kind, p,
                       out + (b0 * n + i0) * m);
        }
    return PCU_B200_OK;
}

// a: (nb, n) weights, b: (nb, m) weights, M: (nb, n, m) costs -> P: (nb, n, m); out_cost (nb) fp64 = sum P * M, or null;
// out_iters: device int32, iterations run (or null).  No host synchronisation: the iteration's three kernels are
// enqueued max_iters times and return at once after the convergence test has passed on the device.
template <typename T>
int sinkhorn_device(pcu_b200_workspace* ws, const T* a, const T* b, const T* M, long long nb, long long n, long long m, double eps,
                    int max_iters, double stop_thresh, T* out_P, double* out_cost, int* out_iters, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || !M || !out_P) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (nb <= 0 || n <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Got unexpected shape for M, should be [nb, m, n] with positive sizes");
    if (max_iters < 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_iters must be >= 0");
    PCU_ON_DEVICE(ws);
    T *u, *v; double *eu, *ev; int* flags;
    auto carve = [&](Carver& cv) {
        u = cv.take<T>((size_t)nb * n);
        v = cv.take<T>((size_t)nb * m);
        eu = cv.take<double>((size_t)nb);
        ev = cv.take<double>((size_t)nb);
        flags = cv.take<int>(2);   // [0] done, [1] iterations
    };
    const size_t bytes = carve_at(nullptr, carve);
    PCU_TRY(carve_scratch(ws, kArena, stream, carve));
    PCU_CUDA(cudaMemsetAsync(u, 0, bytes, stream));   // u = v = 0 (:101-102), accumulators, flags
    if (out_cost) PCU_CUDA(cudaMemsetAsync(out_cost, 0, sizeof(double) * nb, stream));
    const T e = (T)eps;
    for (int it = 0; it < max_iters; ++it) {
        for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ) {
            const unsigned nbc = (unsigned)std::min(nb - b0, kMaxGridYZ);
            PCU_LAUNCH((sinkhorn_half_kernel<T, false>), dim3((unsigned)n, nbc), kThreads, stream, M + b0 * n * m, a + b0 * n, v + b0 * m,
                       u + b0 * n, n, m, e, eu + b0, flags);
        }
        for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ) {
            const unsigned nbc = (unsigned)std::min(nb - b0, kMaxGridYZ);
            PCU_LAUNCH((sinkhorn_half_kernel<T, true>), dim3((unsigned)((m + 31) / 32), nbc), kThreads, stream, M + b0 * n * m, b + b0 * m,
                       u + b0 * n, v + b0 * m, m, n, e, ev + b0, flags);
        }
        PCU_LAUNCH(sinkhorn_check_kernel, 1, kThreads, stream, eu, ev, nb, stop_thresh, flags, flags + 1);
    }
    for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ)
        for (long long i0 = 0; i0 < n; i0 += kMaxGridYZ) {
            const dim3 grid(blocks_for(m), (unsigned)std::min(n - i0, kMaxGridYZ), (unsigned)std::min(nb - b0, kMaxGridYZ));
            PCU_LAUNCH((sinkhorn_plan_kernel<T>), grid, kThreads, stream, M + (b0 * n + i0) * m, u + b0 * n + i0, v + b0 * m, n, m, e,
                       out_P + (b0 * n + i0) * m, out_cost ? out_cost + b0 : nullptr);
        }
    if (out_iters) PCU_CUDA(cudaMemcpyAsync(out_iters, flags + 1, sizeof(int), cudaMemcpyDeviceToDevice, stream));
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

}  // namespace

// =================================================================================================
extern "C" {

int pcu_b200_abi_version(void) { return PCU_B200_ABI_VERSION; }
const char* pcu_b200_last_error(void) { return g_error.c_str(); }
int64_t pcu_b200_launch_count(void) { return g_launches.load(); }

int pcu_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    int usable = 0;
    for (int d = 0; d < n; ++d)
        if (runs_this_build(d)) ++usable;
    return usable;
}

// Which device a call that names none should run on (the reference's interface has no device argument):
// PCU_B200_DEVICE if set; else the CUDA runtime's current device when the caller has chosen one other than 0
// (torch.cuda.set_device / torch.cuda.device(...) in this thread); else LOCAL_RANK when a launcher such as
// torchrun set it and that many devices are visible; else device 0.
int pcu_b200_current_device(void) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) { cudaGetLastError(); return 0; }
    auto from_env = [&](const char* name) {
        const char* v = std::getenv(name);
        if (!v || !*v) return -1;
        char* end = nullptr;
        const long d = std::strtol(v, &end, 10);
        return (end && *end == '\0' && d >= 0 && d < count) ? (int)d : -1;
    };
    int d = from_env("PCU_B200_DEVICE");
    if (d >= 0) return d;
    int cur = 0;
    if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); cur = 0; }
    if (cur > 0) return cur;
    d = from_env("LOCAL_RANK");
    return d >= 0 ? d : 0;
}

int pcu_b200_workspace_device(const pcu_b200_workspace* ws) { return ws ? ws->device : -1; }

int pcu_b200_host_alloc(void** out_ptr, int64_t bytes) {
    if (!out_ptr || bytes <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "bad argument");
    *out_ptr = nullptr;
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) { cudaGetLastError(); device = 0; }
    cudaError_t e;
    {
        NearDevice near(device);   // pages on the NUMA node of the calling thread's current GPU (staging.h)
        e = cudaHostAlloc(out_ptr, (size_t)bytes, cudaHostAllocPortable);
        // touch the pages while bound: placement is decided at first touch if the driver left any of it lazy
        if (e == cudaSuccess) for (size_t off = 0; off < (size_t)bytes; off += 4096) static_cast<volatile char*>(*out_ptr)[off] = 0;
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        *out_ptr = nullptr;
        return fail(PCU_B200_OUT_OF_MEMORY, "cudaHostAlloc of %lld bytes failed: %s", (long long)bytes, cudaGetErrorString(e));
    }
    return PCU_B200_OK;
}

int pcu_b200_host_free(void* ptr) {
    if (!ptr) return PCU_B200_OK;
    cudaError_t e = cudaFreeHost(ptr);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(PCU_B200_CUDA_ERROR, "cudaFreeHost failed: %s", cudaGetErrorString(e)); }
    return PCU_B200_OK;
}

int pcu_b200_workspace_create(int device, pcu_b200_workspace** out_ws) {
    if (!out_ws) return fail(PCU_B200_INVALID_ARGUMENT, "null out_ws");
    *out_ws = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(PCU_B200_NO_DEVICE, "no CUDA device visible: this library has no CPU fallback");
    }
    if (device < 0 || device >= n) return fail(PCU_B200_INVALID_ARGUMENT, "device %d out of range (0..%d)", device, n - 1);
    int major = 0, minor = 0, sms = 0;
    PCU_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    PCU_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    PCU_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    if (!runs_this_build(device))
        return fail(PCU_B200_NO_DEVICE, "device %d has compute capability %d.%d; this build only carries sm_90a code",
                    device, major, minor);
    pcu_b200_workspace* ws = new (std::nothrow) pcu_b200_workspace();
    if (!ws) return fail(PCU_B200_OUT_OF_MEMORY, "out of host memory");
    ws->device = device;
    ws->sm_count = sms;
    DeviceGuard guard(device);
    if (guard.status != cudaSuccess) { delete ws; return fail(PCU_B200_CUDA_ERROR, "cudaSetDevice(%d): %s", device, cudaGetErrorString(guard.status)); }
    cudaError_t e = cudaStreamCreateWithFlags(&ws->own_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ws->copy_stream, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = cudaEventCreateWithFlags(&ws->arrived[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&ws->host_slot, 4096, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        pcu_b200_workspace_destroy(ws);
        return fail(PCU_B200_CUDA_ERROR, "workspace streams / events / pinned slot: %s", cudaGetErrorString(e));
    }
    void* hint = nullptr;
    if (cudaHostAlloc(&hint, 16 * sizeof(unsigned), cudaHostAllocMapped) == cudaSuccess) {
        std::memset(hint, 0, 16 * sizeof(unsigned));
        void* dev_view = nullptr;
        if (cudaHostGetDevicePointer(&dev_view, hint, 0) == cudaSuccess) {
            ws->hint_host = (volatile unsigned*)hint;
            ws->hint_dev = (unsigned*)dev_view;
        } else {
            cudaGetLastError();
            cudaFreeHost(hint);
        }
    } else {
        cudaGetLastError();   // no feedback then; everything else works
    }
    *out_ws = ws;
    return PCU_B200_OK;
}

int pcu_b200_workspace_destroy(pcu_b200_workspace* ws) {
    if (!ws) return PCU_B200_OK;
    DeviceGuard guard(ws->device);
    cudaDeviceSynchronize();
    for (auto* b : ws->block) if (b) cudaFree(b);
    if (ws->handover) cudaEventDestroy(ws->handover);
    if (ws->hint_host) cudaFreeHost((void*)ws->hint_host);
    if (ws->own_stream) cudaStreamDestroy(ws->own_stream);
    if (ws->copy_stream) cudaStreamDestroy(ws->copy_stream);
    for (auto& e : ws->arrived) if (e) cudaEventDestroy(e);
    if (ws->host_slot) cudaFreeHost(ws->host_slot);
    for (auto& e : ws->marks) if (e) cudaEventDestroy(e);
    delete ws->stager;            // (the device is idle: nothing is in flight out of the ring)
    delete ws;
    return PCU_B200_OK;
}

int64_t pcu_b200_workspace_bytes(const pcu_b200_workspace* ws) {
    if (!ws) return 0;
    size_t bytes = 0;
    for (size_t b : ws->block_bytes) bytes += b;
    return (int64_t)bytes;
}

int pcu_b200_workspace_set_profiling(pcu_b200_workspace* ws, int enabled) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_ON_DEVICE(ws);
    if (enabled && !ws->marks[0])
        for (auto& e : ws->marks) PCU_CUDA(cudaEventCreate(&e));
    ws->profiling = enabled != 0;
    ws->marks_used = 0;
    return PCU_B200_OK;
}

int pcu_b200_workspace_last_profile(pcu_b200_workspace* ws, float* out_ms, int capacity) {
    if (!ws || !out_ms) return -1;
    if (!ws->profiling || ws->marks_used < 9) return 0;
    cudaEvent_t last = ws->host_marks ? ws->marks[10] : ws->marks[8];
    if (cudaEventSynchronize(last) != cudaSuccess) { cudaGetLastError(); return -1; }
    int n = 0;
    for (; n < 8 && n < capacity; ++n) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ws->marks[n], ws->marks[n + 1]) != cudaSuccess) { cudaGetLastError(); return -1; }
        out_ms[n] = ms;
    }
    if (ws->host_marks && capacity >= 10) {   // host entry points: the copies either side of the device call
        float h2d = 0.f, d2h = 0.f;
        if (cudaEventElapsedTime(&h2d, ws->marks[9], ws->marks[0]) != cudaSuccess ||
            cudaEventElapsedTime(&d2h, ws->marks[8], ws->marks[10]) != cudaSuccess) { cudaGetLastError(); return -1; }
        out_ms[8] = h2d; out_ms[9] = d2h;
        n = 10;
    }
    return n;
}

const char* pcu_b200_profile_stage_name(int stage) {
    static const char* names[] = {PCU_STAGE_NAMES};
    return stage >= 0 && stage < 10 ? names[stage] : "";
}

int pcu_b200_workspace_grid_refinement(const pcu_b200_workspace* ws, float out_mult[2]) {
    if (!ws || !out_mult) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    out_mult[0] = ws->cell_mult[0];
    out_mult[1] = ws->cell_mult[1];
    return PCU_B200_OK;
}

int pcu_b200_workspace_set_options(pcu_b200_workspace* ws, const pcu_b200_options* opts) {
    if (!ws || !opts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (opts->max_points_per_leaf < 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_points_per_leaf must be >= 0");
    if (opts->cell_occupancy < 0.f) return fail(PCU_B200_INVALID_ARGUMENT, "cell_occupancy must be >= 0");
    if (opts->disable_tie_replay < 0 || opts->disable_tie_replay > 3)
        return fail(PCU_B200_INVALID_ARGUMENT, "disable_tie_replay must be 0 .. 3");
    if (opts->binning < 0 || opts->binning > 3) return fail(PCU_B200_INVALID_ARGUMENT, "binning must be 0, 1, 2 or 3");
    if (opts->host_staging < 0 || opts->host_staging > 2) return fail(PCU_B200_INVALID_ARGUMENT, "host_staging must be 0, 1 or 2");
    ws->opts = *opts;
    return PCU_B200_OK;
}

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

int pcu_b200_voxel_downsample_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, float* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream) {
    return voxel_downsample_dispatch<float>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                            min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows, (cudaStream_t)stream);
}
int pcu_b200_voxel_downsample_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, double* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream) {
    return voxel_downsample_dispatch<double>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                             min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows, (cudaStream_t)stream);
}

int pcu_b200_pairwise_distances_f32(pcu_b200_workspace* ws, const float* a, const float* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, float* out, void* stream) {
    return pairwise_device<float>(ws, a, b, nb, n, m, d, norm_kind, p, out, (cudaStream_t)stream);
}
int pcu_b200_pairwise_distances_f64(pcu_b200_workspace* ws, const double* a, const double* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, double* out, void* stream) {
    return pairwise_device<double>(ws, a, b, nb, n, m, d, norm_kind, p, out, (cudaStream_t)stream);
}
int pcu_b200_sinkhorn_f32(pcu_b200_workspace* ws, const float* a, const float* b, const float* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, float* out_P, double* out_cost, int32_t* out_iters, void* stream) {
    return sinkhorn_device<float>(ws, a, b, M, nb, n, m, eps, max_iters, stop_thresh, out_P, out_cost, out_iters, (cudaStream_t)stream);
}
int pcu_b200_sinkhorn_f64(pcu_b200_workspace* ws, const double* a, const double* b, const double* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, double* out_P, double* out_cost, int32_t* out_iters, void* stream) {
    return sinkhorn_device<double>(ws, a, b, M, nb, n, m, eps, max_iters, stop_thresh, out_P, out_cost, out_iters, (cudaStream_t)stream);
}

int pcu_b200_morton_encode_i32(pcu_b200_workspace* ws, const int32_t* pts, int64_t n, uint64_t* out_codes, void* stream) {
    return morton_encode_device<int32_t>(ws, pts, n, (unsigned long long*)out_codes, (cudaStream_t)stream);
}
int pcu_b200_morton_encode_i64(pcu_b200_workspace* ws, const int64_t* pts, int64_t n, uint64_t* out_codes, void* stream) {
    return morton_encode_device<long long>(ws, (const long long*)pts, n, (unsigned long long*)out_codes, (cudaStream_t)stream);
}
int pcu_b200_morton_decode(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, int32_t* out_pts, void* stream) {
    return morton_decode_device(ws, (const unsigned long long*)codes, n, out_pts, (cudaStream_t)stream);
}
int pcu_b200_morton_add(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream) {
    return morton_addsub_device(ws, (const unsigned long long*)a, (const unsigned long long*)b, n, 0, (unsigned long long*)out, (cudaStream_t)stream);
}
int pcu_b200_morton_subtract(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream) {
    return morton_addsub_device(ws, (const unsigned long long*)a, (const unsigned long long*)b, n, 1, (unsigned long long*)out, (cudaStream_t)stream);
}
int pcu_b200_morton_knn(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, const uint64_t* qcodes, int64_t m, int k,
                        int sort_dist, int64_t* out_idx, void* stream) {
    return morton_knn_device(ws, (const unsigned long long*)codes, n, (const unsigned long long*)qcodes, m, k, sort_dist,
                             (long long*)out_idx, (cudaStream_t)stream);
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

int pcu_b200_mesh_area_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                           pcu_b200_mesh_area* out_area, void* stream) {
    return mesh_area_device<float>(ws, v, nv, f, nf, f_kind, (MeshArea*)out_area, (cudaStream_t)stream);
}
int pcu_b200_mesh_area_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                           pcu_b200_mesh_area* out_area, void* stream) {
    return mesh_area_device<double>(ws, v, nv, f, nf, f_kind, (MeshArea*)out_area, (cudaStream_t)stream);
}
int pcu_b200_sample_mesh_random_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                    int64_t num_samples, uint32_t seed, void* out_fidx, float* out_bc, pcu_b200_mesh_area* out_area,
                                    void* stream) {
    return sample_mesh_random_device<float>(ws, v, nv, f, nf, f_kind, num_samples, seed, out_fidx, out_bc, (MeshArea*)out_area,
                                            (cudaStream_t)stream);
}
int pcu_b200_sample_mesh_random_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                    int64_t num_samples, uint32_t seed, void* out_fidx, double* out_bc, pcu_b200_mesh_area* out_area,
                                    void* stream) {
    return sample_mesh_random_device<double>(ws, v, nv, f, nf, f_kind, num_samples, seed, out_fidx, out_bc, (MeshArea*)out_area,
                                             (cudaStream_t)stream);
}
int pcu_b200_sample_mesh_poisson_disk_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                          double radius, int64_t n_dense, uint32_t seed, void* out_fidx, float* out_bc,
                                          int64_t* out_count, void* stream) {
    return sample_mesh_poisson_disk_device<float>(ws, v, nv, f, nf, f_kind, radius, n_dense, seed, out_fidx, out_bc,
                                                  (long long*)out_count, (cudaStream_t)stream);
}
int pcu_b200_sample_mesh_poisson_disk_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                          double radius, int64_t n_dense, uint32_t seed, void* out_fidx, double* out_bc,
                                          int64_t* out_count, void* stream) {
    return sample_mesh_poisson_disk_device<double>(ws, v, nv, f, nf, f_kind, radius, n_dense, seed, out_fidx, out_bc,
                                                   (long long*)out_count, (cudaStream_t)stream);
}
int pcu_b200_interpolate_barycentric_f32(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, const void* fi, int64_t n,
                                         int fi_kind, const float* bc, const float* attribute, int64_t nv, int64_t dim, float* out,
                                         uint64_t* out_bad, void* stream) {
    return interpolate_device<float>(ws, f, nf, f_kind, fi, n, fi_kind, bc, 0, attribute, 0, nv, dim, out,
                                     (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_interpolate_barycentric_f64(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, const void* fi, int64_t n,
                                         int fi_kind, const void* bc, int bc_is_f64, const void* attribute, int attribute_is_f64,
                                         int64_t nv, int64_t dim, double* out, uint64_t* out_bad, void* stream) {
    return interpolate_device<double>(ws, f, nf, f_kind, fi, n, fi_kind, bc, bc_is_f64, attribute, attribute_is_f64, nv, dim, out,
                                      (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_closest_points_on_mesh_f32(pcu_b200_workspace* ws, const float* p, int64_t np, const float* v, int64_t nv, const void* f,
                                        int64_t nf, int f_kind, float* out_d, void* out_fidx, float* out_bc, uint64_t* out_bad,
                                        void* stream) {
    return closest_points_device<float>(ws, p, np, v, nv, f, nf, f_kind, out_d, out_fidx, out_bc, (unsigned long long*)out_bad,
                                        (cudaStream_t)stream);
}
int pcu_b200_closest_points_on_mesh_f64(pcu_b200_workspace* ws, const double* p, int64_t np, const double* v, int64_t nv, const void* f,
                                        int64_t nf, int f_kind, double* out_d, void* out_fidx, double* out_bc, uint64_t* out_bad,
                                        void* stream) {
    return closest_points_device<double>(ws, p, np, v, nv, f, nf, f_kind, out_d, out_fidx, out_bc, (unsigned long long*)out_bad,
                                         (cudaStream_t)stream);
}

int pcu_b200_fast_winding_number_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                     const float* q, int64_t nq, double accuracy_scale, float* out_w, uint64_t* out_bad, void* stream) {
    return winding_number_device<float>(ws, v, nv, f, nf, f_kind, q, nq, accuracy_scale, out_w, (unsigned long long*)out_bad,
                                        (cudaStream_t)stream);
}
int pcu_b200_fast_winding_number_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                     const double* q, int64_t nq, double accuracy_scale, double* out_w, uint64_t* out_bad, void* stream) {
    return winding_number_device<double>(ws, v, nv, f, nf, f_kind, q, nq, accuracy_scale, out_w, (unsigned long long*)out_bad,
                                         (cudaStream_t)stream);
}
int pcu_b200_point_cloud_fast_winding_number_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* a, int64_t np,
                                                 const float* q, int64_t nq, double accuracy_scale, float* out_w, void* stream) {
    return point_winding_number_device<float>(ws, p, n, a, np, q, nq, accuracy_scale, out_w, (cudaStream_t)stream);
}
int pcu_b200_point_cloud_fast_winding_number_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* a, int64_t np,
                                                 const double* q, int64_t nq, double accuracy_scale, double* out_w, void* stream) {
    return point_winding_number_device<double>(ws, p, n, a, np, q, nq, accuracy_scale, out_w, (cudaStream_t)stream);
}
int pcu_b200_signed_distance_to_mesh_f32(pcu_b200_workspace* ws, const float* p, int64_t np, const float* v, int64_t nv, const void* f,
                                         int64_t nf, int f_kind, float lower_bound, float upper_bound, float* out_s, int32_t* out_fidx,
                                         float* out_bc, uint64_t* out_bad, void* stream) {
    return signed_distance_device<float>(ws, p, np, v, nv, f, nf, f_kind, lower_bound, upper_bound, out_s, out_fidx, out_bc,
                                         (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_signed_distance_to_mesh_f64(pcu_b200_workspace* ws, const double* p, int64_t np, const double* v, int64_t nv, const void* f,
                                         int64_t nf, int f_kind, float lower_bound, float upper_bound, double* out_s, int32_t* out_fidx,
                                         double* out_bc, uint64_t* out_bad, void* stream) {
    return signed_distance_device<double>(ws, p, np, v, nv, f, nf, f_kind, lower_bound, upper_bound, out_s, out_fidx, out_bc,
                                          (unsigned long long*)out_bad, (cudaStream_t)stream);
}

int pcu_b200_ray_mesh_intersection_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                       const float* o, int o_stride, const float* d, int64_t n, float near, float far, void* out_fidx,
                                       float* out_bc, float* out_t, uint64_t* out_bad, void* stream) {
    return ray_mesh_device<float>(ws, v, nv, f, nf, f_kind, o, o_stride, d, n, near, far, out_fidx, out_bc, out_t,
                                  (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_ray_mesh_intersection_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                       const double* o, int o_stride, const double* d, int64_t n, float near, float far, void* out_fidx,
                                       double* out_bc, double* out_t, uint64_t* out_bad, void* stream) {
    return ray_mesh_device<double>(ws, v, nv, f, nf, f_kind, o, o_stride, d, n, near, far, out_fidx, out_bc, out_t,
                                   (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_mesh_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                              pcu_b200_mesh** out_mesh, uint64_t* out_bad, void* stream) {
    return mesh_prepare_device<float>(ws, v, nv, f, nf, f_kind, out_mesh, (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_mesh_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                              pcu_b200_mesh** out_mesh, uint64_t* out_bad, void* stream) {
    return mesh_prepare_device<double>(ws, v, nv, f, nf, f_kind, out_mesh, (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_mesh_destroy(pcu_b200_mesh* mesh) {
    if (!mesh) return PCU_B200_OK;
    DeviceGuard guard(mesh->device);
    cudaDeviceSynchronize();          // calls that use the mesh may still be queued
    if (mesh->block) cudaFree(mesh->block);
    delete mesh;
    return PCU_B200_OK;
}
int64_t pcu_b200_mesh_size(const pcu_b200_mesh* mesh) { return mesh ? mesh->nf : 0; }
int pcu_b200_ray_mesh_intersection_prepared_f32(pcu_b200_workspace* ws, const pcu_b200_mesh* mesh, const float* o, int o_stride,
                                                const float* d, int64_t n, float near, float far, int32_t* out_fidx, float* out_bc,
                                                float* out_t, void* stream) {
    return ray_mesh_prepared_device<float>(ws, mesh, o, o_stride, d, n, near, far, out_fidx, out_bc, out_t, (cudaStream_t)stream);
}
int pcu_b200_ray_mesh_intersection_prepared_f64(pcu_b200_workspace* ws, const pcu_b200_mesh* mesh, const double* o, int o_stride,
                                                const double* d, int64_t n, float near, float far, int32_t* out_fidx, double* out_bc,
                                                double* out_t, void* stream) {
    return ray_mesh_prepared_device<double>(ws, mesh, o, o_stride, d, n, near, far, out_fidx, out_bc, out_t, (cudaStream_t)stream);
}

int pcu_b200_ray_surfel_intersection_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                         const float* o, int o_stride, const float* d, int64_t nr, float near, float far, int32_t* out_pid,
                                         float* out_t, void* stream) {
    return ray_surfel_device<float>(ws, p, n, r, np, subdivs, o, o_stride, d, nr, near, far, out_pid, out_t, (cudaStream_t)stream);
}
int pcu_b200_ray_surfel_intersection_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np, int subdivs,
                                         const double* o, int o_stride, const double* d, int64_t nr, float near, float far, int32_t* out_pid,
                                         double* out_t, void* stream) {
    return ray_surfel_device<double>(ws, p, n, r, np, subdivs, o, o_stride, d, nr, near, far, out_pid, out_t, (cudaStream_t)stream);
}
int pcu_b200_surfel_prepare_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                pcu_b200_mesh** out_surfels, void* stream) {
    return surfel_prepare_device<float>(ws, p, n, r, np, subdivs, out_surfels, (cudaStream_t)stream);
}
int pcu_b200_surfel_prepare_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np, int subdivs,
                                pcu_b200_mesh** out_surfels, void* stream) {
    return surfel_prepare_device<double>(ws, p, n, r, np, subdivs, out_surfels, (cudaStream_t)stream);
}
int pcu_b200_ray_surfel_intersection_prepared_f32(pcu_b200_workspace* ws, const pcu_b200_mesh* surfels, const float* o, int o_stride,
                                                  const float* d, int64_t nr, float near, float far, int32_t* out_pid, float* out_t,
                                                  void* stream) {
    return ray_surfel_prepared_device<float>(ws, surfels, o, o_stride, d, nr, near, far, out_pid, out_t, (cudaStream_t)stream);
}
int pcu_b200_ray_surfel_intersection_prepared_f64(pcu_b200_workspace* ws, const pcu_b200_mesh* surfels, const double* o, int o_stride,
                                                  const double* d, int64_t nr, float near, float far, int32_t* out_pid, double* out_t,
                                                  void* stream) {
    return ray_surfel_prepared_device<double>(ws, surfels, o, o_stride, d, nr, near, far, out_pid, out_t, (cudaStream_t)stream);
}
int pcu_b200_pointcloud_surfel_geometry_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                            float* out_v, int32_t* out_f, void* stream) {
    return surfel_geometry_device<float>(ws, p, n, r, np, subdivs, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_pointcloud_surfel_geometry_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np,
                                            int subdivs, double* out_v, int32_t* out_f, void* stream) {
    return surfel_geometry_device<double>(ws, p, n, r, np, subdivs, out_v, out_f, (cudaStream_t)stream);
}

int pcu_b200_marching_cubes_prepare_f32(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const float* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream) {
    return marching_cubes_prepare_device<float>(ws, scalars, scalars_f64, coords, n, cube_idx, m, idx_kind, isovalue, out_mc,
                                                (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_prepare_f64(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const double* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream) {
    return marching_cubes_prepare_device<double>(ws, scalars, scalars_f64, coords, n, cube_idx, m, idx_kind, isovalue, out_mc,
                                                 (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_emit(pcu_b200_workspace* ws, const pcu_b200_marching_cubes* mc, void* out_v, void* out_f, void* stream) {
    return marching_cubes_emit_device(ws, mc, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_destroy(pcu_b200_marching_cubes* mc) {
    if (!mc) return PCU_B200_OK;
    DeviceGuard guard(mc->device);
    delete mc;
    return PCU_B200_OK;
}
int pcu_b200_sparse_voxel_grid_boundary(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, int64_t* out_idx,
                                        int64_t* out_counts, void* stream) {
    return sparse_voxel_grid_boundary_device(ws, grid, n, idx_kind, (long long*)out_idx, (long long*)out_counts, (cudaStream_t)stream);
}

int pcu_b200_sparse_grid_from_points_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream) {
    return svg_points_prepare<float>(ws, points, n, voxel_size, origin, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_from_points_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream) {
    return svg_points_prepare<double>(ws, points, n, voxel_size, origin, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_dilate_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, pcu_b200_sparse_grid** out_grid,
                                        int64_t out_counts[2], void* stream) {
    return svg_dilate_prepare(ws, grid, n, idx_kind, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_hex_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, const double voxel_size[3],
                                     const double origin[3], int vertices_f64, pcu_b200_sparse_grid** out_grid, int64_t out_counts[2],
                                     void* stream) {
    return svg_hex_prepare(ws, grid, n, idx_kind, voxel_size, origin, vertices_f64, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_emit(pcu_b200_workspace* ws, const pcu_b200_sparse_grid* sg, void* out_rows, int64_t* out_index, void* stream) {
    return svg_emit(ws, sg, out_rows, out_index, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_destroy(pcu_b200_sparse_grid* sg) {
    if (!sg) return PCU_B200_OK;
    DeviceGuard guard(sg->device);
    delete sg;
    return PCU_B200_OK;
}
int pcu_b200_sparse_grid_erode(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, void* out_grid, int64_t* out_counts,
                               void* stream) {
    return svg_erode(ws, grid, n, idx_kind, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_voxel_grid_geometry(pcu_b200_workspace* ws, const void* ijk, int64_t n, int idx_kind, const double voxel_size[3],
                                 const double voxel_origin[3], double gap_fraction, float* out_v, int32_t* out_f, void* stream) {
    return voxel_grid_geometry_device(ws, ijk, n, idx_kind, voxel_size, voxel_origin, gap_fraction, out_v, out_f, (cudaStream_t)stream);
}

int pcu_b200_voxelize_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream) {
    return voxelize_prepare_device<float>(ws, v, nv, f, nf, f_kind, voxel_size, voxel_origin, out_vx, (long long*)out_counts,
                                          (cudaStream_t)stream);
}
int pcu_b200_voxelize_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream) {
    return voxelize_prepare_device<double>(ws, v, nv, f, nf, f_kind, voxel_size, voxel_origin, out_vx, (long long*)out_counts,
                                           (cudaStream_t)stream);
}
int pcu_b200_voxelize_emit(pcu_b200_workspace* ws, const pcu_b200_voxelize* vx, int32_t* out_ijk, void* stream) {
    return voxelize_emit_device(ws, vx, out_ijk, (cudaStream_t)stream);
}
int pcu_b200_voxelize_destroy(pcu_b200_voxelize* vx) {
    if (!vx) return PCU_B200_OK;
    DeviceGuard guard(vx->device);
    delete vx;
    return PCU_B200_OK;
}
int pcu_b200_flood_fill_3d(pcu_b200_workspace* ws, const void* grid, int grid_kind, int64_t w, int64_t h, int64_t d, int64_t seed_x,
                           int64_t seed_y, int64_t seed_z, double fill_value, void* out, void* stream) {
    return flood_fill_3d_device(ws, grid, grid_kind, w, h, d, seed_x, seed_y, seed_z, fill_value, out, (cudaStream_t)stream);
}

int pcu_b200_make_mesh_watertight_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream) {
    return make_mesh_watertight_prepare_device<float>(ws, v, nv, f, nf, f_kind, resolution, out_wt, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream) {
    return make_mesh_watertight_prepare_device<double>(ws, v, nv, f, nf, f_kind, resolution, out_wt, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_emit(pcu_b200_workspace* ws, const pcu_b200_watertight* wt, void* out_v, void* out_f, void* stream) {
    return make_mesh_watertight_emit_device(ws, wt, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_destroy(pcu_b200_watertight* wt) {
    if (!wt) return PCU_B200_OK;
    DeviceGuard guard(wt->device);
    delete wt;
    return PCU_B200_OK;
}

int pcu_b200_connected_components_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_cols, int f_kind,
                                           pcu_b200_components** out_cc, int64_t out_counts[2], void* stream) {
    return connected_components_prepare_device(ws, f, nf, f_cols, f_kind, out_cc, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_connected_components_emit(pcu_b200_workspace* ws, const pcu_b200_components* cc, void* out_cv, void* out_nv, void* out_cf,
                                        void* out_nf, void* stream) {
    return connected_components_emit_device(ws, cc, out_cv, out_nv, out_cf, out_nf, (cudaStream_t)stream);
}
int pcu_b200_connected_components_destroy(pcu_b200_components* cc) {
    if (!cc) return PCU_B200_OK;
    DeviceGuard guard(cc->device);
    delete cc;
    return PCU_B200_OK;
}
int pcu_b200_remove_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, float* out_v, void* out_f, int64_t out_counts[2], void* stream) {
    return remove_mesh_vertices_device<float>(ws, v, nv, f, nf, f_kind, mask, out_v, out_f, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_remove_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, double* out_v, void* out_f, int64_t out_counts[2], void* stream) {
    return remove_mesh_vertices_device<double>(ws, v, nv, f, nf, f_kind, mask, out_v, out_f, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_remove_unreferenced_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   float* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream) {
    return remove_unreferenced_device<float>(ws, v, nv, f, nf, f_kind, out_v, out_f, out_corr_v, out_corr_f, (long long*)out_count,
                                             (cudaStream_t)stream);
}
int pcu_b200_remove_unreferenced_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   double* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream) {
    return remove_unreferenced_device<double>(ws, v, nv, f, nf, f_kind, out_v, out_f, out_corr_v, out_corr_f, (long long*)out_count,
                                              (cudaStream_t)stream);
}
int pcu_b200_orient_mesh_faces(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, void* out_f, void* out_components,
                               void* stream) {
    return orient_mesh_faces_device(ws, f, nf, f_kind, out_f, out_components, (cudaStream_t)stream);
}

int pcu_b200_mesh_face_areas_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_areas,
                                 void* stream) {
    return mesh_face_device<float>(ws, v, nv, f, nf, f_kind, false, out_areas, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_areas_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_areas,
                                 void* stream) {
    return mesh_face_device<double>(ws, v, nv, f, nf, f_kind, false, out_areas, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_n,
                                   void* stream) {
    return mesh_face_device<float>(ws, v, nv, f, nf, f_kind, true, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_n,
                                   void* stream) {
    return mesh_face_device<double>(ws, v, nv, f, nf, f_kind, true, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_vertex_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     float* out_n, void* stream) {
    return vertex_normals_device<float>(ws, v, nv, f, nf, f_kind, weighting, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_vertex_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     double* out_n, void* stream) {
    return vertex_normals_device<double>(ws, v, nv, f, nf, f_kind, weighting, out_n, (cudaStream_t)stream);
}
int pcu_b200_laplacian_smooth_mesh_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, float* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream) {
    return laplacian_smooth_device<float>(ws, v, nv, f, nf, f_kind, num_iters, step_size, use_cotan_weights != 0, max_cg_iters, out_v,
                                          out_cg_iters, out_residual, (cudaStream_t)stream);
}
int pcu_b200_laplacian_smooth_mesh_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, double* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream) {
    return laplacian_smooth_device<double>(ws, v, nv, f, nf, f_kind, num_iters, step_size, use_cotan_weights != 0, max_cg_iters, out_v,
                                           out_cg_iters, out_residual, (cudaStream_t)stream);
}

int pcu_b200_deduplicate_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, float* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream) {
    return dedup_dispatch<float>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                 (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_deduplicate_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, double* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream) {
    return dedup_dispatch<double>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                  (long long*)out_counts, (cudaStream_t)stream);
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

}  // extern "C"

#include "host_entry.inl"
