// runtime.cuh -- the host runtime that every family of the library shares (internal, not installed): error state and
// launch counting, the launch macros, the workspace and its scratch blocks, the device guard, stream hand-over,
// ordered compaction, the record sort and host-to-device staging.  Each family's translation unit (nearest.cu,
// point_ops.cu, mesh_query.cu, voronoi.cu, voxels.cu, mesh_topology.cu, decimate.cu) includes it; runtime.cu defines
// what it declares, and the workspace's C entry points.
//
// A function that one translation unit calls in another lives in namespace pcu_internal and is declared here;
// everything else stays in its file's anonymous namespace.  pcu_internal has hidden visibility: the library exports
// only the C entry points, and calls between its units stay direct.
#pragma once
// Every unit sees the same standard headers ahead of the kernel headers: which math overloads the kernels resolve
// depends on them, and a kernel must compile to the same code whichever unit compiles it.
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
#include "sort.cuh"

namespace pcu {

// Compiled in nearest.cu (kdreplay.cuh); duplicate removal launches it too.
__global__ void widen_counter_kernel(const unsigned* src, long long* dst);

// Compiled in runtime.cu: head[i] = 1 where sorted one-word record i starts a run of equal keys.  Marching cubes, the
// sparse voxel grids, voxelization and the Laplacian's assembly launch it.
__global__ void mc_heads_kernel(const SortRec<unsigned long long, 1>* recs, long long ns, unsigned char* head);

// Defined in meshquery.cuh and mesh_query.cu; the declarations below only refer to them.
template <typename L> struct MeshTree;
struct RvBall;

}  // namespace pcu

namespace __attribute__((visibility("hidden"))) pcu_internal {

using namespace pcu;

extern thread_local std::string g_error;
extern std::atomic<long long> g_launches;

// Blocks of kThreads threads for one thread per row.
inline unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

int fail(int status, const char* fmt, ...);

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

}  // namespace pcu_internal

// The workspace's device scratch blocks (carve_scratch).  Every call carves the blocks it uses afresh, so buffers that
// must outlive a nested call live in a block that the nested call does not carve.
enum Scratch {
    kArena,   // the device-pointer entry points' own scratch; any nested call may re-carve it
    kIo,      // device copies of a host entry point's inputs and outputs: outlive the device call they are passed to
    kAux,     // intermediate results (normals, Poisson disk) that outlive a nested call's re-carving of the arena
    kMesh,    // the face CDF and dense samples of mesh Poisson-disk sampling, which outlive the point-cloud Poisson-disk
              // call it makes (that one re-carves the arena and aux), and the fp64 vertex normals of mesh curvatures,
              // which outlive the ball pass's binning
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
    pcu::HostStager* stager = nullptr; // pinned ring + copy threads for pageable inputs of the host entry points (created on first use)
};

// What the stream-ordered handles below share: the device and stream they were prepared on.  Deleting a handle releases
// its blocks in the order of that stream.
struct StreamHandle {
    int device = 0;
    cudaStream_t stream = nullptr;
    void release(unsigned char* block) const { if (block) cudaFreeAsync(block, stream); }
};

namespace __attribute__((visibility("hidden"))) pcu_internal {

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
inline int adopt_stream(pcu_b200_workspace* ws, cudaStream_t stream) {
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
inline int grow_block(unsigned char*& block, size_t& have, size_t bytes, cudaStream_t stream, const char* what) {
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

inline void mark(pcu_b200_workspace* ws, int index, cudaStream_t stream) {
    if (!ws->profiling) return;
    cudaEventRecord(ws->marks[index], stream);
    if (index <= 8) ws->marks_used = index + 1;
    if (index == 0) ws->host_marks = false;
    if (index == 10) ws->host_marks = true;
}

// Words of the block-count buffer that compacting n flags takes: one per block of keep_count_kernel.
inline size_t keep_count_words(long long n) { return blocks_for(n); }

// Enqueues the first two steps of compact.cuh over n flags: the kept rows of every block into `counts`
// (keep_count_words(n) words), scanned in place into the blocks' offsets, and the total into *out_count (device memory).
// The caller's emit kernel follows, with blocks_for(n) blocks of kThreads threads.
int enqueue_keep_offsets(const unsigned char* keep, long long n, unsigned* counts, long long* out_count, cudaStream_t stream);

// The kept row numbers in ascending order as int32 (keep_rows_kernel<int>) after enqueue_keep_offsets: the last step of
// the compactions of Poisson-disk downsampling and of the Voronoi cells.
int enqueue_keep_rows(const unsigned char* keep, long long n, const unsigned* counts, int* out_idx, cudaStream_t stream);

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
// are skipped.  Compiled in runtime.cu, with its kernels, for the record types in use: SortRec<unsigned, 2>,
// <unsigned long long, 2>, <unsigned long long, 1>, <unsigned, 3> and <unsigned long long, 3>.
template <typename Rec>
int radix_sort_records(const SortScratch<Rec>& s, long long n, int words, cudaStream_t stream, Rec** sorted, int key_bits = 0);

// ---- what the mesh, voxel and topology families share: count records and stream-ordered handles
// Copies a count record to the host and waits for it: one synchronisation of `stream`.
template <class R>
int read_record(const R* dev, R* host, cudaStream_t stream) {
    PCU_CUDA(cudaMemcpyAsync(host, dev, sizeof(R), cudaMemcpyDeviceToHost, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));
    return PCU_B200_OK;
}

// The failure of a call that found `bad` faces with a corner outside [0, #v).
inline int bad_corners(unsigned long long bad) {
    return fail(PCU_B200_INVALID_ARGUMENT, "Invalid face indices: %llu faces have a corner outside [0, #v)", bad);
}

// Whether face indices of this kind are 64 bits wide.
inline bool wide_index(int kind) { return kind & 1; }

// The input check of every call on a mesh (v, f): sampling, queries, rays, restricted Voronoi.
inline int mesh_check(const void* v, long long nv, const void* f, long long m, int fkind) {
    if (!v || !f || nv <= 0 || m <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements: v and f must have shape (n, 3) and (m, 3) (n, m > 0)");
    if (m > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "mesh sampling: at most 2^31 - 1 faces, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

// A handle's block, allocated in the order of `stream`; `what` names the handle's feature when that fails.
inline int alloc_block(unsigned char*& block, size_t bytes, cudaStream_t stream, const char* what) {
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

// The C destroy of a stream-ordered handle: its blocks are released in the order of its stream, on its device.
template <class H>
int destroy_handle(H* h) {
    if (!h) return PCU_B200_OK;
    DeviceGuard guard(h->device);
    delete h;
    return PCU_B200_OK;
}

// A block of device memory that lives for one call, freed in the order of its stream.
struct CallBlock {
    unsigned char* p = nullptr;
    cudaStream_t stream = nullptr;
    explicit CallBlock(cudaStream_t s) : stream(s) {}
    ~CallBlock() { reset(); }
    void reset() { if (p) cudaFreeAsync(p, stream); p = nullptr; }
};

// An emit runs on the device its handle was prepared on; `what` names the handle.
inline int check_handle_device(const pcu_b200_workspace* ws, const StreamHandle* h, const char* what) {
    if (h->device != ws->device)
        return fail(PCU_B200_INVALID_ARGUMENT, "the %s handle lives on device %d, the workspace on %d", what, h->device, ws->device);
    return PCU_B200_OK;
}

// dst (device) <- src (host), in the order of `stream`
inline int h2d(pcu_b200_workspace* ws, void* dst, const void* src, size_t bytes, cudaStream_t stream) {
    if (ws->opts.host_staging != 2 && (ws->opts.host_staging == 1 || HostStager::wants(src, bytes))) {
        if (!ws->stager) ws->stager = new (std::nothrow) HostStager();
        if (ws->stager) {
            const cudaError_t e = ws->stager->copy(dst, src, bytes, stream);
            if (e != cudaSuccess) return fail(PCU_B200_CUDA_ERROR, "staged host-to-device copy failed: %s", cudaGetErrorString(e));
            return PCU_B200_OK;
        }
    }
    PCU_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    return PCU_B200_OK;
}

// ---- what nearest.cu offers the other families: k nearest neighbours (the Voronoi cells) and Poisson-disk selection
// (mesh Poisson-disk sampling), instantiated for float and double
template <typename T>
int knn_device(pcu_b200_workspace* ws, const T* query, long long n, const T* dataset, long long m, int k, int squared,
               T* out_dist, long long* out_idx, long long* out_n_tied, cudaStream_t stream, pcu_b200_cloud* prepared = nullptr,
               bool tie_replay = true);

template <typename T>
int poisson_disk_device(pcu_b200_workspace* ws, const T* points, long long n, double radius, unsigned seed, int* out_idx,
                        long long* out_count, int* out_rounds, cudaStream_t stream);

// The ball mode of mesh_principal_curvatures (curv_ball_kernel of normals.cuh): the nv vertices binned in the arena,
// `normal` their fp64 unit normals (device memory that the arena does not hold), r > 0 the ball's radius.
template <typename T>
int curvature_ball_device(pcu_b200_workspace* ws, const T* v, long long nv, const double* normal, double r, T* out_k1, T* out_k2,
                          T* out_d1, T* out_d2, cudaStream_t stream);

// ---- what mesh_query.cu offers the other families: the fp64 closest-point tree (watertight remeshing's projection), the
// ball tree (restricted Voronoi cells) and sampled positions (the initial sample of sample_mesh_lloyd)
// Bytes of the block build_closest_tree builds the tree of m faces into.
size_t closest_tree_bytes(long long m);

// The closest-point tree of the mesh (v, nv, f, m, fkind), its build's temporaries in the arena and the tree itself in
// `block`; the count of faces with a corner out of range lands in *out_bad (device memory).
int build_closest_tree(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind,
                       unsigned long long* out_bad, unsigned char* block, MeshTree<Pt<double>>& tree, cudaStream_t stream);

// The closest points on the tree's m faces of the n points q: distances, int64 face indices and barycentric coordinates.
int enqueue_closest_points(pcu_b200_workspace* ws, const MeshTree<Pt<double>>& tree, long long m, const double* q, long long n,
                           double* out_d, long long* out_fidx, double* out_bc, cudaStream_t stream);

// The tree over the (m, 4) balls, built in the arena together with its build's temporaries.
int build_ball_tree(pcu_b200_workspace* ws, const double* balls, long long m, MeshTree<RvBall>& tree, cudaStream_t stream);

// The fp64 positions of the first n samples of sample_mesh_random at `seed` into x.  The face CDF lives in kMesh; its
// record is read (one synchronisation), and faces out of range or a zero area fail the call.
int sample_mesh_positions(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind, long long n,
                          unsigned seed, double* x, cudaStream_t stream);

}  // namespace pcu_internal
