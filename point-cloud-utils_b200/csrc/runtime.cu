// runtime.cu -- the shared host runtime (runtime.cuh): error state, launch counting, ordered compaction, the record sort
// (sort.cuh) with its kernels, the run heads of sorted one-word records, and the C entry points of versions, errors,
// devices, pinned host memory and workspaces.
#include "runtime.cuh"
#include "compact.cuh"

namespace pcu {

__global__ void __launch_bounds__(kThreads) keep_count_kernel(const unsigned char* __restrict__ keep, long long n, unsigned* __restrict__ block_count) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? keep[i] : 0u;
    const unsigned total = __syncthreads_count((int)mine);
    if (threadIdx.x == 0) block_count[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) keep_offsets_kernel(unsigned* __restrict__ block_count, long long nblocks, long long* __restrict__ out_count) {
    // nblocks = ceil(n / kThreads) with n < 2^31 rows: fits 32 bits
    const unsigned kept = block_scan_rounds<1024>(
        (unsigned)nblocks, [&](unsigned b) { return block_count[b]; }, [&](unsigned b, unsigned ex, unsigned) { block_count[b] = ex; });
    if (threadIdx.x == 0) *out_count = (long long)kept;
}

template <typename Rec>
__global__ void __launch_bounds__(kSortThreads) sort_hist_kernel(const Rec* __restrict__ in, long long n, int word, int shift,
                                                                 unsigned* __restrict__ hist, unsigned ntiles) {
    __shared__ unsigned h[kSortBins];
    h[threadIdx.x] = 0u;
    __syncthreads();
    const long long base = (long long)blockIdx.x * kSortTile;
#pragma unroll 4
    for (int r = 0; r < kSortRounds; ++r) {
        const long long i = base + r * kSortThreads + threadIdx.x;
        if (i < n) {
            const unsigned d = (unsigned)((in[i].key[word] >> shift) & 255u);
            const unsigned peers = __match_any_sync(__activemask(), d);
            if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&h[d], (unsigned)__popc(peers));
        }
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

template <typename Rec>
__global__ void __launch_bounds__(kSortThreads) sort_scatter_kernel(const Rec* __restrict__ in, Rec* __restrict__ out, long long n,
                                                                    int word, int shift, const unsigned* __restrict__ hist,
                                                                    unsigned ntiles, const unsigned* __restrict__ base,
                                                                    const int* __restrict__ constant) {
    const long long tile0 = (long long)blockIdx.x * kSortTile;
    if (*constant) {                         // the digit is the same everywhere: the pass is the identity
#pragma unroll 4
        for (int r = 0; r < kSortRounds; ++r) {
            const long long i = tile0 + r * kSortThreads + threadIdx.x;
            if (i < n) store_rec<Rec>(out + i, load_rec<Rec>(in + i));
        }
        return;
    }
    __shared__ unsigned pos[kSortWarps][kSortBins];
    for (int j = threadIdx.x; j < kSortWarps * kSortBins; j += kSortThreads) (&pos[0][0])[j] = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const long long slice0 = tile0 + (long long)w * (kSortRounds * 32);
    // 1. this warp's digit counts
    for (int r = 0; r < kSortRounds; ++r) {
        const long long i = slice0 + r * 32 + lane;
        const unsigned d = i < n ? (unsigned)((in[i].key[word] >> shift) & 255u) : 256u + (unsigned)lane;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        if (i < n && (peers & lt) == 0u) pos[w][d] += (unsigned)__popc(peers);
        __syncwarp();
    }
    __syncthreads();
    // 2. counts -> first global position of each (warp, digit)
    {
        const unsigned d = threadIdx.x;
        unsigned running = base[d] + hist[(size_t)d * ntiles + blockIdx.x];
#pragma unroll
        for (int j = 0; j < kSortWarps; ++j) {
            const unsigned c = pos[j][d];
            pos[j][d] = running;
            running += c;
        }
    }
    __syncthreads();
    // 3. the same walk again, placing the records
    for (int r = 0; r < kSortRounds; ++r) {
        const long long i = slice0 + r * 32 + lane;
        const bool live = i < n;
        Rec rec;
        unsigned d = 256u + (unsigned)lane;
        if (live) { rec = load_rec<Rec>(in + i); d = (unsigned)((rec.key[word] >> shift) & 255u); }
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        unsigned dst = 0u;
        if (live) dst = pos[w][d] + (unsigned)__popc(peers & lt);
        __syncwarp();
        if (live) {
            store_rec<Rec>(out + dst, rec);
            if ((peers & lt) == 0u) pos[w][d] += (unsigned)__popc(peers);
        }
        __syncwarp();
    }
}

// grid 256: CTA b turns hist[b][0 .. ntiles) into its exclusive prefix sums and writes the row total.  A row counts
// records, at most n < 2^31, so prefixes and total fit 32 bits.
__global__ void __launch_bounds__(kSortThreads) sort_scan_rows(unsigned* __restrict__ hist, unsigned ntiles, unsigned long long* __restrict__ total) {
    unsigned* row = hist + (size_t)blockIdx.x * ntiles;
    const unsigned all = block_scan_rounds<kSortThreads>(
        ntiles, [&](unsigned i) { return row[i]; }, [&](unsigned i, unsigned ex, unsigned) { row[i] = ex; });
    if (threadIdx.x == 0) total[blockIdx.x] = all;
}

// one CTA of 256 threads: base[bin] = records with a smaller digit; *constant = 1 when one bin holds everything
__global__ void __launch_bounds__(kSortBins) sort_scan_bins(const unsigned long long* __restrict__ total, long long n,
                                                            unsigned* __restrict__ base, int* __restrict__ constant) {
    __shared__ unsigned long long s[kSortBins];
    __shared__ int any_full;
    const unsigned long long mine = total[threadIdx.x];
    s[threadIdx.x] = mine;
    if (threadIdx.x == 0) any_full = 0;
    __syncthreads();
    if (mine == (unsigned long long)n) any_full = 1;
    unsigned long long before = 0ull;
    for (int j = 0; j < (int)threadIdx.x; ++j) before += s[j];
    base[threadIdx.x] = (unsigned)before;
    __syncthreads();
    if (threadIdx.x == 0) *constant = any_full;
}

__global__ void __launch_bounds__(kThreads) mc_heads_kernel(const SortRec<unsigned long long, 1>* __restrict__ recs, long long ns, unsigned char* __restrict__ head) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ns) return;
    head[i] = (i == 0 || recs[i].key[0] != recs[i - 1].key[0]) ? 1 : 0;
}

}  // namespace pcu

namespace __attribute__((visibility("hidden"))) pcu_internal {

thread_local std::string g_error;
std::atomic<long long> g_launches{0};

int fail(int status, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_error = buf;
    return status;
}

int enqueue_keep_offsets(const unsigned char* keep, long long n, unsigned* counts, long long* out_count, cudaStream_t stream) {
    const unsigned nblocks = blocks_for(n);
    PCU_LAUNCH(keep_count_kernel, nblocks, kThreads, stream, keep, n, counts);
    PCU_LAUNCH(keep_offsets_kernel, 1, 1024, stream, counts, (long long)nblocks, out_count);
    return PCU_B200_OK;
}

int enqueue_keep_rows(const unsigned char* keep, long long n, const unsigned* counts, int* out_idx, cudaStream_t stream) {
    PCU_LAUNCH(keep_rows_kernel<int>, blocks_for(n), kThreads, stream, keep, n, counts, out_idx);
    return PCU_B200_OK;
}

template <typename Rec>
int radix_sort_records(const SortScratch<Rec>& s, long long n, int words, cudaStream_t stream, Rec** sorted, int key_bits) {
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

// The record types in use: decimation's and orientation's half-edges (unsigned, 2), orientation's with 64-bit faces
// (unsigned long long, 2), the trees, grids and incidences (unsigned long long, 1), duplicate removal (unsigned and
// unsigned long long, 3).
#define PCU_SORT_RECORDS(K, NW) \
    template int radix_sort_records(const SortScratch<SortRec<K, NW>>&, long long, int, cudaStream_t, SortRec<K, NW>**, int);
PCU_SORT_RECORDS(unsigned, 2)
PCU_SORT_RECORDS(unsigned long long, 2)
PCU_SORT_RECORDS(unsigned long long, 1)
PCU_SORT_RECORDS(unsigned, 3)
PCU_SORT_RECORDS(unsigned long long, 3)
#undef PCU_SORT_RECORDS

}  // namespace pcu_internal

using namespace pcu_internal;

namespace {

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

}  // namespace

#define PCU_STAGE_NAMES "descriptors", "bbox+grid", "slab_count", "partition", "cell_sort", "search", "search_far", "finalize", "h2d", "d2h"

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

}  // extern "C"
