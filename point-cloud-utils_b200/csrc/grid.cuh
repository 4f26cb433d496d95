// grid.cuh -- device-side uniform-grid build (counting sort of a cloud into cells).
//
// Replaces what the reference does before it can answer a query: nanoflann's serial kd-tree build
// (external/nanoflann/nanoflann.hpp:1363-1375, divideTree :1001-1059), which the reference runs three
// times per call (SURVEY.md 3a).  Here: bounding box -> grid shape -> cell order, by one of three builds:
// the slab build (slab histogram -> partition by slab -> per-slab cell sort in shared memory), the
// cell-wise passes (per-cell histogram whose atomics hand out each point's rank in its cell ->
// exclusive scan -> scatter), or one CTA per small cloud.
// Every kernel takes an array of cloud descriptors and uses blockIdx.y as the cloud index, so the
// two clouds of a Chamfer call -- or the 2*B clouds of a batch -- are binned by the same launches.
// Nothing here synchronises with the host: the grid shape is chosen on the device.
#pragma once
#include "common.cuh"

namespace pcu {

// ---------------------------------------------------------------------------------------------
// 1. bounding box.  block_bbox folds the scalars of the chunks chunk0, chunk0 + chunk_step, ... (a chunk
//    is blockDim * kBBoxPerThread consecutive scalars of the flat (n, 3) array) and leaves
//    {lo x, lo y, lo z, hi x, hi y, hi z} in dst (written by threads 0..5; no barrier after the write).
//    The walk is flat and fully coalesced: thread t reads scalars t, t + blockDim, t + 2 blockDim, ...
//    of a chunk.  blockDim = 1 (mod 3) and the chunk length is a multiple of 3, so the k-th scalar a
//    thread reads belongs to axis (t + k) mod 3: three running boxes per thread, no index arithmetic.
template <typename T>
__device__ __forceinline__ void block_bbox(const T* __restrict__ raw, long long total, long long chunk0, long long chunk_step, T* dst) {
    using R = Real<T>;
    static_assert(kBBoxPerThread % 3 == 0, "a chunk must hold whole points per thread column");
    const long long chunk = (long long)blockDim.x * kBBoxPerThread;
    T alo[3] = {R::inf(), R::inf(), R::inf()};
    T ahi[3] = {-R::inf(), -R::inf(), -R::inf()};
    for (long long base = chunk0 * chunk + threadIdx.x; base < total; base += chunk_step * chunk) {
        T v[kBBoxPerThread];
#pragma unroll
        for (int k = 0; k < kBBoxPerThread; ++k) {
            const long long e = base + (long long)k * blockDim.x;
            v[k] = e < total ? __ldg(raw + e) : R::inf();
        }
#pragma unroll
        for (int k = 0; k < kBBoxPerThread; ++k) {
            const long long e = base + (long long)k * blockDim.x;
            alo[k % 3] = R::vmin(alo[k % 3], v[k]);
            if (e < total) ahi[k % 3] = R::vmax(ahi[k % 3], v[k]);
        }
    }
    // slot r of this thread holds axis (threadIdx.x + r) mod 3
    const int t3 = (int)(threadIdx.x % 3);
    T lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const int r = (a - t3 + 3) % 3;
        lo[a] = r == 0 ? alo[0] : (r == 1 ? alo[1] : alo[2]);
        hi[a] = r == 0 ? ahi[0] : (r == 1 ? ahi[1] : ahi[2]);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = R::vmin(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = R::vmax(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    __shared__ T s[32][6];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { s[w][a] = lo[a]; s[w][3 + a] = hi[a]; }
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        T v = s[0][threadIdx.x];
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
            v = threadIdx.x < 3 ? R::vmin(v, s[i][threadIdx.x]) : R::vmax(v, s[i][threadIdx.x]);
        dst[threadIdx.x] = v;
    }
}

//    Folds the bbox_blocks partial boxes of a cloud into `box` (shared); block-wide, ends with a barrier.
template <typename T>
__device__ __forceinline__ void fold_partial_boxes(const Cloud<T>& c, T* box) {
    using R = Real<T>;
    __shared__ T red[kThreads / 32][6];
    T lo[3] = {R::inf(), R::inf(), R::inf()}, hi[3] = {-R::inf(), -R::inf(), -R::inf()};
    for (int i = threadIdx.x; i < c.bbox_blocks; i += blockDim.x)   // possibly written in this very launch: around L1
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            lo[a] = R::vmin(lo[a], __ldcg(c.bbox_partial + i * 6 + a));
            hi[a] = R::vmax(hi[a], __ldcg(c.bbox_partial + i * 6 + 3 + a));
        }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = R::vmin(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = R::vmax(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0)
#pragma unroll
        for (int a = 0; a < 3; ++a) { red[w][a] = lo[a]; red[w][3 + a] = hi[a]; }
    __syncthreads();
    if (threadIdx.x < 6) {
        T v = red[0][threadIdx.x];
        for (int i = 1; i < kThreads / 32; ++i)
            v = threadIdx.x < 3 ? R::vmin(v, red[i][threadIdx.x]) : R::vmax(v, red[i][threadIdx.x]);
        box[threadIdx.x] = v;
    }
    __syncthreads();
}

//    partial boxes of a large cloud: grid (max bbox_blocks, nclouds).
//    kSetup (single pairs): the CTA of a cloud that finishes last (ticket in scan_ticket[1]) folds the
//    partial boxes and sets up the grid (2. below), so the grid needs no launch of its own -- one
//    dependent launch less on the critical path of a call.  Batches keep the separate grid_setup_kernel:
//    thousands of set-ups run side by side there instead of each holding a slot of this streaming kernel.
//    The register budget is the streaming walk's (four CTAs per SM keep enough loads in flight).
template <typename T> __device__ void grid_setup_body(const Cloud<T>& c, const T* box, GridHeader<T>& hdr);
template <typename T, typename CS, bool kSetup>
__global__ void __launch_bounds__(kThreads, 4) bbox_partial_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    static_assert(kThreads % 3 == 1, "block_bbox relies on blockDim = 1 (mod 3)");
    const Cloud<T> c = clouds[blockIdx.y];
    if ((int)blockIdx.x >= c.bbox_blocks) return;
    block_bbox<T>(c.raw, 3 * c.n, blockIdx.x, c.bbox_blocks, c.bbox_partial + blockIdx.x * 6);
    if (!kSetup) return;
    if (threadIdx.x < 6) __threadfence();   // the six writers publish their words before the CTA draws its ticket
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(c.scan_ticket + 1, 1u) == (unsigned)c.bbox_blocks - 1u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ T box[6];
    __shared__ GridHeader<T> hdr;
    fold_partial_boxes<T>(c, box);
    grid_setup_body<T>(c, box, hdr);
}

//    grid (1, nclouds), kThreads threads: the grid set-up of batched calls
template <typename T, typename CS>
__global__ void __launch_bounds__(kThreads) grid_setup_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    const Cloud<T> c = clouds[blockIdx.y];
    __shared__ T box[6];
    __shared__ GridHeader<T> hdr;
    fold_partial_boxes<T>(c, box);
    grid_setup_body<T>(c, box, hdr);
}

// 2. grid shape + wall tables.  grid_setup_body: block-wide; `box` (shared, 6 values, already visible to
//    the block) -> `hdr` (shared) plus the header, pyramid shape and wall tables in device memory.
template <typename T>
__device__ void grid_setup_body(const Cloud<T>& c, const T* box, GridHeader<T>& hdr) {
    using R = Real<T>;
    using bits_t = typename R::bits_t;
    __shared__ double s_ext[3], s_lo, s_hi;
    __shared__ int s_first;
    const int maxdim = c.stride - 1;
    if (threadIdx.x == 0) {
        double emax = 0.0;
        for (int a = 0; a < 3; ++a) {
            double e = (double)box[3 + a] - (double)box[a];
            if (!(e > 0.0)) e = 0.0;        // also swallows NaN
            if (!(e < 1e300)) e = 1e300;    // +inf input: keep the arithmetic finite
            s_ext[a] = e;
            emax = fmax(emax, e);
        }
        // finest admissible cell: no axis exceeds maxdim cells, and not below the caller's limit
        s_lo = fmin(emax, fmax(emax / (double)maxdim, (double)c.min_cell));
        s_hi = emax;                        // a single cell
    }
    __syncthreads();
    const double ext0 = s_ext[0], ext1 = s_ext[1], ext2 = s_ext[2];
    const double emax = s_hi;
    const double cap = (double)c.cell_cap;
    auto cells_at = [&](double hh) {
        const double d0 = fmin(fmax(ceil(ext0 / hh), 1.0), (double)maxdim);
        const double d1 = fmin(fmax(ceil(ext1 / hh), 1.0), (double)maxdim);
        const double d2 = fmin(fmax(ceil(ext2 / hh), 1.0), (double)maxdim);
        return d0 * d1 * d2;
    };
    // Smallest h with cells_at(h) <= cap (cells_at is non-increasing in h): two rounds of a
    // blockDim-ary search over a geometric ladder between s_lo and s_hi (resolution of the ratio
    // hi/lo <= 2048 after two rounds: 2048^(1/65536), i.e. h to ~0.01 %).
    if (emax > 0.0) {
        for (int round = 0; round < 2; ++round) {
            const double lo_h = s_lo, hi_h = s_hi;
            __syncthreads();
            if (threadIdx.x == 0) s_first = blockDim.x - 1;
            __syncthreads();
            const double frac = (double)(threadIdx.x + 1) / (double)blockDim.x;
            const double cand = threadIdx.x + 1 == blockDim.x ? hi_h : lo_h * (double)exp2f((float)frac * log2f((float)(hi_h / lo_h)));
            if (cells_at(cand) <= cap) atomicMin(&s_first, (int)threadIdx.x);
            __syncthreads();
            const int first = s_first;
            __syncthreads();
            if ((int)threadIdx.x == first) {
                s_hi = cand;
                if (first > 0)   // the candidate just below; the ladder is monotone, a float-rounded rung is still a valid bracket
                    s_lo = fmin(cand, lo_h * (double)exp2f((float)first / (float)blockDim.x * log2f((float)(hi_h / lo_h))) * (1.0 - 1e-6));
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        double h = emax > 0.0 ? s_hi : 1.0;
        if (emax > 0.0 && cells_at(s_lo) <= cap) h = s_lo;
        long long nc = 1;
        for (int a = 0; a < 3; ++a) {
            double d = emax > 0.0 ? ceil(s_ext[a] / h) : 1.0;
            d = fmin(fmax(d, 1.0), (double)maxdim);
            hdr.dim[a] = (int)d;
            nc *= (long long)d;
            hdr.origin[a] = box[a];
        }
        if (nc > (long long)c.cell_cap) {  // cannot happen (cells_at(h) <= cap); belt and braces
            hdr.dim[0] = hdr.dim[1] = hdr.dim[2] = 1; nc = 1; h = emax > 0.0 ? emax : 1.0;
        }
        hdr.ncells = (int)nc;
        hdr.h = (T)h;
        hdr.inv_h = (T)(1.0 / h);
        hdr.stride = c.stride;
        hdr.pad = 0;
        // shape of the occupancy pyramid (filled by pyramid_build_kernel only if some query needs it)
        PyramidShape ps;
        int lv = 0, off = 0;
        ps.lvl_dim[0][0] = hdr.dim[0]; ps.lvl_dim[0][1] = hdr.dim[1]; ps.lvl_dim[0][2] = hdr.dim[2];
        ps.lvl_off[0] = 0;
        while ((ps.lvl_dim[lv][0] > 1 || ps.lvl_dim[lv][1] > 1 || ps.lvl_dim[lv][2] > 1) && lv < kMaxLevels) {
            for (int a = 0; a < 3; ++a) ps.lvl_dim[lv + 1][a] = (ps.lvl_dim[lv][a] + 1) / 2;
            ps.lvl_off[lv + 1] = off;
            off += ps.lvl_dim[lv + 1][0] * ps.lvl_dim[lv + 1][1] * ps.lvl_dim[lv + 1][2];
            ++lv;
        }
        ps.levels = lv;
        *c.shape = ps;
        *c.grid = hdr;
    }
    __syncthreads();
    // wall tables: bisection over the ordered-integer image of the reals, using the very cell
    // function the binning kernels use, so the walls are exact by construction.
    // only entries 0 .. dim of each axis are ever read
    const int stride = c.stride;
    const int span = max(hdr.dim[0], max(hdr.dim[1], hdr.dim[2])) + 1;
    for (int t = threadIdx.x; t < 3 * span; t += blockDim.x) {
        const int a = t / span, j = t - a * span;
        const int dim = hdr.dim[a];
        if (j > dim) continue;
        T wl, wh;
        if (j == 0) { wl = -R::inf(); wh = -R::inf(); }
        else if (j >= dim) { wl = R::inf(); wh = R::inf(); }
        else {
            bits_t lo_u = ordered<T>(hdr.origin[a]);   // cell 0 < j
            bits_t hi_u = ordered<T>(R::inf());        // clamps to dim-1 >= j
            while (hi_u - lo_u > 1) {
                const bits_t mid = lo_u + (hi_u - lo_u) / 2;
                if (cell_of<T>(unordered<T>(mid), hdr.origin[a], hdr.inv_h, dim) >= j) hi_u = mid; else lo_u = mid;
            }
            wl = unordered<T>(lo_u);
            wh = unordered<T>(hi_u);
        }
        c.wall_lo[a * stride + j] = wl;
        c.wall_hi[a * stride + j] = wh;
    }
}

// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ int linear_cell(const GridHeader<T>& g, T x, T y, T z) {
    const int cx = cell_of<T>(x, g.origin[0], g.inv_h, g.dim[0]);
    const int cy = cell_of<T>(y, g.origin[1], g.inv_h, g.dim[1]);
    const int cz = cell_of<T>(z, g.origin[2], g.inv_h, g.dim[2]);
    return (cz * g.dim[1] + cy) * g.dim[0] + cx;
}

// Tile staging for the two binning kernels: the kThreads points of a CTA are one contiguous run of
// 3 * kThreads scalars of the caller's (n, 3) array.  One elected thread fetches the whole run with a
// single bulk asynchronous copy (cp.async.bulk -> SASS UBLKCP, completion counted on an mbarrier) into
// shared memory, from where thread t picks scalars 3t, 3t+1, 3t+2 (stride 3: conflict-free).  This
// replaces three stride-3 global loads per thread.  Bulk copies need a 16-byte aligned source and a
// size that is a multiple of 16 bytes; ragged tails and unaligned views take the plain-load path.
__device__ __forceinline__ void mbarrier_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bulk_load_tile(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(b) : "memory");
}
__device__ __forceinline__ void mbarrier_wait(unsigned long long* bar, unsigned parity) {
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
    unsigned done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(b), "r"(parity) : "memory");
    }
}

// Loads the grid header and this thread's point (row blockIdx.x * kThreads + threadIdx.x of the cloud).
// Returns false for threads past the end of the cloud.  Contains block-wide barriers.
template <typename T>
__device__ __forceinline__ bool load_tile_point(const Cloud<T>& c, GridHeader<T>& g, T (&tile)[3 * kThreads],
                                                unsigned long long& bar, long long& i, T& x, T& y, T& z) {
    const long long first = (long long)blockIdx.x * kThreads;
    const long long left = c.n - first;
    const int count = left < kThreads ? (int)left : kThreads;
    const T* src = c.raw + 3 * first;
    const unsigned bytes = (unsigned)(3 * count * sizeof(T));
    const bool bulk = count > 0 && (bytes & 15u) == 0u && (reinterpret_cast<unsigned long long>(src) & 15ull) == 0ull;
    if (threadIdx.x == 0) {
        g = *c.grid;
        if (bulk) mbarrier_init(&bar, 1);
    }
    __syncthreads();
    if (bulk) {
        if (threadIdx.x == 0) bulk_load_tile(tile, src, bytes, &bar);
        mbarrier_wait(&bar, 0);
    }
    i = first + threadIdx.x;
    if ((int)threadIdx.x >= count) return false;
    if (bulk) { x = tile[3 * threadIdx.x]; y = tile[3 * threadIdx.x + 1]; z = tile[3 * threadIdx.x + 2]; }
    else { x = __ldg(src + 3 * threadIdx.x); y = __ldg(src + 3 * threadIdx.x + 1); z = __ldg(src + 3 * threadIdx.x + 2); }
    return true;
}

// How densely the non-empty cells turned out to be filled, left in host-mapped memory for the NEXT call
// with the same shapes on this workspace (nearest.cu sizes that call's grid from it: surfaces and
// other thin sets fill few cells of a box-filling grid, each with many points).  A hint only.
//   words 0..3: {cell_cap, non-empty cells, n, valid}  (binning kernels)
//   words 4..6: {queries the 27 cells around them could not settle, queries, valid}  (first slow pass of a search
//               against this cloud)
template <typename T>
__device__ __forceinline__ void publish_grid_hint(const Cloud<T>& c, unsigned nonempty) {
    volatile unsigned* h = c.hint_out;
    h[0] = (unsigned)c.cell_cap; h[1] = nonempty; h[2] = (unsigned)c.n; h[3] = 1u;
}
template <typename T>
__device__ __forceinline__ void publish_far_hint(const Cloud<T>& dataset, unsigned n_far, long long n_queries) {
    if (dataset.hint_out == nullptr) return;
    volatile unsigned* h = dataset.hint_out;
    h[4] = n_far; h[5] = (unsigned)n_queries; h[6] = 1u;
}

// 3. histogram; the atomic's return value is the point's rank inside its cell.
//    grid (ceil(max_n / kThreads), nclouds)
template <typename T, typename CS>
__global__ void __launch_bounds__(kThreads) cell_count_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    const Cloud<T> c = clouds[blockIdx.y];
    if ((long long)blockIdx.x * kThreads >= c.n) return;
    __shared__ GridHeader<T> g;
    __shared__ __align__(16) T tile[3 * kThreads];
    __shared__ __align__(8) unsigned long long bar;
    long long i; T x, y, z;
    if (!load_tile_point<T>(c, g, tile, bar, i, x, y, z)) return;
    c.rank[i] = atomicAdd(c.cell_start + linear_cell<T>(g, x, y, z), 1u);
}

// ---------------------------------------------------------------------------------------------
// 4. exclusive scan of cell_start[0 .. cell_cap], in place: a single-pass scan with decoupled look-back.
//    Every CTA draws a tile ticket, scans its tile, publishes the tile total, and resolves its carry by walking
//    back over the published states of the tiles before it.
//    state word = status (bits 63:62; 1 = tile total, 2 = inclusive prefix) | value (low 32).
//    Ticket and states must be zero on entry (they live in the call's zeroed region).  grid (tiles, nclouds)
template <typename T, typename CS>
__global__ void __launch_bounds__(kScanThreads) scan_lookback_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    const Cloud<T> c = clouds[blockIdx.y];
    const long long count = (long long)c.cell_cap + 1;
    __shared__ unsigned s_tile, s_carry;
    if (threadIdx.x == 0) s_tile = atomicAdd(c.scan_ticket, 1u);
    __syncthreads();
    const unsigned tile = s_tile;
    const long long base = (long long)tile * kScanTile;
    if (base >= count) return;
    unsigned v[kScanItems];
    unsigned s = 0, nonempty = 0;
    const long long first = base + (long long)threadIdx.x * kScanItems;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        v[k] = (first + k) < count ? c.cell_start[first + k] : 0u;
        s += v[k];
        nonempty += v[k] != 0u;
    }
    nonempty = __reduce_add_sync(0xffffffffu, nonempty);
    if ((threadIdx.x & 31) == 0 && nonempty != 0u) atomicAdd(c.occupied, nonempty);
    unsigned total;
    const unsigned ex = block_exclusive_scan<kScanThreads>(s, &total);
    if (threadIdx.x < 32) {
        // warp-wide look-back: lane l inspects tile (tile - 1 - l), 32 predecessors per step
        volatile unsigned long long* state = c.scan_state;
        const int lane = threadIdx.x;
        if (lane == 0) state[tile] = ((tile == 0 ? 2ull : 1ull) << 62) | total;
        unsigned carry = 0;
        if (tile > 0) {
            for (long long p = (long long)tile - 1;; p -= 32) {
                const long long mine = p - lane;
                unsigned long long w = 2ull << 62;            // lanes before tile 0 act as a zero prefix
                if (mine >= 0) do { w = state[mine]; } while ((w >> 62) == 0);
                const unsigned has_prefix = __ballot_sync(0xffffffffu, (w >> 62) == 2);
                const int stop = has_prefix ? __ffs(has_prefix) - 1 : 31;   // nearest predecessor holding a prefix
                const unsigned part = lane <= stop ? (unsigned)w : 0u;
                carry += __reduce_add_sync(0xffffffffu, part);
                if (has_prefix) break;
            }
            if (lane == 0) state[tile] = (2ull << 62) | (unsigned long long)(carry + total);
        }
        if (lane == 0) s_carry = carry;
    }
    __syncthreads();
    unsigned run = ex + s_carry;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        if ((first + k) < count) c.cell_start[first + k] = run;
        run += v[k];
    }
}

// ---------------------------------------------------------------------------------------------
// 5. scatter into cell order: grid (ceil(max_n / kThreads), nclouds)
template <typename T, typename CS>
__global__ void __launch_bounds__(kThreads) scatter_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    const Cloud<T> c = clouds[blockIdx.y];
    if ((long long)blockIdx.x * kThreads >= c.n) return;
    if (blockIdx.x == 0 && threadIdx.x == 0 && c.hint_out != nullptr) publish_grid_hint<T>(c, *c.occupied);
    __shared__ GridHeader<T> g;
    __shared__ __align__(16) T tile[3 * kThreads];
    __shared__ __align__(8) unsigned long long bar;
    long long i; T x, y, z;
    if (!load_tile_point<T>(c, g, tile, bar, i, x, y, z)) return;
    const unsigned pos = c.cell_start[linear_cell<T>(g, x, y, z)] + c.rank[i];
    store_pt<T>(c.sorted + pos, x, y, z, i);
}

// ---------------------------------------------------------------------------------------------
// 3-5 as a slab build (single pairs above 8192 points).  The linear cell indices 0 .. ncells - 1 are cut
// into c.slabs slabs of W = ceil(ncells / slabs) consecutive cells.  The host picks `slabs` so that a
// slab holds kSlabMeanFill of a staging buffer (kSlabStageBytes) of points on average and its cells fit
// shared-memory counters; W follows from the actual ncells on the device.  Every point is read twice
// from the caller's array and its record is written twice, each time as contiguous runs, instead of
// one returning L2 atomic, one dependent gather and one 16-byte store at a random address per point.
//   slab_hist_kernel       chunk CTAs histogram the slabs of their points; the last one scans the totals
//   slab_partition_kernel  the same chunks: one run per (chunk, slab), reserved with one atomic
//   slab_sort_kernel       one CTA per slab sorts its records by cell in shared memory
// The result is the layout of the cell-wise passes: same cell_start, same set of points per cell.
// Only the order inside a cell differs, and that order was arrival order there too.
//
// The chunk CTAs (grid (max slab_chunks, nclouds)) walk their chunk kSlabTile points at a time: the
// 3 * kSlabTile scalars of a tile are read flat (coalesced, any alignment) into registers, put in shared
// memory, and thread t takes points t, t + kSlabThreads, ... of the tile.  The next tile's loads are
// issued before the current tile is processed.  Dynamic shared memory: the per-slab counters, then the
// tile (slab_hist_smem / slab_part_smem below).
template <typename T>
__device__ __forceinline__ int slab_width(const GridHeader<T>& g, int slabs) { return (g.ncells + slabs - 1) / slabs; }

// n / w for any 32-bit n without a divide instruction: m = floor((2^32 - 1) / w) makes umulhi(n, m) either
// the quotient or one less, and the remainder tells which.
struct SlabOf {
    unsigned w, m;
    __device__ explicit SlabOf(unsigned width) : w(width), m(0xffffffffu / width) {}
    __device__ __forceinline__ unsigned operator()(unsigned n) const {
        const unsigned q = __umulhi(n, m);
        return q + (n - q * w >= w ? 1u : 0u);
    }
};

// f(t0, count) runs once per tile, with points t0 .. t0 + count - 1 of the cloud in `tile` (x, y, z each).
template <typename T, typename F>
__device__ __forceinline__ void for_chunk_tiles(const Cloud<T>& c, T* tile, F&& f) {
    constexpr int kPer = 3 * kSlabTile / kSlabThreads;
    const long long len = (((c.n + c.slab_chunks - 1) / c.slab_chunks) + 3) & ~3ll;
    const long long first = (long long)blockIdx.x * len;
    const long long end = first + len < c.n ? first + len : c.n;
    T v[kPer];
    auto fetch = [&](long long t0) {
        const long long left = 3 * (end - t0);
        const T* src = c.raw + 3 * t0;
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int e = (int)threadIdx.x + k * kSlabThreads;
            v[k] = e < left ? __ldg(src + e) : (T)0;
        }
    };
    if (first < end) fetch(first);
    for (long long t0 = first; t0 < end; t0 += kSlabTile) {
        __syncthreads();   // the previous tile has been consumed
#pragma unroll
        for (int k = 0; k < kPer; ++k) tile[threadIdx.x + k * kSlabThreads] = v[k];
        __syncthreads();
        if (t0 + kSlabTile < end) fetch(t0 + kSlabTile);
        f(t0, end - t0 < kSlabTile ? (int)(end - t0) : kSlabTile);
    }
}

__host__ __device__ __forceinline__ size_t slab_counter_bytes(int slabs) { return ((size_t)slabs * sizeof(unsigned) + 15) & ~(size_t)15; }

// The partition stages a tile in slab order when the tile holds at least one point per slab on average;
// with fewer, the scan over the slab counters costs more than the coalesced stores win back, and every
// point goes straight to its run.
__host__ __device__ __forceinline__ bool slab_staged(int slabs) { return slabs <= kSlabTile; }

template <typename T>
__host__ __device__ __forceinline__ size_t slab_hist_smem(int slabs) { return slab_counter_bytes(slabs) + (size_t)3 * kSlabTile * sizeof(T); }

// Staged partition: cursors, tile counts and tile offsets (one counter array each), the tile, then the
// tile's order by slab (one word per point).
template <typename T>
__host__ __device__ __forceinline__ size_t slab_part_smem(int slabs) {
    return slab_staged(slabs) ? 2 * slab_counter_bytes(slabs) + slab_hist_smem<T>(slabs) + (size_t)kSlabTile * sizeof(unsigned)
                              : slab_hist_smem<T>(slabs);
}

// 3. slab histogram + scan of the slab totals: grid (max slab_chunks, nclouds), kSlabThreads threads.
//    Row blockIdx.x of slab_hist gets this chunk's count of every slab; the CTA that finishes last (ticket
//    in scan_ticket[0]) scans the totals into slab_base and resets slab_count to those bases.
template <typename T, typename CS>
__global__ void __launch_bounds__(kSlabThreads) slab_hist_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    const Cloud<T> c = clouds[blockIdx.y];
    if ((int)blockIdx.x >= c.slab_chunks) return;
    extern __shared__ __align__(16) unsigned char slab_smem[];
    const int S = c.slabs;
    unsigned* cnt = reinterpret_cast<unsigned*>(slab_smem);
    T* tile = reinterpret_cast<T*>(slab_smem + slab_counter_bytes(S));
    __shared__ GridHeader<T> g;
    __shared__ bool s_last;
    if (threadIdx.x == 0) g = *c.grid;
    for (int i = threadIdx.x; i < S; i += kSlabThreads) cnt[i] = 0u;
    __syncthreads();
    const SlabOf slab_of((unsigned)slab_width<T>(g, S));
    for_chunk_tiles<T>(c, tile, [&](long long, int count) {
#pragma unroll
        for (int j = 0; j < kSlabTile / kSlabThreads; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) atomicAdd(&cnt[slab_of((unsigned)linear_cell<T>(g, tile[3 * p], tile[3 * p + 1], tile[3 * p + 2]))], 1u);
        }
    });
    __syncthreads();
    unsigned* row = c.slab_hist + (size_t)blockIdx.x * S;
    for (int i = threadIdx.x; i < S; i += kSlabThreads) {
        const unsigned v = cnt[i];
        row[i] = v;
        if (v != 0u) atomicAdd(c.slab_count + i, v);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(c.scan_ticket, 1u) == (unsigned)c.slab_chunks - 1u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const unsigned all = block_scan_rounds<kSlabThreads>(
        S, [&](int i) { return __ldcg(c.slab_count + i); },
        [&](int i, unsigned ex, unsigned) { c.slab_base[i] = ex; c.slab_count[i] = ex; });
    if (threadIdx.x == 0) c.slab_base[S] = all;
}

// 4. slab partition: grid as slab_hist_kernel, dynamic shared memory slab_part_smem.  The chunk's run in
//    slab s is reserved with one atomic on slab_count[s]; cur[s] is the next free position of that run.
//    When slab_staged(S), each tile is counting-sorted by slab in shared memory first: its slab counts are
//    scanned into the tile's order by slab, and thread q stores the q-th point of that order, so consecutive
//    lanes store consecutive addresses of a run.  Otherwise each point is stored at its run's cursor.
template <typename T, typename CS>
__global__ void __launch_bounds__(kSlabThreads) slab_partition_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    constexpr int kPer = kSlabTile / kSlabThreads;
    static_assert(kSlabTile <= (1 << 16), "slab and tile position share one word");
    const Cloud<T> c = clouds[blockIdx.y];
    if ((int)blockIdx.x >= c.slab_chunks) return;
    extern __shared__ __align__(16) unsigned char slab_smem[];
    const int S = c.slabs;
    const bool staged = slab_staged(S);
    const size_t counters = slab_counter_bytes(S);
    unsigned* cur = reinterpret_cast<unsigned*>(slab_smem);
    unsigned* tcnt = reinterpret_cast<unsigned*>(slab_smem + counters);       // tile counts, then their prefix
    unsigned* off = reinterpret_cast<unsigned*>(slab_smem + 2 * counters);    // run position - position in the order
    T* tile = reinterpret_cast<T*>(slab_smem + (staged ? 3 : 1) * counters);
    unsigned* order = reinterpret_cast<unsigned*>(tile + 3 * kSlabTile);      // slab << 16 | tile position
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *c.grid;
    const unsigned* row = c.slab_hist + (size_t)blockIdx.x * S;
    for (int i = threadIdx.x; i < S; i += kSlabThreads) {
        const unsigned v = row[i];
        cur[i] = v != 0u ? atomicAdd(c.slab_count + i, v) : 0u;
        if (staged) tcnt[i] = 0u;
    }
    __syncthreads();
    const SlabOf slab_of((unsigned)slab_width<T>(g, S));
    if (!staged) {
        for_chunk_tiles<T>(c, tile, [&](long long t0, int count) {
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int p = (int)threadIdx.x + j * kSlabThreads;
                if (p < count) {
                    const T x = tile[3 * p], y = tile[3 * p + 1], z = tile[3 * p + 2];
                    const unsigned pos = atomicAdd(&cur[slab_of((unsigned)linear_cell<T>(g, x, y, z))], 1u);
                    store_pt<T>(c.part + pos, x, y, z, t0 + p);
                }
            }
        });
        return;
    }
    for_chunk_tiles<T>(c, tile, [&](long long t0, int count) {
        unsigned key[kPer];   // slab << 16 | rank inside the tile's share of the slab
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) {
                const unsigned s = slab_of((unsigned)linear_cell<T>(g, tile[3 * p], tile[3 * p + 1], tile[3 * p + 2]));
                key[j] = s << 16 | atomicAdd(&tcnt[s], 1u);
            }
        }
        __syncthreads();
        block_scan_rounds<kSlabThreads>(S, [&](int i) { return tcnt[i]; }, [&](int i, unsigned ex, unsigned v) {
            const unsigned run = cur[i];
            tcnt[i] = ex;
            off[i] = run - ex;
            cur[i] = run + v;
        });
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) order[tcnt[key[j] >> 16] + (key[j] & 0xffffu)] = (key[j] & 0xffff0000u) | (unsigned)p;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int q = (int)threadIdx.x + j * kSlabThreads;
            if (q < count) {
                const unsigned w = order[q], p = w & 0xffffu;
                store_pt<T>(c.part + off[w >> 16] + q, tile[3 * p], tile[3 * p + 1], tile[3 * p + 2], t0 + p);
            }
        }
        for (int i = threadIdx.x; i < S; i += kSlabThreads) tcnt[i] = 0u;
    });
}

// 5. per-slab cell sort: grid (max slabs, nclouds), kSlabThreads threads, dynamic shared memory
//    kSlabStageBytes + 4 * (most cells a slab can have).  A slab that fits the staging buffer ranks its
//    records with shared counters (cell and rank stay in one register per record), reads them again (from
//    L2: the slab was just read), places them in shared memory and writes them out coalesced.  A larger slab (clusters, duplicates, surfaces) counts from global memory, then
//    scatters with shared cursors into its own range of `sorted`: slower, bounded by the slab's size.
//    Writes cell_start for the slab's cells (slab_base + local prefix), and the last slab also the entries
//    ncells .. cell_cap (= n).  The last CTA to finish publishes the count of non-empty cells.
template <typename T, typename CS>
__global__ void __launch_bounds__(kSlabThreads) slab_sort_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    constexpr int kCap = kSlabStageBytes / (int)sizeof(Pt<T>);
    constexpr int kPer = kCap / kSlabThreads;
    const Cloud<T> c = clouds[blockIdx.y];
    const int S = c.slabs, s = blockIdx.x;
    if (s >= S) return;
    extern __shared__ __align__(16) unsigned char slab_smem[];
    Pt<T>* stage = reinterpret_cast<Pt<T>*>(slab_smem);
    unsigned* cnt = reinterpret_cast<unsigned*>(slab_smem + kSlabStageBytes);
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *c.grid;
    __syncthreads();
    const int W = slab_width<T>(g, S);
    const int cell0 = s * W;
    const int ncell = max(0, min(W, g.ncells - cell0));
    const unsigned base = c.slab_base[s];
    const int count = (int)(c.slab_base[s + 1] - base);
    const Pt<T>* src = c.part + base;
    for (int i = threadIdx.x; i < ncell; i += kSlabThreads) cnt[i] = 0u;
    __syncthreads();
    const bool staged = count <= kCap;
    static_assert(kSlabMaxCells <= (1 << 18) && kCap <= (1 << 14), "cell and rank share one word");
    unsigned slot[kPer];   // cell inside the slab << 14 | rank inside the cell
    if (staged) {
        Pt<T> r[kPer];
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) r[j] = load_pt<T>(src + p);
        }
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) {
                const unsigned lc = (unsigned)(linear_cell<T>(g, r[j].x, r[j].y, r[j].z) - cell0);
                slot[j] = lc << 14 | atomicAdd(&cnt[lc], 1u);
            }
        }
    } else {
        for (int p = threadIdx.x; p < count; p += kSlabThreads) {
            const Pt<T> q = load_pt<T>(src + p);
            atomicAdd(&cnt[linear_cell<T>(g, q.x, q.y, q.z) - cell0], 1u);
        }
    }
    __syncthreads();
    unsigned nonempty = 0;
    block_scan_rounds<kSlabThreads>(ncell, [&](int i) { return cnt[i]; }, [&](int i, unsigned ex, unsigned v) {
        cnt[i] = ex;
        c.cell_start[cell0 + i] = base + ex;
        nonempty += v != 0u;
    });
    if (s == S - 1)
        for (int i = g.ncells + threadIdx.x; i <= c.cell_cap; i += kSlabThreads) c.cell_start[i] = (unsigned)c.n;
    if (staged) {
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int p = (int)threadIdx.x + j * kSlabThreads;
            if (p < count) stage[cnt[slot[j] >> 14] + (slot[j] & 0x3fffu)] = load_pt<T>(src + p);
        }
        __syncthreads();
        for (int p = threadIdx.x; p < count; p += kSlabThreads) c.sorted[base + p] = stage[p];
    } else {
        for (int p = threadIdx.x; p < count; p += kSlabThreads) {
            const Pt<T> q = load_pt<T>(src + p);
            const unsigned pos = atomicAdd(&cnt[linear_cell<T>(g, q.x, q.y, q.z) - cell0], 1u);
            store_pt<T>(c.sorted + base + pos, q.x, q.y, q.z, q.i);
        }
    }
    if (c.hint_out != nullptr) {
        __shared__ bool s_last;
        nonempty = __reduce_add_sync(0xffffffffu, nonempty);
        if ((threadIdx.x & 31) == 0 && nonempty != 0u) atomicAdd(c.occupied, nonempty);
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) s_last = atomicAdd(c.scan_ticket + 2, 1u) == (unsigned)S - 1u;
        __syncthreads();
        if (s_last && threadIdx.x == 0) publish_grid_hint<T>(c, atomicAdd(c.occupied, 0u));
    }
}

// ---------------------------------------------------------------------------------------------
// 1-5 in one launch for small clouds: one CTA of kSmallThreads threads bins one whole cloud.  The cell
// counters (cell_cap + 1 words, dynamic shared memory) never leave the SM: the histogram and the
// scatter cursors are shared-memory atomics instead of L2 atomics, the scan is block-local, and a batch
// of B pairs is one launch of 2B independent CTAs instead of five grid-wide passes.  The order of the
// points inside a cell is arbitrary here as in the general path (every consumer orders candidates by
// (distance, index)).  grid (nclouds), dynamic shared memory 4 * (max cell_cap + 1) bytes.
template <typename T, typename CS>
__global__ void __launch_bounds__(kSmallThreads, 1) bin_small_kernel(const __grid_constant__ CS clouds) {
    grid_dependency_wait();
    static_assert(kSmallThreads % 3 == 1, "block_bbox relies on blockDim = 1 (mod 3)");
    extern __shared__ __align__(16) unsigned char small_smem[];
    unsigned* cnt = reinterpret_cast<unsigned*>(small_smem);
    const Cloud<T> c = clouds[blockIdx.x];
    __shared__ T box[6];
    __shared__ GridHeader<T> hdr;
    __shared__ unsigned s_nonempty;
    const int t = threadIdx.x, lane = t & 31;
    const int ncount = c.cell_cap + 1;
    if (t == 0) s_nonempty = 0u;
    for (int i = t; i < ncount; i += kSmallThreads) cnt[i] = 0u;
    block_bbox<T>(c.raw, 3 * c.n, 0, 1, box);
    __syncthreads();
    grid_setup_body<T>(c, box, hdr);
    const GridHeader<T> g = hdr;
    const int n = (int)c.n;
    constexpr int kBatch = 4;
    // histogram
    for (int first = t; first < n; first += kBatch * kSmallThreads) {
        T p[kBatch][3];
#pragma unroll
        for (int b = 0; b < kBatch; ++b) {
            const int i = first + b * kSmallThreads;
            if (i < n) { p[b][0] = __ldg(c.raw + 3ll * i); p[b][1] = __ldg(c.raw + 3ll * i + 1); p[b][2] = __ldg(c.raw + 3ll * i + 2); }
        }
#pragma unroll
        for (int b = 0; b < kBatch; ++b)
            if (first + b * kSmallThreads < n) atomicAdd(&cnt[linear_cell<T>(g, p[b][0], p[b][1], p[b][2])], 1u);
    }
    __syncthreads();
    // exclusive scan of the counters; the prefix goes to cell_start and stays in shared memory as the scatter cursors
    unsigned nonempty = 0;
    block_scan_rounds<kSmallThreads>(ncount, [&](int i) { return cnt[i]; }, [&](int i, unsigned ex, unsigned v) {
        cnt[i] = ex;
        c.cell_start[i] = ex;
        nonempty += v != 0u;
    });
    if (c.hint_out != nullptr) {
        nonempty = __reduce_add_sync(0xffffffffu, nonempty);
        if (lane == 0 && nonempty != 0u) atomicAdd(&s_nonempty, nonempty);
        __syncthreads();
        if (t == 0) publish_grid_hint<T>(c, s_nonempty);
    }
    // scatter
    for (int first = t; first < n; first += kBatch * kSmallThreads) {
        T p[kBatch][3];
#pragma unroll
        for (int b = 0; b < kBatch; ++b) {
            const int i = first + b * kSmallThreads;
            if (i < n) { p[b][0] = __ldg(c.raw + 3ll * i); p[b][1] = __ldg(c.raw + 3ll * i + 1); p[b][2] = __ldg(c.raw + 3ll * i + 2); }
        }
#pragma unroll
        for (int b = 0; b < kBatch; ++b) {
            const int i = first + b * kSmallThreads;
            if (i < n) {
                const unsigned pos = atomicAdd(&cnt[linear_cell<T>(g, p[b][0], p[b][1], p[b][2])], 1u);
                store_pt<T>(c.sorted + pos, p[b][0], p[b][1], p[b][2], i);
            }
        }
    }
}

}  // namespace pcu
