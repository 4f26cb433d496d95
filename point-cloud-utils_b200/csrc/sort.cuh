// sort.cuh -- stable least-significant-digit radix sort of fixed-size records (multi-word keys + one payload word).
//
// Used where the reference needs a lexicographic ROW order (igl::sortrows inside igl::unique_rows, called by
// src/remove_duplicates.cpp:27-33): the keys are the order-preserving integer images of the coordinates, most
// significant word first, and a stable sort keeps records with equal keys in payload (= row) order.
//
// One pass = one 8-bit digit:
//   sort_hist_kernel     per-tile histogram of the digit                      -> hist[bin][tile]
//   sort_scan_rows       one CTA per bin: exclusive scan over the tiles       -> hist (in place), total[bin]
//   sort_scan_bins       one CTA: exclusive scan over the 256 bin totals      -> base[bin]; constant-digit flag
//   sort_scatter_kernel  every warp owns a contiguous 512-record slice of its tile: it counts its digits
//                        (match.any, no atomics), the CTA turns the 8 x 256 warp counts into running global
//                        positions, and the warp walks its slice again in the same order, placing each record
//                        at position[digit] + (rank among the lanes of this step with the same digit).
// A digit that is the same in every record (common in the high bytes of coordinates) degenerates into a plain
// coalesced copy.  HBM traffic per pass: the records are read twice (the second time from L2) and written once.
#pragma once
#include "common.cuh"

namespace pcu {

constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortRounds = 16;                             // records per lane
constexpr int kSortTile = kSortThreads * kSortRounds;       // 4096 records per CTA
constexpr int kSortBins = 256;

// K: uint32_t or unsigned long long.  key[0] is the most significant word.
template <typename K, int NW>
struct __align__(sizeof(K) * 4) SortRec {
    K key[NW];
    K idx;
};

template <typename Rec>
__device__ __forceinline__ Rec load_rec(const Rec* p) {
    Rec r;
    if (sizeof(Rec) == 16) {
        const uint4 v = *reinterpret_cast<const uint4*>(p);
        *reinterpret_cast<uint4*>(&r) = v;
    } else {
        const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
        reinterpret_cast<uint4*>(&r)[0] = a;
        reinterpret_cast<uint4*>(&r)[1] = b;
    }
    return r;
}
template <typename Rec>
__device__ __forceinline__ void store_rec(Rec* p, const Rec& r) {
    if (sizeof(Rec) == 16) {
        *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&r);
    } else {
        reinterpret_cast<uint4*>(p)[0] = reinterpret_cast<const uint4*>(&r)[0];
        reinterpret_cast<uint4*>(p)[1] = reinterpret_cast<const uint4*>(&r)[1];
    }
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

// The two scans of a pass are compiled once, in runtime.cu; radix_sort_records (runtime.cuh) launches them.
__global__ void sort_scan_rows(unsigned* __restrict__ hist, unsigned ntiles, unsigned long long* __restrict__ total);
__global__ void sort_scan_bins(const unsigned long long* __restrict__ total, long long n, unsigned* __restrict__ base,
                               int* __restrict__ constant);

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

}  // namespace pcu
