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
// The four kernels and radix_sort_records (runtime.cuh), which launches them, are compiled once, in runtime.cu; this
// header keeps the record type and the record loads and stores that the kernels writing and reading records share.
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

}  // namespace pcu
