// compact.cuh -- order-preserving compaction of flagged rows, shared by every feature that keeps a subset of its rows
// (normals, voxel and Poisson-disk downsampling, duplicate removal, marching cubes, the voxel-grid boundary).
//
// Three steps over n one-byte flags, one thread per row and kThreads rows per block:
//   keep_count_kernel     kept rows of every block                                    -> block_count[block]
//   keep_offsets_kernel   one CTA: exclusive scan of the block counts, in place       -> block_offset[block]; the total
//   an emit kernel        every thread asks keep_rank for the kept rows before its own and writes its row there
// so the kept rows leave in ascending order, as a sequential loop that appends them would write them.  n < 2^31 rows:
// ranks and block counts fit 32 bits.
// The first two kernels are compiled once, in runtime.cu, and launched through enqueue_keep_offsets (runtime.cuh).
#pragma once
#include "common.cuh"

namespace pcu {

// The number of kept rows before this thread's row (kInclusive: up to and including it), over the whole array: the
// block's offset, the kept rows of the earlier warps of the block, those of the earlier lanes of the warp.  `mine`:
// this thread's row is kept (false for a thread past the end); block_offset: what keep_offsets_kernel left.
// It holds a barrier: EVERY thread of the block (kThreads threads, one row each, block b at rows b * kThreads...) calls
// it, once, and a thread with nothing to write returns only afterwards.
template <bool kInclusive = false>
__device__ __forceinline__ unsigned keep_rank(bool mine, const unsigned* __restrict__ block_offset) {
    __shared__ unsigned warp_sum[kThreads / 32];
    const unsigned ballot = __ballot_sync(0xffffffffu, mine);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_sum[w] = __popc(ballot);
    __syncthreads();
    unsigned before = block_offset[blockIdx.x];
    for (int j = 0; j < w; ++j) before += warp_sum[j];
    return before + __popc(ballot & (((kInclusive ? 2u : 1u) << lane) - 1u));
}

// The kept row numbers in ascending order, as I (int32 or int64).
template <typename I>
__global__ void __launch_bounds__(kThreads) keep_rows_kernel(const unsigned char* __restrict__ keep, long long n,
                                                             const unsigned* __restrict__ block_offset, I* __restrict__ out_idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mine = i < n ? keep[i] : 0u;
    const unsigned pos = keep_rank(mine, block_offset);
    if (mine) out_idx[pos] = (I)i;
}

}  // namespace pcu
