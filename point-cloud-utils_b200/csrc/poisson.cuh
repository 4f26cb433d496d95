// poisson.cuh -- Poisson-disk downsampling of a point cloud (downsample_point_cloud_poisson_disk of the reference,
// src/sample_point_cloud.cpp:14-109, :240-333).
//
// The reference draws its subset with libigl's blue-noise helpers and std::mt19937 over an std::unordered_map, so its
// exact subset cannot be reproduced.  The sample here is defined exactly instead (DESIGN.md §3, Poisson-disk sample):
//   conflict   rows p, q conflict iff d2(p, q) < rr, d2 the reference-rounded metric of common.cuh, rr = fl_T(r * r);
//   priority   key(row) = (mix32(seed ^ mix32(row * 0x9e3779b9 + 0x85ebca6b)), row), compared lexicographically;
//   sample     the greedy maximal independent set in key order: visit rows by ascending key, keep a row when it
//              conflicts with no kept row.
// It is computed in rounds.  Every undecided point walks its ball (walk_ball_until):
//   a neighbour already IN                        -> the point is OUT (the walk stops there);
//   else an undecided neighbour with a smaller key -> the point stays undecided;
//   else                                          -> the point is IN.
// A state only ever leaves "undecided", and each such move is the sequential greedy's own decision (an IN neighbour
// is a kept row the point conflicts with; all smaller-key neighbours OUT means no kept row precedes it), so what a
// point reads of its neighbours in the middle of a round cannot change the result -- only how soon it is decided.
// The undecided point of smallest key is decided in every round, so the rounds end.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"
#include "normals.cuh"

namespace pcu {

constexpr unsigned char kPoissonUndecided = 0, kPoissonIn = 1, kPoissonOut = 2;

__device__ __forceinline__ unsigned long long poisson_key(unsigned seed, unsigned row) {
    return ((unsigned long long)mix32(seed ^ mix32(row * 0x9e3779b9u + 0x85ebca6bu)) << 32) | row;
}

struct PoissonScratch {
    unsigned* ring;          // [3] lengths of the undecided lists, cycled over the rounds; zeroed per call
    unsigned char* state;    // n, by sorted position: kPoisson*; zeroed per call
    unsigned char* keep;     // n, by row: 1 = sample; zeroed per call
    unsigned* list[2];       // undecided positions: read in one round, written for the next
};

// All rounds in one cooperative launch: a grid barrier separates them, and between them the undecided points are
// compacted (warp ballot, one atomic per warp: the order inside a list does not matter, the result does not depend
// on it), so late rounds touch only what is left.  rounds_out (may be null): rounds run.
template <typename T>
__global__ void __launch_bounds__(kThreads) poisson_rounds_kernel(Cloud<T> cl, T rr, unsigned seed, PoissonScratch s,
                                                                  int* __restrict__ rounds_out) {
    namespace cg = cooperative_groups;
    grid_dependency_wait();
    __shared__ GridHeader<T> g;
    if (threadIdx.x == 0) g = *cl.grid;
    __syncthreads();
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long gsize = (long long)gridDim.x * blockDim.x;
    volatile unsigned char* state = s.state;   // neighbours decide while we read: no cached or hoisted loads
    long long todo = cl.n;
    int round = 0;
    for (; todo > 0; ++round) {
        const unsigned* in_list = s.list[round & 1];
        unsigned* out_list = s.list[(round + 1) & 1];
        unsigned* next = s.ring + (round + 1) % 3;
        // the slot after next was last read right after the previous barrier but one, and is next written after the
        // coming barrier
        if (gtid == 0) s.ring[(round + 2) % 3] = 0u;
        for (long long i = gtid; i - lane < todo; i += gsize) {    // whole warps: the ballot below needs every lane
            bool undecided = false;
            unsigned pos = 0;
            if (i < todo) {
                pos = round == 0 ? (unsigned)i : in_list[i];
                const Pt<T> q = load_pt<T>(cl.sorted + pos);
                const unsigned long long mine = poisson_key(seed, (unsigned)q.i);
                bool blocked = false;
                const bool out = walk_ball_until<T>(cl, g, q, rr, [&](unsigned j, const Pt<T>& p, T) {
                    if (j == pos) return false;
                    const unsigned char st = state[j];
                    if (st == kPoissonIn) return true;
                    if (st == kPoissonUndecided && !blocked && poisson_key(seed, (unsigned)p.i) < mine) blocked = true;
                    return false;
                });
                if (out) {
                    state[pos] = kPoissonOut;
                } else if (!blocked) {
                    state[pos] = kPoissonIn;
                    s.keep[q.i] = 1;
                } else {
                    undecided = true;
                }
            }
            const unsigned ballot = __ballot_sync(0xffffffffu, undecided);
            if (ballot != 0u) {
                unsigned base = 0u;
                if (lane == 0) base = atomicAdd(next, (unsigned)__popc(ballot));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (undecided) out_list[base + __popc(ballot & ((1u << lane) - 1u))] = pos;
            }
        }
        grid.sync();
        todo = *(volatile unsigned*)next;
    }
    if (gtid == 0 && rounds_out != nullptr) *rounds_out = round;
}

}  // namespace pcu
