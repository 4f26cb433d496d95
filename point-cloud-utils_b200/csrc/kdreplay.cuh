// kdreplay.cuh -- GPU replica of the reference's kd-tree, used ONLY for queries whose answer
// depends on how exactly-equal distances are ordered.
//
// nanoflann breaks distance ties by kd-tree visit order (strict comparisons at
// external/nanoflann/nanoflann.hpp:206 and :1563 of the reference; NANOFLANN_FIRST_MATCH is not
// defined), so bit-identical indices for tied queries need the very tree the reference builds:
// the same split dimension / value at every node and the same permutation of points inside every
// leaf.  The grid search flags such queries (search.cuh); this file rebuilds that tree on the GPU
// and re-answers just those queries by walking it exactly like nanoflann does.
//
//   build   : level-synchronous restatement of divideTree / middleSplit_ / planeSplit
//             (nanoflann.hpp:1001-1059, :1061-1110, :1121-1162).  planeSplit's two-pointer exchange
//             is deterministic -- the j-th misplaced element from the left trades places with the
//             j-th misplaced element from the right -- so it is reproduced with prefix sums.
//             ONE cooperative launch builds the whole tree: the phases of a level are separated by
//             grid-wide barriers, the level loop runs on the device, and the kernel returns at once
//             when its gate (the number of flagged queries) is zero -- no host synchronisation.
//   search  : findNeighbors / searchLevel / KNNResultSet (nanoflann.hpp:1394-1418, :1545-1624,
//             :157-230) with an explicit stack; one thread per flagged query.
//
// The build only does work when at least one query is flagged (uniform random clouds: none for
// k = 1, a handful per million queries for k = 16).
#pragma once
#include <atomic>
#include <cfloat>
#include <cooperative_groups.h>
#include "common.cuh"
#include "grid.cuh"
#include "host_util.h"
#include "../../include/pcu_b200.h"

namespace pcu {

constexpr int kKdItems = 8;                       // slots per thread and scan tile
constexpr int kKdTile = kThreads * kKdItems;      // slots per scan tile
// A node of at most this many points leaves the level-synchronous grid-wide build: its whole subtree is built by
// ONE CTA (block barriers instead of grid barriers, the levels of all such subtrees advance independently).
// Small on purpose: a CTA walks its range with blockDim threads, so the subtrees must be numerous enough to keep as
// many threads busy as the grid-wide passes do (a cap of 8192 leaves only ~128 CTAs for 10^6 points).
constexpr int kKdLocalCap = 1024;

template <typename T>
struct KdNode {
    int feat;            // split dimension; -1 = leaf; -2 = not decided yet; -3 = stub (pruned build: left unsplit);
                         // -4 = root of a subtree handed to one CTA (kKdLocalCap), split in the second phase of the build
    int first, last;     // slot range [first, last) in order[]
    int kid0, kid1;
    int parent;          // parent node (-1 for the root); side: 0 = left child, 1 = right child
    int side;
    int n_less, n_less_eq;
    unsigned mask[4];    // pruned build: bit j set = flagged query j may walk into this node (all ones otherwise)
    T cut;
    T div_lo, div_hi;
    T loose_lo[3], loose_hi[3];
    typename Real<T>::bits_t tight_lo[3], tight_hi[3];   // order-preserving integer images (atomics)
};

struct KdCounters {
    int n_nodes;        // nodes allocated so far
    int level_begin;    // first node id of the current level
    int level_end;      // one past the last node id of the current level
    int n_split;        // nodes of the current level that were split
    int done;           // set when a level split nothing
    int levels;         // levels processed (diagnostic)
    int any_eq;         // current level: some live point equals its node's cut (sweep 2 has work to do)
    int n_local;        // subtree roots handed to single CTAs so far (KdReplayBuffers::local_roots)
};

// How a pass reads the flag prefix sums: the grid-wide phases store in-tile prefixes plus tile offsets over all
// slots; a CTA building a subtree stores absolute prefixes over its own slot range [.., range_end) and keeps the
// grand total ("the prefix at range_end", a slot that belongs to the neighbouring subtree) to itself.
struct KdScope {
    bool local;
    int range_end;
    unsigned total;
    const unsigned* tile_off;   // grid-wide phases: the tile offsets in THIS CTA's shared memory (null: in scan_partial)
};
constexpr int kKdSharedTiles = 4096;   // tile offsets a CTA keeps to itself (clouds up to kKdTile * 4096 = 8.4 M points)

template <typename T>
struct KdReplayBuffers {
    long long capacity = 0;   // points
    int* order = nullptr;
    int* node_of = nullptr;
    unsigned* prefix = nullptr;       // capacity + 1
    unsigned* scan_partial = nullptr;
    int* left_pos = nullptr;
    int* right_pos = nullptr;
    KdNode<T>* nodes = nullptr;       // 2 * capacity
    KdCounters* counters = nullptr;
    int* local_roots = nullptr;       // capacity: nodes whose subtrees single CTAs build
    int* level_lists = nullptr;       // 2 * capacity: per subtree, the node ids of the current / the next level (in its slot range)
    unsigned* stub_hits = nullptr;    // searches that ran into a stub of the pruned build (-> full rebuild)
    unsigned* overflows = nullptr;    // searches whose walk was deeper than kKdStack (adversarially deep trees): reported
    long long* one_row = nullptr;     // scratch for the single-query (witness) replay
    T* one_dist = nullptr;
    long long* one_idx = nullptr;

    void carve(Carver& cv, long long points) {
        capacity = points;
        order = cv.take<int>((size_t)points);
        node_of = cv.take<int>((size_t)points);
        prefix = cv.take<unsigned>((size_t)points + 1);
        scan_partial = cv.take<unsigned>(((size_t)points + 1 + kKdTile - 1) / kKdTile + 1);
        left_pos = cv.take<int>((size_t)points);
        right_pos = cv.take<int>((size_t)points);
        nodes = cv.take<KdNode<T>>((size_t)2 * points + 2);
        counters = cv.take<KdCounters>(1);
        local_roots = cv.take<int>((size_t)points);
        level_lists = cv.take<int>((size_t)2 * points);
        stub_hits = cv.take<unsigned>(1);
        overflows = cv.take<unsigned>(1);
        one_row = cv.take<long long>(1);
        one_dist = cv.take<T>(1);
        one_idx = cv.take<long long>(1);
    }
};

__global__ void widen_counter_kernel(const unsigned* src, long long* dst) { *dst = (long long)*src; }

// ---- build -----------------------------------------------------------------------------------------
// tight bounding box contribution of slot s to its node (atomics on the ordered integer image; a warp
// whose lanes all sit in the same node reduces first).  Called by whole warps.
template <typename T>
__device__ __forceinline__ void kd_tight_box_slot(const KdReplayBuffers<T>& b, const T* __restrict__ pts, int s, int m) {
    using bits_t = typename Real<T>::bits_t;
    const int node = s < m ? b.node_of[s] : -1;
    bits_t v[3] = {0, 0, 0};
    if (node >= 0) {
        const long long p = b.order[s];
        for (int d = 0; d < 3; ++d) v[d] = ordered<T>(pts[3 * p + d]);
    }
    const int lead = __shfl_sync(0xffffffffu, node, 0);
    const bool uniform = __all_sync(0xffffffffu, node == lead);
    if (uniform) {
        if (lead < 0) return;
        bits_t lo[3], hi[3];
        for (int d = 0; d < 3; ++d) {
            lo[d] = hi[d] = v[d];
            for (int o = 16; o > 0; o >>= 1) {
                const bits_t a = __shfl_xor_sync(0xffffffffu, lo[d], o), c = __shfl_xor_sync(0xffffffffu, hi[d], o);
                lo[d] = a < lo[d] ? a : lo[d];
                hi[d] = c > hi[d] ? c : hi[d];
            }
        }
        if ((threadIdx.x & 31) == 0)
            for (int d = 0; d < 3; ++d) { atomicMin(&b.nodes[lead].tight_lo[d], lo[d]); atomicMax(&b.nodes[lead].tight_hi[d], hi[d]); }
    } else if (node >= 0) {
        for (int d = 0; d < 3; ++d) { atomicMin(&b.nodes[node].tight_lo[d], v[d]); atomicMax(&b.nodes[node].tight_hi[d], v[d]); }
    }
}

// Pruned build.  The tree is only needed by the handful of flagged queries, and a query's walk only
// enters a far child whose bound (searchLevel's mindistsq, nanoflann.hpp:1600-1612) is at most the
// current k-th distance.  That distance is never below its final value d_k -- which the grid search
// already knows -- and exceeds it only early in the walk, deep in the tree.  So a node that is the FAR
// child of its parent for every flagged query that can reach the parent, with a bound above
// slack * d_k^2 (slack = 4), is left as an unsplit stub (its slots retire like a leaf's), unless it is small.
// This is a heuristic, not a proof: a walk that does run into a stub reports it (kd_search_one returns
// false) and the caller rebuilds the full tree for that call, so results never depend on the pruning.
constexpr int kKdMaskWords = 4;
constexpr int kKdMaxPruneQueries = 64;   // one mask bit per flagged query (at most 32 * kKdMaskWords); more -> full build:
                                         // the walks of that many flagged rows reach most of the tree anyway
constexpr int kKdSmallNode = 256;        // nodes up to this many points always follow their parent

template <typename T>
struct KdPrune {
    const T* query = nullptr;           // the call's query cloud
    const long long* rows = nullptr;    // flagged rows
    const unsigned* n_rows = nullptr;
    const T* kth = nullptr;             // the call's distance output, k per row (the fast answer's distances are final)
    int k = 0;
    int squared = 0;
    int enabled = 0;
    float slack = 4.f;                  // 0 (diagnostic): every far child is a stub, which forces the full-rebuild path
};

// (bound, per-axis offsets) searchLevel holds on arrival at `target` for query q; false if the node
// is deeper than the walk stack (then the caller keeps the node).
template <typename T>
__device__ bool kd_arrival_state(const KdReplayBuffers<T>& b, int target, const T q[3], T& bound, T off[3]) {
    using R = Real<T>;
    int chain[96];
    int depth = 0;
    for (int a = target; a >= 0; a = b.nodes[a].parent) {
        if (depth == 96) return false;
        chain[depth++] = a;
    }
    const KdNode<T>& root = b.nodes[chain[depth - 1]];
    bound = (T)0;
    for (int d = 0; d < 3; ++d) {
        off[d] = (T)0;
        const T lo = unordered<T>(root.tight_lo[d]), hi = unordered<T>(root.tight_hi[d]);
        if (q[d] < lo) { off[d] = sq_gap<T>(q[d], lo); bound = R::add(bound, off[d]); }
        if (q[d] > hi) { off[d] = sq_gap<T>(q[d], hi); bound = R::add(bound, off[d]); }
    }
    for (int i = depth - 1; i > 0; --i) {
        const KdNode<T>& nd = b.nodes[chain[i]];
        const int ft = nd.feat;
        const T v = q[ft];
        const bool left_near = R::add(R::sub(v, nd.div_lo), R::sub(v, nd.div_hi)) < (T)0;
        if (chain[i - 1] != (left_near ? nd.kid0 : nd.kid1)) {
            const T cut = left_near ? sq_gap<T>(v, nd.div_hi) : sq_gap<T>(v, nd.div_lo);
            bound = R::sub(R::add(bound, cut), off[ft]);
            off[ft] = cut;
        }
    }
    return true;
}

// Which flagged queries may walk into node `id` (a child whose tight box and whose sibling's are final).
// Writes the node's mask; returns whether any bit is set.
template <typename T>
__device__ bool kd_node_mask(const KdReplayBuffers<T>& b, const KdPrune<T>& pr, int id) {
    using R = Real<T>;
    KdNode<T>& nd = b.nodes[id];
    const KdNode<T>& par = b.nodes[nd.parent];
    if (nd.last - nd.first <= kKdSmallNode) {
        unsigned any = 0u;
        for (int w = 0; w < kKdMaskWords; ++w) { nd.mask[w] = par.mask[w]; any |= par.mask[w]; }
        return any != 0u;
    }
    const int ft = par.feat;
    const T div_lo = unordered<T>(b.nodes[par.kid0].tight_hi[ft]);   // what the two children hand up (divlow / divhigh)
    const T div_hi = unordered<T>(b.nodes[par.kid1].tight_lo[ft]);
    unsigned any = 0u;
    for (int w = 0; w < kKdMaskWords; ++w) {
        unsigned mask = 0u;
        for (unsigned rest = par.mask[w]; rest != 0u; rest &= rest - 1u) {
            const int bit = __ffs((int)rest) - 1;
            const long long row = pr.rows[32 * w + bit];
            const T q[3] = {pr.query[3 * row], pr.query[3 * row + 1], pr.query[3 * row + 2]};
            const T v = q[ft];
            const bool left_near = R::add(R::sub(v, div_lo), R::sub(v, div_hi)) < (T)0;
            if (left_near == (nd.side == 0)) { mask |= 1u << bit; continue; }     // near child: entered whenever the parent is
            const T kth = pr.kth[row * pr.k + pr.k - 1];
            if (kth < (T)0) { mask |= 1u << bit; continue; }                     // fewer than k points in the cloud: everything is visited
            const T limit = R::mul(pr.squared ? kth : R::mul(kth, kth), (T)pr.slack);
            T bound, off[3];
            if (!kd_arrival_state<T>(b, nd.parent, q, bound, off)) { mask |= 1u << bit; continue; }
            const T cut = left_near ? sq_gap<T>(v, div_hi) : sq_gap<T>(v, div_lo);
            if (R::sub(R::add(bound, cut), off[ft]) <= limit) mask |= 1u << bit;
        }
        nd.mask[w] = mask;
        any |= mask;
    }
    return any != 0u;
}

// leaf-or-split decision + split plane of one node; also hands this node's tight extent along the
// parent's split axis up to the parent (divlow / divhigh, nanoflann.hpp:1047-1048).
template <typename T>
__device__ __forceinline__ void kd_decide_node(const KdReplayBuffers<T>& b, int id, int leaf_cap, const KdPrune<T>& pr, unsigned n_flagged,
                                               bool may_hand_off) {
    using R = Real<T>;
    KdNode<T>& nd = b.nodes[id];
    T tlo[3], thi[3];
    for (int d = 0; d < 3; ++d) { tlo[d] = unordered<T>(nd.tight_lo[d]); thi[d] = unordered<T>(nd.tight_hi[d]); }
    if (nd.parent >= 0) {
        KdNode<T>& par = b.nodes[nd.parent];
        if (nd.side == 0) par.div_lo = thi[par.feat]; else par.div_hi = tlo[par.feat];
    } else {
        for (int d = 0; d < 3; ++d) { nd.loose_lo[d] = tlo[d]; nd.loose_hi[d] = thi[d]; }  // root: computeBoundingBox
    }
    // n_flagged == 0: full build (every mask all ones); otherwise bit j < n_flagged stands for flagged row j
    bool wanted = true;
    if (n_flagged == 0u) {
        for (int w = 0; w < kKdMaskWords; ++w) nd.mask[w] = 0xffffffffu;
    } else if (nd.parent < 0) {
        for (int w = 0; w < kKdMaskWords; ++w)
            nd.mask[w] = n_flagged >= 32u * (w + 1) ? 0xffffffffu : (n_flagged > 32u * w ? (1u << (n_flagged - 32u * w)) - 1u : 0u);
    } else {
        wanted = kd_node_mask<T>(b, pr, id);
    }
    const int count = nd.last - nd.first;
    if (count <= leaf_cap) { nd.feat = -1; return; }
    if (!wanted) { nd.feat = -3; return; }   // no flagged query comes here: stub
    if (may_hand_off && count <= kKdLocalCap) {   // small enough: one CTA builds the whole subtree later
        nd.feat = -4;
        b.local_roots[atomicAdd(&b.counters->n_local, 1)] = id;
        return;
    }
    // middleSplit_ (nanoflann.hpp:1061-1096)
    const T eps = (T)0.00001;
    T widest = R::sub(nd.loose_hi[0], nd.loose_lo[0]);
    for (int d = 1; d < 3; ++d) {
        const T w = R::sub(nd.loose_hi[d], nd.loose_lo[d]);
        if (w > widest) widest = w;
    }
    const T gate = R::mul(R::sub((T)1, eps), widest);
    T best_spread = (T)-1;
    int feat = 0;
    for (int d = 0; d < 3; ++d) {
        const T w = R::sub(nd.loose_hi[d], nd.loose_lo[d]);
        if (w > gate) {
            const T spread = R::sub(thi[d], tlo[d]);
            if (spread > best_spread) { feat = d; best_spread = spread; }
        }
    }
    const T mid = R::mul(R::add(nd.loose_lo[feat], nd.loose_hi[feat]), (T)0.5);
    T cut;
    if (mid < tlo[feat]) cut = tlo[feat];
    else if (mid > thi[feat]) cut = thi[feat];
    else cut = mid;
    nd.feat = feat;
    nd.cut = cut;
}

// sweep 1: flag = (value < cut); sweep 2: flag = (value <= cut) on the part right of n_less.
// Bit 0 of the result is the flag; in sweep 1, bit 1 says that the value EQUALS the cut (only then does
// sweep 2 have anything to move, see kd_build_kernel).
template <typename T, int kSweep>
__device__ __forceinline__ unsigned kd_flag(const KdReplayBuffers<T>& b, const T* __restrict__ pts, int s, int m) {
    if (s >= m) return 0u;    // entry m is the sentinel that carries the grand total
    const int node = b.node_of[s];
    if (node < 0) return 0u;
    const KdNode<T>& nd = b.nodes[node];
    if (nd.feat < 0) return 0u;
    const T v = pts[3 * (long long)b.order[s] + nd.feat];
    if (kSweep == 1) return (v < nd.cut ? 1u : 0u) | (v == nd.cut ? 2u : 0u);
    return (s >= nd.first + nd.n_less && v <= nd.cut) ? 1u : 0u;
}

// exclusive prefix of the flags at slot s: in-tile prefix + offset of the tile
template <typename T>
__device__ __forceinline__ unsigned kd_prefix(const KdReplayBuffers<T>& b, int s, const KdScope& sc) {
    if (sc.local) return s == sc.range_end ? sc.total : b.prefix[s];
    return b.prefix[s] + (sc.tile_off != nullptr ? sc.tile_off[s / kKdTile] : b.scan_partial[s / kKdTile]);
}

// Who trades places with whom (nanoflann.hpp:1125-1160): inside a node, with F = number of flagged
// slots of the swept range [lo, last), the flagged slots must end up in [lo, lo + F).  The j-th
// unflagged slot of [lo, lo + F) (ascending) exchanges with the j-th flagged slot of [lo + F, last)
// (descending).
template <typename T, int kSweep>
__device__ __forceinline__ void kd_partner_slot(const KdReplayBuffers<T>& b, int s, const KdScope& sc) {
    const int node = b.node_of[s];
    if (node < 0) return;
    const KdNode<T>& nd = b.nodes[node];
    if (nd.feat < 0) return;
    const int lo = kSweep == 1 ? nd.first : nd.first + nd.n_less;
    const unsigned at_lo = kd_prefix<T>(b, lo, sc), at_last = kd_prefix<T>(b, nd.last, sc);
    const int F = (int)(at_last - at_lo);   // (kd_children_node, in the same phase, stores it as n_less / n_less_eq)
    if (s < lo) return;
    const unsigned here = kd_prefix<T>(b, s, sc), next = kd_prefix<T>(b, s + 1, sc);
    const bool flagged = next != here;
    const int r = s - lo;
    if (r < F && !flagged) b.left_pos[lo + (r - (int)(here - at_lo))] = s;
    else if (r >= F && flagged) b.right_pos[lo + (int)(at_last - next)] = s;
}

template <typename T, int kSweep>
__device__ __forceinline__ void kd_exchange_slot(const KdReplayBuffers<T>& b, int s, const KdScope& sc) {
    const int node = b.node_of[s];
    if (node < 0) return;
    const KdNode<T>& nd = b.nodes[node];
    if (nd.feat < 0) return;
    // n_less / n_less_eq were stored by the partner phase
    const int lo = kSweep == 1 ? nd.first : nd.first + nd.n_less;
    if (s < lo) return;
    const int F = kSweep == 1 ? nd.n_less : nd.n_less_eq - nd.n_less;
    const int misplaced = F - (int)(kd_prefix<T>(b, lo + F, sc) - kd_prefix<T>(b, lo, sc));   // unflagged slots inside [lo, lo + F)
    const int j = s - lo;
    if (j >= misplaced) return;
    const int a = b.left_pos[lo + j], c = b.right_pos[lo + j];
    const int t = b.order[a];
    b.order[a] = b.order[c];
    b.order[c] = t;
}

// children of one split node (nanoflann.hpp:1098-1110, :1033-1045)
// Runs in the partner phase of sweep kSweep (the prefix sums of that sweep are final, nobody reads n_less_eq and
// only sweep 2 reads n_less, which sweep 1 left): stores the sweep's counts -- what planeSplit returns as lim1 / lim2 --
// and, when this is the node's last sweep (`create`), allocates the two children.
template <typename T, int kSweep>
__device__ __forceinline__ void kd_children_node(const KdReplayBuffers<T>& b, int id, const KdScope& sc, bool create,
                                                 int* next_list = nullptr, int* next_count = nullptr) {
    using R = Real<T>;
    KdNode<T>& nd = b.nodes[id];
    if (nd.feat < 0) return;
    {
        const int lo = kSweep == 1 ? nd.first : nd.first + nd.n_less;
        const int F = (int)(kd_prefix<T>(b, nd.last, sc) - kd_prefix<T>(b, lo, sc));
        if (kSweep == 1) { nd.n_less = F; nd.n_less_eq = F; }   // sweep 2, when it runs, overwrites n_less_eq
        else nd.n_less_eq = nd.n_less + F;
    }
    if (!create) return;
    const int count = nd.last - nd.first;
    int left;
    if (nd.n_less > count / 2) left = nd.n_less;
    else if (nd.n_less_eq < count / 2) left = nd.n_less_eq;
    else left = count / 2;
    const int k0 = atomicAdd(&b.counters->n_nodes, 2);
    if (next_list == nullptr) atomicAdd(&b.counters->n_split, 1);
    else {   // a CTA building a subtree keeps its own list of the next level's nodes (shared-memory counter)
        const int at = atomicAdd(next_count, 2);
        next_list[at] = k0; next_list[at + 1] = k0 + 1;
    }
    nd.kid0 = k0; nd.kid1 = k0 + 1;
    for (int side = 0; side < 2; ++side) {
        KdNode<T> ch{};
        ch.feat = -2;
        ch.first = side == 0 ? nd.first : nd.first + left;
        ch.last = side == 0 ? nd.first + left : nd.last;
        ch.kid0 = ch.kid1 = -1; ch.parent = id; ch.side = side;
        for (int d = 0; d < 3; ++d) {
            ch.loose_lo[d] = nd.loose_lo[d]; ch.loose_hi[d] = nd.loose_hi[d];
            ch.tight_lo[d] = ordered<T>(R::inf()); ch.tight_hi[d] = ordered<T>(-R::inf());
        }
        if (side == 0) ch.loose_hi[nd.feat] = nd.cut; else ch.loose_lo[nd.feat] = nd.cut;
        b.nodes[k0 + side] = ch;
    }
}

// One flag-and-scan phase of the cooperative build: in-tile exclusive prefixes + tile totals, then
// (after a grid barrier) the first CTA turns the totals into tile offsets.
template <typename T, int kSweep>
__device__ __forceinline__ void kd_scan_phase(cooperative_groups::grid_group& grid, const KdReplayBuffers<T>& b,
                                              const T* __restrict__ pts, int m, unsigned* tile_off) {
    const int count = m + 1;
    const int ntiles = (count + kKdTile - 1) / kKdTile;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int first = tile * kKdTile + threadIdx.x * kKdItems;
        unsigned v[kKdItems];
        unsigned sum = 0, eq = 0;
#pragma unroll
        for (int k = 0; k < kKdItems; ++k) {
            const unsigned r = (first + k) < count ? kd_flag<T, kSweep>(b, pts, first + k, m) : 0u;
            v[k] = r & 1u; eq |= r >> 1; sum += v[k];
        }
        if (kSweep == 1 && __syncthreads_or((int)eq) && threadIdx.x == 0) atomicOr(&b.counters->any_eq, 1);
        unsigned total;
        unsigned run = block_exclusive_scan<kThreads>(sum, &total);
#pragma unroll
        for (int k = 0; k < kKdItems; ++k) {
            if ((first + k) < count) b.prefix[first + k] = run;
            run += v[k];
        }
        if (threadIdx.x == 0) b.scan_partial[tile] = total;
    }
    grid.sync();
    if (tile_off != nullptr) {
        // every CTA turns the tile totals into offsets for itself (shared memory): no serial CTA, no second barrier
        constexpr int kPer = kKdSharedTiles / kThreads;
        unsigned v[kPer];
        unsigned sum = 0;
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int i = threadIdx.x * kPer + k;
            v[k] = i < ntiles ? b.scan_partial[i] : 0u;
            sum += v[k];
        }
        unsigned total;
        unsigned run = block_exclusive_scan<kThreads>(sum, &total);
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int i = threadIdx.x * kPer + k;
            if (i < ntiles) tile_off[i] = run;
            run += v[k];
        }
        __syncthreads();
        return;
    }
    if (blockIdx.x == 0) {
        unsigned carry = 0;
        for (int base = 0; base < ntiles; base += kThreads) {
            const int i = base + threadIdx.x;
            const unsigned v = i < ntiles ? b.scan_partial[i] : 0u;
            unsigned total;
            const unsigned ex = block_exclusive_scan<kThreads>(v, &total);
            if (i < ntiles) b.scan_partial[i] = carry + ex;
            carry += total;
        }
    }
    grid.sync();
}

// One flag-and-scan phase of a CTA building a subtree: absolute exclusive prefixes over the slots [first, last);
// the grand total stays in shared memory (KdScope::total).  Block-wide.
template <typename T, int kSweep>
__device__ __forceinline__ void kd_scan_subtree(const KdReplayBuffers<T>& b, const T* __restrict__ pts, int first, int last,
                                                unsigned* s_total, int* s_any_eq) {
    unsigned carry = 0;
    for (int base = first; base < last; base += kKdTile) {
        const int at = base + threadIdx.x * kKdItems;
        unsigned v[kKdItems];
        unsigned sum = 0, eq = 0;
#pragma unroll
        for (int k = 0; k < kKdItems; ++k) {
            const unsigned r = (at + k) < last ? kd_flag<T, kSweep>(b, pts, at + k, last) : 0u;
            v[k] = r & 1u; eq |= r >> 1; sum += v[k];
        }
        if (kSweep == 1 && eq) *s_any_eq = 1;   // benign race: every writer stores 1
        unsigned total;
        unsigned run = carry + block_exclusive_scan<kThreads>(sum, &total);
#pragma unroll
        for (int k = 0; k < kKdItems; ++k) {
            if ((at + k) < last) b.prefix[at + k] = run;
            run += v[k];
        }
        carry += total;
    }
    if (threadIdx.x == 0) *s_total = carry;
    __syncthreads();
}

// The whole subtree below `root` (a node the grid-wide phase handed off: feat == -4, at most kKdLocalCap slots),
// built level by level by ONE CTA with the very passes of the grid-wide build, over the subtree's own slot range,
// separated by block barriers.  The node ids of a level live in the subtree's part of level_lists.
template <typename T>
__device__ void kd_build_subtree(const KdReplayBuffers<T>& b, const T* __restrict__ pts, int root, int leaf_cap,
                                 const KdPrune<T>& pr, unsigned n_flagged) {
    __shared__ int s_count[2];       // nodes in the current / the next level
    __shared__ int s_any_eq;
    __shared__ unsigned s_total;
    const int first = b.nodes[root].first, last = b.nodes[root].last;
    int* cur = b.level_lists + first;
    int* nxt = b.level_lists + b.capacity + first;
    const int warp_first = first & ~31;   // whole warps take part in the tight-box reduction
    __syncthreads();                  // the previous subtree of this CTA is finished with the shared variables
    if (threadIdx.x == 0) { cur[0] = root; s_count[0] = 1; s_count[1] = 0; b.nodes[root].feat = -2; }
    for (int s = first + threadIdx.x; s < last; s += blockDim.x) b.node_of[s] = root;   // the grid phase had retired them
    __syncthreads();
    for (int level = 0; level < 4096; ++level) {
        const int ncur = s_count[0];
        if (ncur == 0) break;
        if (threadIdx.x == 0) s_any_eq = 0;
        for (int i = threadIdx.x; i < ncur; i += blockDim.x) kd_decide_node<T>(b, cur[i], leaf_cap, pr, n_flagged, false);
        __syncthreads();
        kd_scan_subtree<T, 1>(b, pts, first, last, &s_total, &s_any_eq);
        KdScope sc{true, last, s_total, nullptr};
        const bool second = s_any_eq != 0;   // stable: last written before the barrier that ended the scan
        for (int s = first + threadIdx.x; s < last; s += blockDim.x) kd_partner_slot<T, 1>(b, s, sc);
        for (int i = threadIdx.x; i < ncur; i += blockDim.x) kd_children_node<T, 1>(b, cur[i], sc, !second, nxt, &s_count[1]);
        __syncthreads();
        for (int s = first + threadIdx.x; s < last; s += blockDim.x) kd_exchange_slot<T, 1>(b, s, sc);
        __syncthreads();
        if (second) {
            kd_scan_subtree<T, 2>(b, pts, first, last, &s_total, &s_any_eq);
            sc.total = s_total;
            for (int s = first + threadIdx.x; s < last; s += blockDim.x) kd_partner_slot<T, 2>(b, s, sc);
            for (int i = threadIdx.x; i < ncur; i += blockDim.x) kd_children_node<T, 2>(b, cur[i], sc, true, nxt, &s_count[1]);
            __syncthreads();
            for (int s = first + threadIdx.x; s < last; s += blockDim.x) kd_exchange_slot<T, 2>(b, s, sc);
            __syncthreads();
        }
        for (int s = warp_first + threadIdx.x; s < ((last + 31) & ~31); s += blockDim.x) {
            const bool mine = s >= first && s < last;
            if (mine) {
                const int node = b.node_of[s];
                if (node >= 0) {
                    const KdNode<T>& nd = b.nodes[node];
                    b.node_of[s] = nd.feat < 0 ? -1 : (s < b.nodes[nd.kid0].last ? nd.kid0 : nd.kid1);
                }
            }
            kd_tight_box_slot<T>(b, pts, mine ? s : last, last);   // slots outside the range take no part
        }
        // the tight boxes were updated by atomics (performed at L2); the device-scope fence also drops the stale copies
        // of those node records from this SM's L1 before the next level's decide reads them with plain loads
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) { s_count[0] = s_count[1]; s_count[1] = 0; }
        int* t = cur; cur = nxt; nxt = t;
        __syncthreads();
    }
}

// Diagnostics: globaltimer stamps of the last build (ns): [0] start, [1] after the set-up, [2 + l] after grid-wide
// level l (l < 28), [30] end of the grid-wide phase, [31] the last CTA's end of the second phase, [32] grid-wide levels,
// [33] handed-off subtrees.  Read with pcu_b200_debug_kd_times.
__device__ unsigned long long g_kd_times[40];
__device__ __forceinline__ unsigned long long kd_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// The whole build in one cooperative launch.  `gate` (may be null): device counter; when it reads
// zero nobody needs the tree and every CTA returns immediately.
template <typename T>
__global__ void __launch_bounds__(kThreads, (sizeof(T) == 4 ? 6 : 4)) kd_build_kernel(KdReplayBuffers<T> b, const T* __restrict__ pts, int m,
                                                            int leaf_cap, const unsigned* __restrict__ gate, KdPrune<T> pr) {
    namespace cg = cooperative_groups;
    using R = Real<T>;
    const unsigned gate_value = gate != nullptr ? *gate : 1u;
    // the pruned build opens a call's replay: it clears the stub counter (even when it has nothing to do)
    if (pr.enabled && blockIdx.x == 0 && threadIdx.x == 0) *b.stub_hits = 0u;
    if (gate != b.stub_hits && blockIdx.x == 0 && threadIdx.x == 0) *b.overflows = 0u;   // first build of a replay
    if (gate_value == 0u) return;   // uniform over the grid
    unsigned n_flagged = 0u;   // 0: full build
    if (pr.enabled) {
        const unsigned nt = *pr.n_rows;
        if (nt <= (unsigned)kKdMaxPruneQueries) n_flagged = nt;
    }
    cg::grid_group grid = cg::this_grid();
    __shared__ unsigned s_tile_off[kKdSharedTiles];
    unsigned* const tile_off = (m + 1 + kKdTile - 1) / kKdTile <= kKdSharedTiles ? s_tile_off : nullptr;
    const KdScope grid_scope{false, 0, 0u, tile_off};
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
    const int gsize = gridDim.x * blockDim.x;
    const int m_warp = (m + 31) & ~31;            // whole warps take part in the tight-box reduction

    for (int s = gtid; s < m; s += gsize) { b.order[s] = s; b.node_of[s] = 0; }
    if (gtid == 0) {
        g_kd_times[0] = kd_now(); g_kd_times[31] = 0ull;
        KdNode<T> nd{};
        nd.feat = -2; nd.first = 0; nd.last = m; nd.kid0 = nd.kid1 = -1; nd.parent = -1; nd.side = 0;
        for (int d = 0; d < 3; ++d) { nd.tight_lo[d] = ordered<T>(R::inf()); nd.tight_hi[d] = ordered<T>(-R::inf()); }
        b.nodes[0] = nd;
        KdCounters c{}; c.n_nodes = 1; c.level_begin = 0; c.level_end = 1;
        *b.counters = c;
    }
    grid.sync();
    for (int s = gtid; s < m_warp; s += gsize) kd_tight_box_slot<T>(b, pts, s, m);
    grid.sync();
    if (gtid == 0) g_kd_times[1] = kd_now();

    for (int level = 0; level < 4096; ++level) {
        const int lb = *(volatile int*)&b.counters->level_begin, le = *(volatile int*)&b.counters->level_end;
        for (int id = lb + gtid; id < le; id += gsize) kd_decide_node<T>(b, id, leaf_cap, pr, n_flagged, true);
        grid.sync();
        // sweep 1: strictly-less-than-the-cut to the front
        kd_scan_phase<T, 1>(grid, b, pts, m, tile_off);
        const bool second = *(volatile int*)&b.counters->any_eq != 0;
        for (int s = gtid; s < m; s += gsize) kd_partner_slot<T, 1>(b, s, grid_scope);
        for (int id = lb + gtid; id < le; id += gsize) kd_children_node<T, 1>(b, id, grid_scope, !second);
        grid.sync();
        for (int s = gtid; s < m; s += gsize) kd_exchange_slot<T, 1>(b, s, grid_scope);
        grid.sync();
        // sweep 2: equal-to-the-cut next.  planeSplit's second loop (nanoflann.hpp:1143-1158) moves nothing
        // when no point of the node equals the cut (lim2 == lim1); any_eq was raised by sweep 1's scan and
        // is stable since the barrier that ended it, so the whole grid takes the same branch.
        if (second) {
            kd_scan_phase<T, 2>(grid, b, pts, m, tile_off);
            for (int s = gtid; s < m; s += gsize) kd_partner_slot<T, 2>(b, s, grid_scope);
            for (int id = lb + gtid; id < le; id += gsize) kd_children_node<T, 2>(b, id, grid_scope, true);
            grid.sync();
            for (int s = gtid; s < m; s += gsize) kd_exchange_slot<T, 2>(b, s, grid_scope);
            grid.sync();
        }
        // slots move down to the child that now owns them (slots of leaves retire) and immediately
        // contribute to that child's tight box
        for (int s = gtid; s < m_warp; s += gsize) {
            if (s < m) {
                const int node = b.node_of[s];
                if (node >= 0) {
                    const KdNode<T>& nd = b.nodes[node];
                    b.node_of[s] = nd.feat < 0 ? -1 : (s < b.nodes[nd.kid0].last ? nd.kid0 : nd.kid1);
                }
            }
            kd_tight_box_slot<T>(b, pts, s, m);
        }
        if (gtid == 0) {
            KdCounters c = *b.counters;
            c.done = c.n_split == 0;
            c.level_begin = c.level_end;
            c.level_end = c.n_nodes;
            c.n_split = 0;
            c.levels = level + 1;
            c.any_eq = 0;
            *b.counters = c;
        }
        grid.sync();
        if (gtid == 0 && level < 28) g_kd_times[2 + level] = kd_now();
        if (*(volatile int*)&b.counters->done) break;
    }
    // second phase: the subtrees handed off above, one CTA each, all of them side by side
    const int n_local = *(volatile int*)&b.counters->n_local;
    if (gtid == 0) { g_kd_times[30] = kd_now(); g_kd_times[32] = (unsigned long long)b.counters->levels; g_kd_times[33] = (unsigned long long)n_local; }
    for (int i = blockIdx.x; i < n_local; i += gridDim.x) kd_build_subtree<T>(b, pts, b.local_roots[i], leaf_cap, pr, n_flagged);
    if (threadIdx.x == 0) atomicMax(&g_kd_times[31], kd_now());
}

// ---- search ---------------------------------------------------------------------------------------
// nanoflann.hpp:157-230 with the list stored in the caller's output row (squared distances while
// searching).
template <typename T>
struct KdBest {
    T* d2; long long* id; int cap; int have;
    __device__ void init(T* d, long long* i, int k) {
        d2 = d; id = i; cap = k; have = 0;
        d2[cap - 1] = sizeof(T) == 4 ? (T)FLT_MAX : (T)DBL_MAX;
    }
    __device__ T worst() const { return d2[cap - 1]; }
    __device__ void offer(T dist, long long index) {
        int i = have;
        for (; i > 0; --i) {
            if (d2[i - 1] > dist) {
                if (i < cap) { d2[i] = d2[i - 1]; id[i] = id[i - 1]; }
            } else break;
        }
        if (i < cap) { d2[i] = dist; id[i] = index; }
        if (have < cap) ++have;
    }
};

constexpr int kKdStack = 96;

// Returns false (and writes nothing) when the walk ran into a stub of the pruned build.
template <typename T>
__device__ bool kd_search_one(const KdReplayBuffers<T>& b, const T* __restrict__ pts, const T q[3], int k, bool squared,
                              T* out_d, long long* out_i) {
    using R = Real<T>;
    // short lists live in (L1-cached) local memory while the tree is walked; long ones in the output row
    T local_d[32];
    long long local_i[32];
    T* work_d = k <= 32 ? local_d : out_d;
    long long* work_i = k <= 32 ? local_i : out_i;
    KdBest<T> best;
    best.init(work_d, work_i, k);
    struct Frame { int node; T bound; T off[3]; bool far; };
    Frame stack[kKdStack];
    int top = 0;
    {   // computeInitialDistances (nanoflann.hpp:1164-1187)
        const KdNode<T>& root = b.nodes[0];
        Frame f; f.node = 0; f.bound = (T)0; f.far = false;
        for (int d = 0; d < 3; ++d) {
            f.off[d] = (T)0;
            const T lo = unordered<T>(root.tight_lo[d]), hi = unordered<T>(root.tight_hi[d]);
            if (q[d] < lo) { f.off[d] = sq_gap<T>(q[d], lo); f.bound = R::add(f.bound, f.off[d]); }
            if (q[d] > hi) { f.off[d] = sq_gap<T>(q[d], hi); f.bound = R::add(f.bound, f.off[d]); }
        }
        stack[top++] = f;
    }
    while (top > 0) {
        Frame f = stack[--top];
        // the far-side test is made when the near side has been searched completely (:1609)
        if (f.far && !(f.bound <= best.worst())) continue;
        for (;;) {
            const KdNode<T>& nd = b.nodes[f.node];
            if (nd.feat == -3) return false;
            if (nd.feat < 0) {
                const T worst_on_entry = best.worst();   // cached for the whole leaf (:1555)
                for (int s = nd.first; s < nd.last; ++s) {
                    const long long p = b.order[s];
                    const T d = dist2<T>(q[0], q[1], q[2], pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
                    if (d < worst_on_entry) best.offer(d, p);
                }
                break;
            }
            const int ft = nd.feat;
            const T v = q[ft];
            const T d1 = R::sub(v, nd.div_lo), d2 = R::sub(v, nd.div_hi);
            int near_kid, far_kid;
            T cut;
            if (R::add(d1, d2) < (T)0) { near_kid = nd.kid0; far_kid = nd.kid1; cut = sq_gap<T>(v, nd.div_hi); }
            else                       { near_kid = nd.kid1; far_kid = nd.kid0; cut = sq_gap<T>(v, nd.div_lo); }
            Frame g = f;
            g.node = far_kid;
            g.bound = R::sub(R::add(f.bound, cut), f.off[ft]);
            g.off[ft] = cut;
            g.far = true;
            if (top < kKdStack) stack[top++] = g;
            else atomicAdd(b.overflows, 1u);   // never silently: the host entry points turn this into an error
            f.node = near_kid;
        }
    }
    for (int c = 0; c < best.have; ++c) {
        out_d[c] = squared ? work_d[c] : R::root(work_d[c]);
        out_i[c] = work_i[c];
    }
    for (int c = best.have; c < k; ++c) { out_d[c] = (T)-1; out_i[c] = -1; }
    return true;
}

// `gate` (may be null): the pass only runs when *gate != 0 (second pass after a full rebuild).
template <typename T>
__global__ void kd_replay_kernel(KdReplayBuffers<T> b, const T* __restrict__ query, const T* __restrict__ pts, int k,
                                 int squared, const long long* __restrict__ rows, const unsigned* __restrict__ n_rows,
                                 T* out_dist, long long* out_idx, const unsigned* __restrict__ gate) {
    if (gate != nullptr && *gate == 0u) return;
    const unsigned n = *n_rows;
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const long long row = rows[t];
        const T q[3] = {query[3 * row], query[3 * row + 1], query[3 * row + 2]};
        if (!kd_search_one<T>(b, pts, q, k, squared != 0, out_dist + row * k, out_idx + row * k) && gate == nullptr)
            atomicAdd(b.stub_hits, 1u);
    }
}

// single query taken from a stats record (the Hausdorff witness)
template <typename T>
__global__ void kd_witness_kernel(KdReplayBuffers<T> b, const T* __restrict__ query, const T* __restrict__ pts,
                                  long long n_queries, pcu_b200_nn_stats* stats) {
    const long long row = stats->argmax_query;
    if (row < 0 || row >= n_queries) { stats->witness_tied = 0; return; }   // a record without a witness
    const T q[3] = {query[3 * row], query[3 * row + 1], query[3 * row + 2]};
    (void)kd_search_one<T>(b, pts, q, 1, true, b.one_dist, b.one_idx);   // full tree: no stubs
    stats->argmax_data = *b.one_idx;
    stats->witness_tied = 0;
}

// ---- host-side sequencing ---------------------------------------------------------------------------
#define KD_LAUNCH(kernel, grid, block, stream, ...)                                   \
    do {                                                                              \
        kernel<<<grid, block, 0, stream>>>(__VA_ARGS__);                              \
        launches.fetch_add(1, std::memory_order_relaxed);                             \
        if (cudaGetLastError() != cudaSuccess) return PCU_B200_CUDA_ERROR;            \
    } while (0)

// Enqueues the build of the reference-tree replica for `pts` (m points): one cooperative launch, no
// host synchronisation.  With a non-null `gate` the kernel is a no-op when *gate == 0.
template <typename T>
int build_kd_replica(KdReplayBuffers<T>& b, const T* pts, long long m_ll, int leaf_cap, const unsigned* gate,
                     KdPrune<T> prune, cudaStream_t stream, std::atomic<long long>& launches) {
    if (m_ll > b.capacity || m_ll >= 0x7fffffffLL) return PCU_B200_INTERNAL;
    int m = (int)m_ll;
    // co-residency limits of the cooperative launch, cached per device (a process may drive several GPUs)
    constexpr int kMaxDevices = 64;
    static std::atomic<int> cached_blocks[kMaxDevices], cached_sms[kMaxDevices];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return PCU_B200_CUDA_ERROR;
    const int slot = dev >= 0 && dev < kMaxDevices ? dev : 0;
    int blocks_per_sm = cached_blocks[slot].load(std::memory_order_acquire), sms = cached_sms[slot].load(std::memory_order_acquire);
    if (blocks_per_sm == 0 || slot != dev) {
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return PCU_B200_CUDA_ERROR;
        int fit = 0;   // (the statics above are per instantiation: fp32 and fp64 builds have their own limits)
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, kd_build_kernel<T>, kThreads, 0) != cudaSuccess) return PCU_B200_CUDA_ERROR;
        blocks_per_sm = std::max(1, std::min(8, fit));   // enough threads to cover the latency of the element passes
        cached_sms[slot].store(sms, std::memory_order_release);
        cached_blocks[slot].store(blocks_per_sm, std::memory_order_release);
    }
    const long long want = (m_ll + kThreads - 1) / kThreads;
    const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>(want, (long long)blocks_per_sm * sms));
    void* args[] = {(void*)&b, (void*)&pts, (void*)&m, (void*)&leaf_cap, (void*)&gate, (void*)&prune};
    if (cudaLaunchCooperativeKernel((void*)kd_build_kernel<T>, dim3(grid), dim3(kThreads), args, 0, stream) != cudaSuccess)
        return PCU_B200_CUDA_ERROR;
    launches.fetch_add(1, std::memory_order_relaxed);
    return PCU_B200_OK;
}

// The same for a tree that already exists (a prepared cloud owns it: pcu_b200_cloud_prepare_knn_*): one launch,
// a no-op when no row was flagged.
template <typename T>
int enqueue_tie_replay_prebuilt(KdReplayBuffers<T>& b, const T* query, const T* dataset, int k, int squared,
                                const long long* tie_list, const unsigned* tie_count, long long max_rows, T* out_dist,
                                long long* out_idx, cudaStream_t stream, std::atomic<long long>& launches) {
    if (cudaMemsetAsync(b.overflows, 0, sizeof(unsigned), stream) != cudaSuccess) return PCU_B200_CUDA_ERROR;
    const unsigned blocks = (unsigned)std::max<long long>(1, std::min<long long>((max_rows + 127) / 128, 1184));
    // (the gate argument only tells the kernel not to count stub hits: a full tree has no stubs)
    KD_LAUNCH(kd_replay_kernel<T>, blocks, 128, stream, b, query, dataset, k, squared, tie_list, tie_count, out_dist, out_idx, tie_count);
    return PCU_B200_OK;
}

// Re-answers the rows listed in tie_list with the reference's own tie order.  Both launches are gated on
// the device-side list length: nothing happens (and nothing synchronises) when no query was flagged.
template <typename T>
int enqueue_tie_replay(KdReplayBuffers<T>& b, const T* query, const T* dataset, long long m, int k, int squared,
                       int leaf_cap, const long long* tie_list, const unsigned* tie_count, long long max_rows,
                       T* out_dist, long long* out_idx, int mode, cudaStream_t stream, std::atomic<long long>& launches) {
    // pass 1: tree pruned to what the flagged queries can reach; pass 2 (device-gated on a walk having hit
    // a stub, which the pruning heuristic makes rare): the full tree, every flagged row again.
    // k = 1 calls (exact ties are rare there and the call is short) skip the pruning and with it the two
    // gated launches of pass 2, which cost ~15 us even when they have nothing to do.
    const bool pruned = mode != 2 && (k > 1 || mode == 3);
    KdPrune<T> prune;
    prune.query = query; prune.rows = tie_list; prune.n_rows = tie_count; prune.kth = out_dist;
    prune.k = k; prune.squared = squared;
    prune.enabled = pruned ? 1 : 0;             // pcu_b200_options::disable_tie_replay: 2 = full trees only
    prune.slack = mode == 3 ? 0.f : 4.f;        // 3 = zero slack (exercises the rebuild path)
    int st = build_kd_replica<T>(b, dataset, m, leaf_cap, tie_count, prune, stream, launches);
    if (st != PCU_B200_OK) return st;
    const unsigned blocks = (unsigned)std::max<long long>(1, std::min<long long>((max_rows + 127) / 128, 1184));
    KD_LAUNCH(kd_replay_kernel<T>, blocks, 128, stream, b, query, dataset, k, squared, tie_list, tie_count, out_dist, out_idx,
              (const unsigned*)nullptr);
    if (!pruned) return PCU_B200_OK;
    st = build_kd_replica<T>(b, dataset, m, leaf_cap, b.stub_hits, KdPrune<T>{}, stream, launches);
    if (st != PCU_B200_OK) return st;
    KD_LAUNCH(kd_replay_kernel<T>, blocks, 128, stream, b, query, dataset, k, squared, tie_list, tie_count, out_dist, out_idx,
              (const unsigned*)b.stub_hits);
    return PCU_B200_OK;
}

// Replays the single query stats->argmax_query (already known to be tie-dependent).
template <typename T>
int enqueue_witness_replay(KdReplayBuffers<T>& b, const T* query, long long n, const T* dataset, long long m, int leaf_cap,
                           pcu_b200_nn_stats* stats, cudaStream_t stream, std::atomic<long long>& launches) {
    const int st = build_kd_replica<T>(b, dataset, m, leaf_cap, nullptr, KdPrune<T>{}, stream, launches);
    if (st != PCU_B200_OK) return st;
    KD_LAUNCH(kd_witness_kernel<T>, 1, 1, stream, b, query, dataset, n, stats);
    return PCU_B200_OK;
}

}  // namespace pcu
