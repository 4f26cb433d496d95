// union_find.cuh -- union-find on int32 parents in global memory, shared by the 3-D flood fill (voxelize.cuh) and the
// mesh connected components (mesh_topology.cuh).  Roots point at themselves; a union points the larger root at the
// smaller one, so every root stays the smallest index of its tree whatever order the unions run in.
#pragma once
#include "common.cuh"

namespace pcu {

// Root of x with path halving: every store points an element at an ancestor, so concurrent unions keep their meaning.
// Parents are read through volatile loads: other threads (other SMs) change them while a union runs.
__device__ __forceinline__ int uf_find(int* P, int x) {
    volatile int* q = P;
    while (true) {
        const int p = q[x];
        if (p == x) return x;
        const int gp = q[p];
        if (gp != p) q[x] = gp;
        x = gp;
    }
}
// Unites the trees of a and b: the larger root is pointed at the smaller one with atomicMin; when that root had
// meanwhile been given another parent, that parent is united with the smaller root in turn.
__device__ __forceinline__ void uf_union(int* P, int a, int b) {
    while (true) {
        a = uf_find(P, a);
        b = uf_find(P, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(&P[a], b);
        if (old == a) return;
        a = old;
    }
}

}  // namespace pcu
