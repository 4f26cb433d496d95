// mesh_query.cu -- mesh sampling and barycentric interpolation, closest points, winding numbers of meshes and oriented
// point clouds, signed distances, rays against meshes and surfels, and the surfel and sphere geometry of point clouds
// (meshsample.cuh, meshquery.cuh, winding.cuh, raycast.cuh): launch sequencing and C entry points.  It owns the tree builder and offers the other mesh families
// (runtime.cuh) the fp64 closest-point tree, the ball tree of restricted Voronoi cells and the sampling CDF's positions.
#include "runtime.cuh"
#include "meshsample.cuh"
#include "winding.cuh"
#include "raycast.cuh"

namespace pcu {

// The CDF, a multi-CTA inclusive scan of the weights in three launches: each CTA sums its tile of kMeshScanTile faces,
// one CTA scans those sums, each CTA rescans its tile from its offset.  `cdf` holds the area bits on entry and C on
// exit (every element is read and rewritten by the same thread).  Integer sums are exact, so the result does not
// depend on how the scan associates them.
__global__ void __launch_bounds__(kMeshScanThreads) mesh_cdf_reduce_kernel(const unsigned long long* __restrict__ cdf, long long m,
                                                                           const MeshScratch* __restrict__ sc,
                                                                           unsigned long long* __restrict__ tile_sum) {
    const double s = mesh_weight_scale(sc->max_bits, m);
    const long long base = (long long)blockIdx.x * kMeshScanTile;
    const int count = (int)(m - base < kMeshScanTile ? m - base : kMeshScanTile);
    unsigned long long sum = 0;
    for (int i = threadIdx.x; i < count; i += kMeshScanThreads) sum += mesh_weight(cdf[base + i], s);
    unsigned long long total;
    block_exclusive_scan<kMeshScanThreads, unsigned long long>(sum, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) mesh_cdf_tiles_kernel(unsigned long long* __restrict__ tile_sum, long long tiles, long long m,
                                                              const MeshScratch* __restrict__ sc, MeshArea* __restrict__ out) {
    const unsigned long long W = block_scan_rounds<1024, unsigned long long>(
        (unsigned)tiles, [&](unsigned b) { return tile_sum[b]; },
        [&](unsigned b, unsigned long long ex, unsigned long long) { tile_sum[b] = ex; });
    if (threadIdx.x == 0) {
        out->total = W;
        out->scale = mesh_weight_scale(sc->max_bits, m);
        out->bad = sc->bad;
    }
}

__global__ void __launch_bounds__(kMeshScanThreads) mesh_cdf_scan_kernel(unsigned long long* __restrict__ cdf, long long m,
                                                                         const MeshScratch* __restrict__ sc,
                                                                         const unsigned long long* __restrict__ tile_offset) {
    const double s = mesh_weight_scale(sc->max_bits, m);
    const long long base = (long long)blockIdx.x * kMeshScanTile;
    const int count = (int)(m - base < kMeshScanTile ? m - base : kMeshScanTile);
    const unsigned long long off = tile_offset[blockIdx.x];
    block_scan_rounds<kMeshScanThreads, unsigned long long>(
        count, [&](int i) { return mesh_weight(cdf[base + i], s); },
        [&](int i, unsigned long long ex, unsigned long long w) { cdf[base + i] = off + ex + w; });
}

__global__ void __launch_bounds__(kThreads) sf_upload_kernel(const SfUpload u) {
    for (int k = threadIdx.x; k < u.count; k += blockDim.x) u.dst[k] = u.v[k];
    if (threadIdx.x == 0 && u.dst_src) *u.dst_src = u.src;
}

// Ball leaf i (i < m - bad): its ball, its face id and its box.
__global__ void __launch_bounds__(kThreads) rv_ball_leaves_kernel(const double* __restrict__ balls, long long m,
                                                                  const MqScratch* __restrict__ sc, const MqRec* __restrict__ sorted,
                                                                  RvBall* __restrict__ leaves, int* __restrict__ ids,
                                                                  MqBox* __restrict__ boxes) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m - (long long)sc->bad) return;
    const long long t = (long long)sorted[i].idx;
    double a[3], b[3], c[3];
    mq_leaf_corners<RvBall, double>(balls, 0, nullptr, 0, t, a, b, c);
    RvBall r;
    r.c[0] = a[0]; r.c[1] = a[1]; r.c[2] = a[2]; r.r = b[0];
    leaves[i] = r;
    ids[i] = (int)t;
    boxes[i] = mq_leaf_box<RvBall, double>(a, b, c);
}

__device__ __forceinline__ int mq_delta(const MqRec* __restrict__ recs, long long n, long long i, unsigned long long ci, long long j) {
    if (j < 0 || j >= n) return -1;
    const unsigned long long cj = recs[j].key[0];
    return ci == cj ? 64 + __clz((int)(i ^ j)) : __clzll((long long)(ci ^ cj));
}

// Karras 2012, internal node i of n - 1 (n = valid leaves); node 0 is the root.
__global__ void __launch_bounds__(kThreads) mq_nodes_kernel(const MqRec* __restrict__ recs, long long m, const MqScratch* __restrict__ sc,
                                                            MqNode* __restrict__ nodes, int* __restrict__ node_parent,
                                                            int* __restrict__ leaf_parent) {
    const long long n = m - (long long)sc->bad;   // < 2^31
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const unsigned long long ci = recs[i].key[0];
    const int d = mq_delta(recs, n, i, ci, i + 1) - mq_delta(recs, n, i, ci, i - 1) >= 0 ? 1 : -1;
    const int dmin = mq_delta(recs, n, i, ci, i - d);
    long long lmax = 2;
    while (mq_delta(recs, n, i, ci, i + lmax * d) > dmin) lmax <<= 1;
    long long l = 0;
    for (long long t = lmax >> 1; t >= 1; t >>= 1)
        if (mq_delta(recs, n, i, ci, i + (l + t) * d) > dmin) l += t;
    const int dnode = mq_delta(recs, n, i, ci, i + l * d);
    long long s = 0;
    for (int k = 1; k < 33; ++k) {                 // t = ceil(l / 2^k) down to 1
        const long long t = (l + (1ll << k) - 1) >> k;
        if (mq_delta(recs, n, i, ci, i + (s + t) * d) > dnode) s += t;
        if (t <= 1) break;
    }
    const int gamma = (int)(i + s * d) + (d < 0 ? -1 : 0);
    const int c0 = (d < 0 ? i - l : i) == gamma ? ~gamma : gamma;             // the range's ends are min / max(i, j)
    const int c1 = (d < 0 ? i : i + l) == gamma + 1 ? ~(gamma + 1) : gamma + 1;
    nodes[i].c0 = c0;
    nodes[i].c1 = c1;
    if (c0 < 0) leaf_parent[~c0] = (int)i; else node_parent[c0] = (int)i;
    if (c1 < 0) leaf_parent[~c1] = (int)i; else node_parent[c1] = (int)i;
}

__device__ __forceinline__ MqBox mq_child_box(const MqNode* nodes, const MqBox* boxes, int c) {
    if (c < 0) return boxes[~c];
    const float4* p = reinterpret_cast<const float4*>(nodes + c);
    const float4 q0 = __ldcg(p), q1 = __ldcg(p + 1), q2 = __ldcg(p + 2);   // written by other threads of this launch
    MqBox b;
    b.lo[0] = fminf(q0.x, q1.z); b.lo[1] = fminf(q0.y, q1.w); b.lo[2] = fminf(q0.z, q2.x);
    b.hi[0] = fmaxf(q0.w, q2.y); b.hi[1] = fmaxf(q1.x, q2.z); b.hi[2] = fmaxf(q1.y, q2.w);
    return b;
}

// One thread per leaf climbs towards the root; at each node the first arrival stops and the second, which finds both
// children's boxes complete, writes them into the node.
__global__ void __launch_bounds__(kThreads) mq_refit_kernel(long long m, const MqScratch* __restrict__ sc, MqNode* nodes,
                                                            const int* __restrict__ node_parent, const int* __restrict__ leaf_parent,
                                                            const MqBox* __restrict__ boxes, int* __restrict__ arrivals) {
    const long long n = m - (long long)sc->bad;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n < 2 || i >= n) return;
    int node = leaf_parent[i];
    while (true) {
        __threadfence();
        if (atomicAdd(&arrivals[node], 1) == 0) return;
        const int c0 = nodes[node].c0, c1 = nodes[node].c1;
        const MqBox b0 = mq_child_box(nodes, boxes, c0), b1 = mq_child_box(nodes, boxes, c1);
        float4* p = reinterpret_cast<float4*>(nodes + node);
        p[0] = make_float4(b0.lo[0], b0.lo[1], b0.lo[2], b0.hi[0]);
        p[1] = make_float4(b0.hi[1], b0.hi[2], b1.lo[0], b1.lo[1]);
        p[2] = make_float4(b1.lo[2], b1.hi[0], b1.hi[1], b1.hi[2]);
        if (node == 0) return;
        node = node_parent[node];
    }
}

}  // namespace pcu

using namespace pcu;
using namespace pcu_internal;

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

namespace {

// ---- mesh sampling and barycentric interpolation (sample_mesh_random / sample_mesh_poisson_disk) -----------------
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

// ---- closest points, winding numbers and signed distances on a mesh or a point cloud (meshquery.cuh, winding.cuh) ----
// The tree over the valid faces, or over the points, built per call by the one builder below, then one traversal per
// query.  The count of faces with a corner out of range lands in *out_bad; the caller reads it (the call's one
// synchronisation) and raises when it is not zero.

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

// The sphere table of DESIGN.md §3, as the reference computes its angles in fp64: t[a] = cos(pi / 2 - a (pi / stacks))
// and t[stacks + 1 + a] = sin of it for a = 0 .. stacks, then cos and sin of b (2 pi / slices) for b = 0 .. slices, from
// the C library.
void sphere_table(int stacks, int slices, double* t) {
    const double stack_step = M_PI / stacks, sector_step = 2 * M_PI / slices;
    for (int a = 0; a <= stacks; ++a) {
        const double angle = M_PI / 2 - a * stack_step;
        t[a] = std::cos(angle);
        t[stacks + 1 + a] = std::sin(angle);
    }
    double* u = t + 2 * ((size_t)stacks + 1);
    for (int b = 0; b <= slices; ++b) {
        const double angle = b * sector_step;
        u[b] = std::cos(angle);
        u[slices + 1 + b] = std::sin(angle);
    }
}

// pointcloud_sphere_geometry: (stacks + 1)(slices + 1) m vertices in T and 2 (stacks - 1) slices m int32 faces.
template <typename T>
int sphere_geometry_device(pcu_b200_workspace* ws, const T* p, const T* r, long long m, int stacks, int slices, T* out_v, int* out_f,
                           cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (m < 0) return fail(PCU_B200_INVALID_ARGUMENT, "sphere geometry: negative point count %lld", m);
    if (stacks < 1 || slices < 1)
        return fail(PCU_B200_INVALID_ARGUMENT, "sphere geometry: num_stacks and num_slices must be at least 1, got %d and %d", stacks, slices);
    const long long V = ((long long)stacks + 1) * ((long long)slices + 1), F = 2 * ((long long)stacks - 1) * slices;
    if (m > 0 && (m >= INT_MAX || V >= INT_MAX || m * V >= INT_MAX))
        return fail(PCU_B200_INVALID_ARGUMENT, "sphere geometry: int32 faces index at most 2^31 - 2 vertices, got %lld points of %lld", m, V);
    if (m > 0 && (!p || !r || !out_v || (F > 0 && !out_f))) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    if (m == 0) return PCU_B200_OK;
    const size_t entries = 2 * ((size_t)stacks + 1) + 2 * ((size_t)slices + 1);
    double* tab = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { tab = cv.take<double>(entries); }));
    std::vector<double> host(entries);
    sphere_table(stacks, slices, host.data());
    PCU_TRY(h2d(ws, tab, host.data(), sizeof(double) * entries, stream));
    const long long nv = m * V, nf = m * F;
    PCU_LAUNCH(sp_geometry_kernel<T>, blocks_for(nv + nf), kThreads, stream, p, r, (const double*)tab, (unsigned)stacks, (unsigned)slices,
               (unsigned)nv, (unsigned)nf, out_v, out_f);
    return PCU_B200_OK;
}

}  // namespace

namespace __attribute__((visibility("hidden"))) pcu_internal {

size_t closest_tree_bytes(long long m) {
    MeshTree<Pt<double>> t;
    return carve_at(nullptr, [&](Carver& cv) { carve_mesh_tree<Pt<double>>(cv, m, false, t); });
}

int build_closest_tree(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind,
                       unsigned long long* out_bad, unsigned char* block, MeshTree<Pt<double>>& tree, cudaStream_t stream) {
    return build_mesh_tree<double>(ws, v, nv, f, m, fkind, false, out_bad, stream, tree, block);
}

int enqueue_closest_points(pcu_b200_workspace* ws, const MeshTree<Pt<double>>& t, long long m, const double* q, long long n,
                           double* out_d, long long* out_fidx, double* out_bc, cudaStream_t stream) {
    PCU_LAUNCH((mq_query_kernel<double>), query_blocks(ws, n), kThreads, stream, q, n, m, (const MqScratch*)t.sc,
               (const MqNode*)t.nodes, (const Pt<double>*)t.leaves, out_d, (void*)out_fidx, 1, out_bc);
    return PCU_B200_OK;
}

int build_ball_tree(pcu_b200_workspace* ws, const double* balls, long long m, MeshTree<RvBall>& tree, cudaStream_t stream) {
    return build_mesh_tree<double, RvBall>(ws, balls, m, nullptr, m, 0, false, nullptr, stream, tree);
}

int sample_mesh_positions(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind, long long n,
                          unsigned seed, double* x, cudaStream_t stream) {
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
}

}  // namespace pcu_internal

extern "C" {

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
int pcu_b200_pointcloud_sphere_geometry_f32(pcu_b200_workspace* ws, const float* p, const float* r, int64_t np, int num_stacks,
                                            int num_slices, float* out_v, int32_t* out_f, void* stream) {
    return sphere_geometry_device<float>(ws, p, r, np, num_stacks, num_slices, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_pointcloud_sphere_geometry_f64(pcu_b200_workspace* ws, const double* p, const double* r, int64_t np, int num_stacks,
                                            int num_slices, double* out_v, int32_t* out_f, void* stream) {
    return sphere_geometry_device<double>(ws, p, r, np, num_stacks, num_slices, out_v, out_f, (cudaStream_t)stream);
}

}  // extern "C"
