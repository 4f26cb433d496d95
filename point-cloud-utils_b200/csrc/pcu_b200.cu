// pcu_b200.cu -- launch sequencing and C entry points of the families not split into files of their own: mesh sampling
// and queries, rays, marching cubes and sparse voxel grids, voxelization, watertight remeshing, mesh topology and
// geometry, and Voronoi cells.  The shared runtime is in runtime.cuh; the nearest-neighbour family is in nearest.cu,
// the point-cloud operations in point_ops.cu.
#include "runtime.cuh"
#include "compact.cuh"
#include "meshsample.cuh"
#include "winding.cuh"
#include "raycast.cuh"
#include "sparse_voxels.cuh"
#include "voxelize.cuh"
#include "watertight.cuh"
#include "mesh_topology.cuh"
#include "orient.cuh"
#include "laplacian.cuh"
#include "voronoi.cuh"
#include "rvd.cuh"

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
// Marching cubes between pcu_b200_marching_cubes_prepare_* and _emit: the inputs, the cube block (case bytes, tile
// offsets, counts; sized by m) and the slot block (run of every slot, vertex id of every run, owner flags; sized by the
// slot count).
struct pcu_b200_marching_cubes : StreamHandle {
    int t_f64 = 0, s_f64 = 0, width = 4;   // coordinates, scalars, bytes per cube index
    const void* scalars = nullptr;
    const void* coords = nullptr;
    const void* idx = nullptr;
    long long n = 0, m = 0;
    double iso = 0.0;                       // T(S(isovalue)), exactly
    long long slots = 0, faces = 0, verts = 0;
    unsigned char* cube_block = nullptr;
    unsigned char* slot_block = nullptr;
    unsigned char* cases = nullptr;
    unsigned* tile_sum = nullptr;
    unsigned long long* tile_slot0 = nullptr;
    unsigned long long* tile_face0 = nullptr;
    McCounts* counts = nullptr;
    unsigned* slot_run = nullptr;
    unsigned* run_vid = nullptr;
    unsigned char* owner = nullptr;
    ~pcu_b200_marching_cubes() { release(cube_block); release(slot_block); }
};
// Voxelization between pcu_b200_voxelize_prepare_* and _emit: the sorted codes, their run heads and the heads' block
// offsets, in one block.
struct pcu_b200_voxelize : StreamHandle {
    long long recs = 0, n = 0;              // accepted (face, voxel) pairs; distinct voxels
    unsigned char* block = nullptr;
    const McRec* sorted = nullptr;
    unsigned char* head = nullptr;
    unsigned* offsets = nullptr;
    ~pcu_b200_voxelize() { release(block); }
};
// Watertight remeshing between pcu_b200_make_mesh_watertight_prepare_* and _emit: the result in one block, vertices in
// fp64 and faces in int32, which emit converts to the input's types.
struct pcu_b200_watertight : StreamHandle {
    int t_f64 = 0, fkind = 0, depth = 0;
    long long nv = 0, nf = 0;
    unsigned char* block = nullptr;
    const double* x = nullptr;
    const int* faces = nullptr;
    ~pcu_b200_watertight() { release(block); }
};
// Connected components between pcu_b200_connected_components_prepare and _emit: int32 labels and counts in one block
// (cv over n = max(f) + 1 vertices, cf over m faces, nv and nf over the k components, sized n).
struct pcu_b200_components : StreamHandle {
    int fkind = 0;
    long long n = 0, m = 0, k = 0;
    unsigned char* block = nullptr;
    const int* cv = nullptr;
    const int* cf = nullptr;
    const int* nv = nullptr;
    const int* nf = nullptr;
    ~pcu_b200_components() { release(block); }
};
// A sparse voxel grid's code set between pcu_b200_sparse_grid_*_prepare and pcu_b200_sparse_grid_emit: the sorted code
// records, their run heads, the heads' block offsets and the count record, in one block.  Prepared from points, by a
// dilation round or from a grid's cube corners; the mode says what emit writes.
struct SvgCounts { long long rows; unsigned long long bad; };
struct pcu_b200_sparse_grid : StreamHandle {
    int mode = 0;                           // SvgMode
    int out_kind = 0;                       // dilation: the grid's index kind; hex mesh: vertices in double (1) or float (0)
    const void* grid = nullptr;             // dilation: the input rows, which emit copies ahead of the new ones
    long long n = 0;                        // input rows (points or voxels)
    long long recs = 0;                     // sorted records
    long long rows = 0;                     // distinct codes: grid rows, new rows or vertices
    SvgPlace place{};
    unsigned char* block = nullptr;
    const McRec* sorted = nullptr;
    unsigned char* head = nullptr;          // nullptr: the records are distinct already (dilation)
    unsigned* offsets = nullptr;
    SvgCounts* counts = nullptr;
    ~pcu_b200_sparse_grid() { release(block); }
};

namespace {

// The input check of every call on a mesh (v, f): sampling, queries, rays, restricted Voronoi.
int mesh_check(const void* v, long long nv, const void* f, long long m, int fkind) {
    if (!v || !f || nv <= 0 || m <= 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements: v and f must have shape (n, 3) and (m, 3) (n, m > 0)");
    if (m > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "mesh sampling: at most 2^31 - 1 faces, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

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
template <typename L>
struct MeshTree {
    MqScratch* sc;
    MqNode* nodes;
    L* leaves;
    WnNode* wn;   // far-field data per node (with `moments` only)
    int* ids;     // surfel leaves: the point id of each leaf
};

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

// ---- marching cubes and the boundary of a sparse voxel grid (sparse_voxels.cuh) ------------------------------------
// Classify + scan, read the counts (first synchronisation), then the slot records, their sort, the runs and the owners'
// vertex ids, and read the vertex count (second synchronisation).
template <typename T, typename S, int W>
int mc_build(pcu_b200_workspace* ws, pcu_b200_marching_cubes* h, cudaStream_t stream) {
    const long long m = h->m;
    const unsigned tiles = blocks_for(m);
    PCU_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(McCounts), stream));
    PCU_LAUNCH((mc_classify_kernel<T, S, W>), tiles, kThreads, stream, (const S*)h->scalars, h->n, h->idx, m, (T)h->iso,
               h->cases, h->tile_sum, h->counts);
    PCU_LAUNCH(mc_tiles_kernel, 1, 1024, stream, (const unsigned*)h->tile_sum, (long long)tiles, h->tile_slot0, h->tile_face0, h->counts);
    McCounts c;
    PCU_TRY(read_record(h->counts, &c, stream));
    if (c.bad) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid cube_indices: %llu cubes have a corner outside [0, %lld)", c.bad, h->n);
    if (c.slots >= (1ull << 32))
        return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: at most 2^32 - 1 crossing edges are supported, got %llu", c.slots);
    h->slots = (long long)c.slots;
    h->faces = (long long)c.faces;
    const long long ns = h->slots;
    if (ns == 0) return PCU_B200_OK;
    PCU_TRY(alloc_block(h->slot_block, carve_at(nullptr, [&](Carver& cv) {
        cv.take<unsigned>((size_t)ns); cv.take<unsigned>((size_t)ns); cv.take<unsigned char>((size_t)ns); }), stream, "marching cubes"));
    carve_at(h->slot_block, [&](Carver& cv) {
        h->slot_run = cv.take<unsigned>((size_t)ns);
        h->run_vid = cv.take<unsigned>((size_t)ns);
        h->owner = cv.take<unsigned char>((size_t)ns);
    });
    struct { SortScratch<McRec> sort; unsigned char* head; unsigned* counts; unsigned* ocounts; long long* owners; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, ns);
        sc.head = cv.take<unsigned char>((size_t)ns);
        sc.counts = cv.take<unsigned>(keep_count_words(ns));
        sc.ocounts = cv.take<unsigned>(keep_count_words(ns));
        sc.owners = cv.take<long long>(1);
    }));
    int b = 1;                                       // bits of the largest corner index, n - 1
    while (b < 31 && ((h->n - 1) >> b) != 0) ++b;
    PCU_LAUNCH((mc_slots_kernel<W>), tiles, kThreads, stream, h->idx, (const unsigned char*)h->cases, m,
               (const unsigned long long*)h->tile_slot0, (const unsigned long long*)h->tile_face0, b, sc.sort.a);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, ns, 1, stream, &sorted, 2 * b));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(ns), kThreads, stream, (const McRec*)sorted, ns, sc.head);
    PCU_TRY(enqueue_keep_offsets(sc.head, ns, sc.counts, &h->counts->verts, stream));
    PCU_LAUNCH(mc_runs_kernel, blocks_for(ns), kThreads, stream, (const McRec*)sorted, ns, (const unsigned char*)sc.head,
               (const unsigned*)sc.counts, h->slot_run, h->owner);
    PCU_TRY(enqueue_keep_offsets(h->owner, ns, sc.ocounts, sc.owners, stream));
    PCU_LAUNCH(mc_owner_kernel, blocks_for(ns), kThreads, stream, (const unsigned char*)h->owner, ns, (const unsigned*)sc.ocounts,
               (const unsigned*)h->slot_run, h->run_vid);
    PCU_TRY(read_record(h->counts, &c, stream));
    h->verts = c.verts;
    return PCU_B200_OK;
}

template <typename T, typename S>
int mc_build_width(pcu_b200_workspace* ws, pcu_b200_marching_cubes* h, cudaStream_t stream) {
    return h->width == 8 ? mc_build<T, S, 8>(ws, h, stream) : mc_build<T, S, 4>(ws, h, stream);
}

template <typename T>
int marching_cubes_prepare_device(pcu_b200_workspace* ws, const void* scalars, int s_f64, const T* coords, long long n, const void* idx,
                                  long long m, int kind, double isovalue, pcu_b200_marching_cubes** out, long long* out_counts,
                                  cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!scalars || !coords || !idx) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (n <= 0 || n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: n must be in [1, 2^31 - 2], got %lld", n);
    if (m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid cube_indices has zero rows!");
    if (kind < kIdxI32 || kind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind %d", kind);
    if ((uintptr_t)idx % 16 != 0) return fail(PCU_B200_INVALID_ARGUMENT, "cube_idx must be 16-byte aligned");
    if ((m + kThreads - 1) / kThreads > 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "too many cubes (%lld)", m);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_marching_cubes* h) -> int {
        h->t_f64 = sizeof(T) == 8; h->s_f64 = s_f64 != 0; h->width = wide_index(kind) ? 8 : 4;
        h->scalars = scalars; h->coords = coords; h->idx = idx; h->n = n; h->m = m;
        h->iso = s_f64 ? (double)(T)isovalue : (double)(T)(float)isovalue;
        const long long tiles = (m + kThreads - 1) / kThreads;
        const auto carve = [&](Carver& cv) {
            h->cases = cv.take<unsigned char>((size_t)m);
            h->tile_sum = cv.take<unsigned>((size_t)tiles);
            h->tile_slot0 = cv.take<unsigned long long>((size_t)tiles);
            h->tile_face0 = cv.take<unsigned long long>((size_t)tiles);
            h->counts = cv.take<McCounts>(1);
        };
        PCU_TRY(alloc_block(h->cube_block, carve_at(nullptr, carve), stream, "marching cubes"));
        carve_at(h->cube_block, carve);
        PCU_TRY((h->s_f64 ? mc_build_width<T, double>(ws, h, stream) : mc_build_width<T, float>(ws, h, stream)));
        const long long most = kind == kIdxI32 ? (1ll << 31) : kind == kIdxU32 ? (1ll << 32) : LLONG_MAX;
        if (h->verts > most)
            return fail(PCU_B200_INVALID_ARGUMENT, "marching cubes: %lld vertices cannot be indexed by cube_indices' dtype", h->verts);
        return PCU_B200_OK;
    }));
    out_counts[0] = (*out)->verts;
    out_counts[1] = (*out)->faces;
    return PCU_B200_OK;
}

template <typename T, typename S, int W>
int mc_emit_launch(const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    PCU_LAUNCH((mc_emit_kernel<T, S, W>), blocks_for(h->m), kThreads, stream, (const S*)h->scalars, (const T*)h->coords, h->idx,
               (const unsigned char*)h->cases, h->m, (const unsigned long long*)h->tile_slot0,
               (const unsigned long long*)h->tile_face0, (T)h->iso, (const unsigned*)h->slot_run, (const unsigned*)h->run_vid,
               (const unsigned char*)h->owner, (T*)out_v, out_f);
    return PCU_B200_OK;
}

template <typename T, typename S>
int mc_emit_width(const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    return h->width == 8 ? mc_emit_launch<T, S, 8>(h, out_v, out_f, stream) : mc_emit_launch<T, S, 4>(h, out_v, out_f, stream);
}

int marching_cubes_emit_device(pcu_b200_workspace* ws, const pcu_b200_marching_cubes* h, void* out_v, void* out_f, cudaStream_t stream) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "marching-cubes"));
    if (h->slots == 0) return PCU_B200_OK;
    if (!out_v || (h->faces > 0 && !out_f)) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    if (h->t_f64) return h->s_f64 ? mc_emit_width<double, double>(h, out_v, out_f, stream) : mc_emit_width<double, float>(h, out_v, out_f, stream);
    return h->s_f64 ? mc_emit_width<float, double>(h, out_v, out_f, stream) : mc_emit_width<float, float>(h, out_v, out_f, stream);
}

// Codes, their sort, the six-neighbour lookups, the ordered compaction.  out_counts (device): {boundary rows, bad rows}.
template <typename I>
int svb_device(pcu_b200_workspace* ws, const I* g, long long n, long long* out_idx, long long* out_counts, cudaStream_t stream) {
    struct { SortScratch<McRec> sort; unsigned char* keep; unsigned* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.keep = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 2 * sizeof(long long), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, (unsigned long long*)(out_counts + 1));
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH((svb_flag_kernel<I>), blocks_for(n), kThreads, stream, g, n, (const McRec*)sorted, sc.keep);
    PCU_TRY(enqueue_keep_offsets(sc.keep, n, sc.counts, out_counts, stream));
    PCU_LAUNCH(keep_rows_kernel<long long>, blocks_for(n), kThreads, stream, (const unsigned char*)sc.keep, n, (const unsigned*)sc.counts, out_idx);
    return PCU_B200_OK;
}

int sparse_voxel_grid_boundary_device(pcu_b200_workspace* ws, const void* g, long long n, int kind, long long* out_idx,
                                      long long* out_counts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!g || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid grid_coordinates has zero rows!");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "sparse_voxel_grid_boundary: at most 2^31 - 2 voxels, got %lld", n);
    if (kind != kIdxI32 && kind != kIdxI64)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small.");
    if (!out_idx || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    return kind == kIdxI64 ? svb_device<long long>(ws, (const long long*)g, n, out_idx, out_counts, stream)
                           : svb_device<int>(ws, (const int*)g, n, out_idx, out_counts, stream);
}

// ---- Voronoi cells in the unit cube / square and Lloyd relaxation (voronoi.cuh) ----------------------------------
// One evaluation of the cells of n seeds (fp64, (n, dim)):
//   pass 1  the seeds' self k-NN (k = 64 in 3-D, 24 in 2-D; no tie replay: the order among equidistant neighbours
//           cannot change a cell, and the certificate only reads the k-th distance), then every cell on the thread's
//           stack at 96 (3-D) / 48 (2-D) vertices;
//   pass 2  the cells pass 1 left uncertified, compacted in ascending order: their k-NN with k = 160 (3-D) / 64 (2-D),
//           at 252 / 250 vertices;
//   pass 3  what pass 2 left: its list, then every seed that can still cut the cell, with the cell in device memory at
//           2 048 (3-D) / 1 024 (2-D) vertices; the cells that outgrow it are compacted and redone at twice the
//           capacity, until every cell is certified.
// The host reads the count after pass 1 (one synchronisation), after pass 2 when it ran, and after every round of
// pass 3.  passes[p] += cells handled by pass p (pass 3: summed over its rounds).
constexpr int kVorK1[2] = {24, 64}, kVorK2[2] = {64, 160};   // by dim - 2
constexpr int kVorSmall[2] = {48, 96}, kVorLarge[2] = {250, 252};
constexpr int kVorWide[2] = {1024, 2048};
constexpr int kVorWideMax = 1 << 22;   // vertices of one cell: 150 MB of device memory in 3-D

// pass 0, 1: the small and the large capacity on the stack
template <int D>
int vor_pass_launch(const VorPass& p, int pass, cudaStream_t stream) {
    const unsigned blocks = (unsigned)((p.count + kVorThreads - 1) / kVorThreads);
    if (pass == 0) PCU_LAUNCH((vor_clip_kernel<D, kVorSmall[D - 2]>), blocks, kVorThreads, stream, p);
    else           PCU_LAUNCH((vor_clip_kernel<D, kVorLarge[D - 2]>), blocks, kVorThreads, stream, p);
    return PCU_B200_OK;
}

// How the passes clip one kind of entry: the cells in the unit cube / square, or the (face, seed) pairs of restricted
// cells (rvd.cuh).  k2: the longer lists of pass 2; wide: the first capacity of pass 3.
template <int D>
struct VorCube {
    static constexpr int k2 = kVorK2[D - 2], wide = kVorWide[D - 2];
    static int launch(const VorPass& p, int pass, cudaStream_t stream) { return vor_pass_launch<D>(p, pass, stream); }
    static size_t cell_bytes(int V) { return vor_cell_bytes<D>(V); }
    static int launch_wide(const VorPass& p, int V, cudaStream_t stream) {
        PCU_LAUNCH(vor_clip_wide_kernel<D>, (unsigned)((p.count + kVorThreads - 1) / kVorThreads), kVorThreads, stream, p, V);
        return PCU_B200_OK;
    }
};

// Restricted pairs: the k-NN lists of a 2-D cell (a restricted cell is a surface patch), polygons of 16 / 64 vertices on
// the stack, then 256 in device memory.
constexpr int kRvK1 = 24, kRvK2 = 64, kRvSmall = 16, kRvLarge = 64, kRvWide = 256;
struct VorRestricted {
    static constexpr int k2 = kRvK2, wide = kRvWide;
    static int launch(const VorPass& p, int pass, cudaStream_t stream) {
        const unsigned blocks = (unsigned)((p.count + kVorThreads - 1) / kVorThreads);
        if (pass == 0) PCU_LAUNCH(rv_clip_kernel<kRvSmall>, blocks, kVorThreads, stream, p);
        else           PCU_LAUNCH(rv_clip_kernel<kRvLarge>, blocks, kVorThreads, stream, p);
        return PCU_B200_OK;
    }
    static size_t cell_bytes(int V) { return poly_bytes(V); }
    static int launch_wide(const VorPass& p, int V, cudaStream_t stream) {
        PCU_LAUNCH(rv_clip_wide_kernel, (unsigned)((p.count + kVorThreads - 1) / kVorThreads), kVorThreads, stream, p, V);
        return PCU_B200_OK;
    }
};

// Passes 2 and 3 over the entries pass 1 (p, already enqueued over p.count entries) left uncertified in `flag`; `counts`
// holds keep_count_words(p.count) words.
template <class K>
int vor_fallback(pcu_b200_workspace* ws, VorPass p, unsigned char* flag, unsigned* counts, VorSync* sync, long long* passes,
                 VorSync* seen, cudaStream_t stream) {
    const long long n = p.n, entries = p.count;
    PCU_TRY(enqueue_keep_offsets(flag, entries, counts, &sync->count, stream));
    PCU_TRY(read_record(sync, seen, stream));
    const long long c1 = seen->count;
    if (c1 == 0) return PCU_B200_OK;
    const int k2 = (int)std::min<long long>(K::k2, n);
    int *rows, *sub[2]; double *q, *d2; long long* i2; unsigned char* flag2; unsigned* counts2;
    PCU_TRY(carve_scratch(ws, kVorList, stream, [&](Carver& cv) {
        rows = cv.take<int>((size_t)c1);
        sub[0] = cv.take<int>((size_t)c1);
        sub[1] = cv.take<int>((size_t)c1);
        q = cv.take<double>((size_t)3 * c1);
        d2 = cv.take<double>((size_t)k2 * c1);
        i2 = cv.take<long long>((size_t)k2 * c1);
        flag2 = cv.take<unsigned char>((size_t)c1);
        counts2 = cv.take<unsigned>(keep_count_words(c1));
    }));
    PCU_TRY(enqueue_keep_rows(flag, entries, counts, rows, stream));
    PCU_LAUNCH(vor_gather_kernel, blocks_for(c1), kThreads, stream, p.x3, (const int*)rows, c1, q, p.pair_seed);
    PCU_TRY(knn_device<double>(ws, q, c1, p.x3, n, k2, 1, d2, i2, nullptr, stream, nullptr, false));
    p.rows = rows; p.count = c1; p.nn_idx = i2; p.nn_d2 = d2; p.k = k2; p.list_is_all = k2 >= n; p.uncert = flag2;
    p.list_of_seed = 0;
    PCU_TRY(K::launch(p, 1, stream));
    passes[1] += c1;
    PCU_TRY(enqueue_keep_offsets(flag2, c1, counts2, &sync->count, stream));
    PCU_TRY(read_record(sync, seen, stream));
    long long cnt = seen->count;
    if (cnt == 0) return PCU_B200_OK;
    // the last resort; sub[r & 1]: the pass-2 entries of round r
    PCU_TRY(enqueue_keep_rows(flag2, c1, counts2, sub[0], stream));
    p.scan_all = 1; p.list_is_all = 0; p.uncert = flag2;
    for (int V = K::wide, r = 0;; V *= 2, ++r) {
        if (V > kVorWideMax)
            return fail(PCU_B200_OUT_OF_MEMORY, "voronoi: %lld cells have more than %d vertices", cnt, kVorWideMax);
        // the cells live in the arena: the k-NN searches, its only other users here, are enqueued already
        PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
            p.cells = cv.take<unsigned char>((size_t)cnt * K::cell_bytes(V));
        }));
        p.sub = sub[r & 1]; p.count = cnt;
        PCU_TRY(K::launch_wide(p, V, stream));
        passes[2] += cnt;
        PCU_TRY(enqueue_keep_offsets(flag2, cnt, counts2, &sync->count, stream));
        PCU_TRY(read_record(sync, seen, stream));
        if (seen->count == 0) break;
        PCU_LAUNCH(vor_keep_sub_kernel, blocks_for(cnt), kThreads, stream, (const unsigned char*)flag2, cnt, (const unsigned*)counts2,
                   (const int*)sub[r & 1], sub[(r + 1) & 1]);
        cnt = seen->count;
    }
    return PCU_B200_OK;
}

template <int D>
int vor_eval(pcu_b200_workspace* ws, const double* x, long long n, VorSync* sync, double** mom_out, long long* passes,
             VorSync* seen, cudaStream_t stream) {
    const int k1 = (int)std::min<long long>(kVorK1[D - 2], n);
    double *x3 = nullptr, *mom, *d1; long long* i1; unsigned char* flag; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        if (D == 2) x3 = cv.take<double>((size_t)3 * n);
        mom = cv.take<double>((size_t)kVorMoments * n);
        d1 = cv.take<double>((size_t)k1 * n);
        i1 = cv.take<long long>((size_t)k1 * n);
        flag = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    if (D == 3) x3 = (double*)x;
    else PCU_LAUNCH(vor_lift_kernel, blocks_for(n), kThreads, stream, x, n, x3);
    *mom_out = mom;
    PCU_TRY(knn_device<double>(ws, x3, n, x3, n, k1, 1, d1, i1, nullptr, stream, nullptr, false));
    VorPass p{};
    p.x = x; p.x3 = x3; p.n = n; p.count = n; p.nn_idx = i1; p.nn_d2 = d1; p.k = k1; p.list_is_all = k1 >= n;
    p.mom = mom; p.uncert = flag;
    PCU_TRY(vor_pass_launch<D>(p, 0, stream));
    passes[0] += n;
    return vor_fallback<VorCube<D>>(ws, p, flag, counts, sync, passes, seen, stream);
}

int vor_check(long long n, int dim) {
    if (dim != 2 && dim != 3) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: dim must be 2 or 3, got %d", dim);
    if (n > 0x7fffffffLL - 1) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: at most 2^31 - 2 seeds, got %lld", n);
    return PCU_B200_OK;
}

template <int D>
int voronoi_centroids_device(pcu_b200_workspace* ws, const double* x, long long n, double* out, double* out_moments,
                             long long* passes, cudaStream_t stream) {
    VorSync* sync;
    PCU_TRY(carve_scratch(ws, kLloyd, stream, [&](Carver& cv) { sync = cv.take<VorSync>(1); }));
    PCU_CUDA(cudaMemsetAsync(sync, 0, sizeof(VorSync), stream));
    double* mom; VorSync seen;
    PCU_TRY(vor_eval<D>(ws, x, n, sync, &mom, passes, &seen, stream));
    PCU_LAUNCH(vor_centroid_kernel<D>, blocks_for(n), kThreads, stream, x, n, (const double*)mom, out);
    if (out_moments)
        PCU_CUDA(cudaMemcpyAsync(out_moments, mom, (size_t)n * kVorMoments * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return PCU_B200_OK;
}

// Blocks of the cooperative L-BFGS step: at most 4 per SM, no more than the vectors need.
int lbfgs_grid_blocks(const pcu_b200_workspace* ws, long long N, unsigned* out_blocks) {
    int fit = 0;
    PCU_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, lbfgs_step_kernel, kThreads, 0));
    if (fit < 1) return fail(PCU_B200_CUDA_ERROR, "lbfgs_step_kernel cannot be resident on this device");
    const long long want = (N + kThreads - 1) / kThreads;
    *out_blocks = (unsigned)std::max<long long>(1, std::min<long long>(want, (long long)std::min(4, fit) * ws->sm_count));
    return PCU_B200_OK;
}

// The initial sample, num_lloyd Lloyd steps, then the Newton phase (L-BFGS, voronoi.cuh), for either kind of cell:
// init(x) writes the (n, D) initial sample; eval(x, sync, &mom, &seen) evaluates the cells of x (their (n, 5) moments
// into mom); cube: trial points must lie in the unit cube.  Synchronisations: those of init and of every cell evaluation,
// one for the initial L-BFGS state, one after every L-BFGS step (its verdict decides whether the trial point is
// evaluated), and one for the energies at the end.
template <int D, class Init, class Eval>
int lloyd_run(pcu_b200_workspace* ws, long long n, int cube, int num_lloyd, int num_newton, double* out, double* energy_host,
              int* iters_host, cudaStream_t stream, Init&& init, Eval&& eval) {
    const long long N = n * D;
    const bool newton = num_newton > 0;
    unsigned blocks = 1;
    if (newton) PCU_TRY(lbfgs_grid_blocks(ws, N, &blocks));
    double *x, *x_acc = nullptr, *g = nullptr, *p = nullptr, *S = nullptr, *Y = nullptr, *partial = nullptr, *energy = nullptr;
    LbState* st = nullptr; VorSync* sync;
    PCU_TRY(carve_scratch(ws, kLloyd, stream, [&](Carver& cv) {
        sync = cv.take<VorSync>(1);
        x = cv.take<double>((size_t)N);
        if (newton) {
            st = cv.take<LbState>(1);
            energy = cv.take<double>((size_t)num_newton + 1);
            partial = cv.take<double>((size_t)2 * blocks);
            x_acc = cv.take<double>((size_t)N);
            g = cv.take<double>((size_t)N);
            p = cv.take<double>((size_t)N);
            S = cv.take<double>((size_t)kLbSlots * N);
            Y = cv.take<double>((size_t)kLbSlots * N);
        }
    }));
    PCU_CUDA(cudaMemsetAsync(sync, 0, sizeof(VorSync), stream));
    PCU_TRY(init(x));
    double* mom; VorSync seen;
    for (int it = 0; it < num_lloyd; ++it) {
        PCU_TRY(eval((const double*)x, sync, &mom, &seen));
        PCU_LAUNCH(vor_centroid_kernel<D>, blocks_for(n), kThreads, stream, (const double*)x, n, (const double*)mom, x);
    }
    if (!newton) {
        PCU_CUDA(cudaMemcpyAsync(out, x, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, stream));
        if (iters_host) *iters_host = 0;
        return PCU_B200_OK;
    }
    LbState s0{};
    s0.t = 1.0; s0.gamma = 1.0; s0.init = 1;
    PCU_CUDA(cudaMemcpyAsync(st, &s0, sizeof(LbState), cudaMemcpyHostToDevice, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));   // s0 lives on this stack
    LbArgs a{};
    a.n = n; a.D = D; a.x_acc = x_acc; a.g = g; a.x_t = x; a.p = p; a.S = S; a.Y = Y; a.partial = partial;
    a.st = st; a.sync = sync; a.energy = energy; a.num_newton = num_newton; a.cube = cube;
    PCU_TRY(eval((const double*)x, sync, &mom, &seen));
    for (;;) {
        a.mom = mom;
        void* args[] = {(void*)&a};
        PCU_CUDA(cudaLaunchCooperativeKernel((void*)lbfgs_step_kernel, dim3(blocks), dim3(kThreads), args, 0, stream));
        g_launches.fetch_add(1, std::memory_order_relaxed);
        PCU_TRY(read_record(sync, &seen, stream));   // the step's verdict: evaluate its trial point, or stop
        if (seen.done) break;
        PCU_TRY(eval((const double*)x, sync, &mom, &seen));
    }
    PCU_CUDA(cudaMemcpyAsync(out, x_acc, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    if (energy_host) PCU_CUDA(cudaMemcpyAsync(energy_host, energy, ((size_t)seen.iter + 1) * sizeof(double), cudaMemcpyDeviceToHost, stream));
    PCU_CUDA(cudaStreamSynchronize(stream));
    if (iters_host) *iters_host = seen.iter;
    return PCU_B200_OK;
}

// lloyd_3d / lloyd_2d: the counter-based initial sample of (n, D, seed) and the cube's cells.
template <int D>
int lloyd_device(pcu_b200_workspace* ws, long long n, unsigned seed, int num_lloyd, int num_newton, double* out,
                 double* energy_host, int* iters_host, long long* passes, cudaStream_t stream) {
    const long long N = n * D;
    return lloyd_run<D>(
        ws, n, 1, num_lloyd, num_newton, out, energy_host, iters_host, stream,
        [&](double* x) -> int {
            PCU_LAUNCH(lloyd_init_kernel, blocks_for(N), kThreads, stream, seed, N, x);
            return PCU_B200_OK;
        },
        [&](const double* x, VorSync* sync, double** mom, VorSync* seen) -> int {
            return vor_eval<D>(ws, x, n, sync, mom, passes, seen, stream);
        });
}

// ---- Voronoi cells restricted to a triangle mesh and Lloyd sampling of its surface (rvd.cuh) ---------------------
// One evaluation of the cells of n seeds x (fp64, (n, 3)) on the faces:
//   the faces' candidate balls (a k = 1 search of the face centroids among the seeds), their tree, the pair count
//   (one synchronisation sizes the pairs), the pairs, the seeds' self k-NN (k = 24, no tie replay), then pass 1 over
//   every pair with the polygon on the stack at 16 vertices, and the fallback passes of the cube's cells (vor_fallback:
//   k = 64 and 64 vertices, then every seed from 256 vertices in device memory up); finally each seed's pairs summed in
//   order.  Synchronisations: the pair count, the count pass 1 leaves, and one per fallback pass or round that runs.
//   passes[p] += pairs handled by pass p.
struct RvScratch {
    long long n = 0, m = 0;
    int k1 = 1;
    double *tri, *cen, *rad, *fd2, *balls, *sd2, *mom;
    long long *fidx, *sidx, *start;
    unsigned long long *local, *tiles, *bad;
    VorSync* sync;
    void carve(Carver& cv) {
        tri = cv.take<double>((size_t)9 * m);
        cen = cv.take<double>((size_t)3 * m);
        rad = cv.take<double>((size_t)m);
        fd2 = cv.take<double>((size_t)m);
        fidx = cv.take<long long>((size_t)m);
        balls = cv.take<double>((size_t)4 * m);
        sd2 = cv.take<double>((size_t)k1 * n);
        sidx = cv.take<long long>((size_t)k1 * n);
        mom = cv.take<double>((size_t)kVorMoments * n);
        start = cv.take<long long>((size_t)n);
        local = cv.take<unsigned long long>((size_t)n);
        tiles = cv.take<unsigned long long>((size_t)blocks_for(n));
        bad = cv.take<unsigned long long>(1);
        sync = cv.take<VorSync>(1);
    }
};

int rv_check(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind, long long n) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(mesh_check(v, nv, f, m, fkind));
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "num_samples must be > 0");
    if (n > 0x7fffffffLL - 1) return fail(PCU_B200_INVALID_ARGUMENT, "restricted Voronoi: at most 2^31 - 2 seeds, got %lld", n);
    return PCU_B200_OK;
}

// Carves the call's RvScratch and enqueues the per-face pass (corners, centroids, radii, faces out of range).
int rv_prepare(pcu_b200_workspace* ws, RvScratch& r, const double* v, long long nv, const void* f, long long m, int fkind,
               long long n, cudaStream_t stream) {
    r.n = n; r.m = m; r.k1 = (int)std::min<long long>(kRvK1, n);
    PCU_TRY(carve_scratch(ws, kRvd, stream, [&](Carver& cv) { r.carve(cv); }));
    PCU_CUDA(cudaMemsetAsync(r.bad, 0, sizeof(unsigned long long), stream));
    PCU_CUDA(cudaMemsetAsync(r.sync, 0, sizeof(VorSync), stream));
    PCU_LAUNCH(rv_face_kernel, blocks_for(m), kThreads, stream, v, nv, f, fkind, m, r.tri, r.cen, r.rad, r.bad);
    return PCU_B200_OK;
}

int rv_eval(pcu_b200_workspace* ws, const RvScratch& r, const double* x, VorSync* sync, double** mom_out, long long* passes,
            VorSync* seen, cudaStream_t stream) {
    const long long n = r.n, m = r.m;
    *mom_out = r.mom;
    PCU_TRY(knn_device<double>(ws, r.cen, m, x, n, 1, 1, r.fd2, r.fidx, nullptr, stream, nullptr, false));
    PCU_LAUNCH(rv_ball_kernel, blocks_for(m), kThreads, stream, (const double*)r.cen, (const double*)r.rad, (const double*)r.fd2,
               (const long long*)r.fidx, m, r.balls);
    PCU_TRY(knn_device<double>(ws, x, n, x, n, r.k1, 1, r.sd2, r.sidx, nullptr, stream, nullptr, false));
    MeshTree<RvBall> tree;   // in the arena, with its build's temporaries: nothing re-carves it before the pairs are out
    PCU_TRY((build_mesh_tree<double, RvBall>)(ws, r.balls, m, nullptr, m, 0, false, nullptr, stream, tree));
    const unsigned sb = blocks_for(n);
    PCU_LAUNCH(rv_count_kernel, sb, kThreads, stream, x, n, m, (const MqScratch*)tree.sc, (const MqNode*)tree.nodes,
               (const RvBall*)tree.leaves, (const int*)tree.ids, r.local, r.tiles);
    PCU_LAUNCH(rv_tiles_kernel, 1, 1024, stream, r.tiles, (long long)sb, sync);
    PCU_TRY(read_record(sync, seen, stream));
    const long long P = seen->count;
    if (P == 0) {   // every face has zero area
        PCU_CUDA(cudaMemsetAsync(r.mom, 0, (size_t)n * kVorMoments * sizeof(double), stream));
        return PCU_B200_OK;
    }
    int *pseed, *pface; double* pmom; unsigned char* flag; unsigned* counts;
    const int rs = P > 0x7fffffffLL ? PCU_B200_OUT_OF_MEMORY : carve_scratch(ws, kAux, stream, [&](Carver& cv) {
        pseed = cv.take<int>((size_t)P);
        pface = cv.take<int>((size_t)P);
        pmom = cv.take<double>((size_t)kVorMoments * P);
        flag = cv.take<unsigned char>((size_t)P);
        counts = cv.take<unsigned>(keep_count_words(P));
    });
    if (rs == PCU_B200_OUT_OF_MEMORY)
        return fail(PCU_B200_OUT_OF_MEMORY, "restricted Voronoi: %lld (face, seed) pairs do not fit (%zu bytes of scratch, at most "
                    "2^31 - 1 pairs)", P, (size_t)P * (8 + 8 * kVorMoments + 1));
    PCU_TRY(rs);
    PCU_LAUNCH(rv_emit_kernel, sb, kThreads, stream, x, n, m, (const MqScratch*)tree.sc, (const MqNode*)tree.nodes,
               (const RvBall*)tree.leaves, (const int*)tree.ids, (const unsigned long long*)r.local, (const unsigned long long*)r.tiles,
               r.start, pseed, pface);
    VorPass p{};
    p.x = x; p.x3 = x; p.n = n; p.count = P; p.nn_idx = r.sidx; p.nn_d2 = r.sd2; p.k = r.k1; p.list_is_all = r.k1 >= n;
    p.list_of_seed = 1; p.mom = pmom; p.uncert = flag; p.pair_seed = pseed; p.pair_face = pface; p.tri = r.tri;
    PCU_TRY(VorRestricted::launch(p, 0, stream));
    passes[0] += P;
    PCU_TRY(vor_fallback<VorRestricted>(ws, p, flag, counts, sync, passes, seen, stream));
    PCU_LAUNCH(rv_reduce_kernel, sb, kThreads, stream, (const long long*)r.start, n, P, (const double*)pmom, r.mom);
    return PCU_B200_OK;
}

int restricted_moments_device(pcu_b200_workspace* ws, const double* x, long long n, const double* v, long long nv, const void* f,
                              long long m, int fkind, double* out_moments, long long* passes, cudaStream_t stream) {
    RvScratch r;
    PCU_TRY(rv_prepare(ws, r, v, nv, f, m, fkind, n, stream));
    unsigned long long bad = 0;
    PCU_TRY(read_record(r.bad, &bad, stream));
    if (bad) return bad_corners(bad);
    double* mom; VorSync seen;
    PCU_TRY(rv_eval(ws, r, x, r.sync, &mom, passes, &seen, stream));
    PCU_CUDA(cudaMemcpyAsync(out_moments, mom, (size_t)n * kVorMoments * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return PCU_B200_OK;
}

// sample_mesh_lloyd: the first n samples of sample_mesh_random at `seed` (their fp64 positions) relaxed on the
// restricted cells, with no domain test for the Newton phase's trial points.  The initial sample reads the face CDF's
// record (one synchronisation) and fails as sample_mesh_random's caller does on faces out of range or a zero area.
int sample_mesh_lloyd_device(pcu_b200_workspace* ws, const double* v, long long nv, const void* f, long long m, int fkind,
                             long long n, unsigned seed, int num_lloyd, int num_newton, double* out, double* energy_host,
                             int* iters_host, long long* passes, cudaStream_t stream) {
    RvScratch r;
    PCU_TRY(rv_prepare(ws, r, v, nv, f, m, fkind, n, stream));
    return lloyd_run<3>(
        ws, n, 0, num_lloyd, num_newton, out, energy_host, iters_host, stream,
        [&](double* x) -> int {
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
        },
        [&](const double* x, VorSync* sync, double** mom, VorSync* seen) -> int {
            return rv_eval(ws, r, x, sync, mom, passes, seen, stream);
        });
}

// ---- sparse voxel grids and voxel cube meshes (sparse_voxels.cuh) -------------------------------------------------
enum SvgMode { kSvgPoints = 0, kSvgDilate = 1, kSvgHex = 2 };
// Dilation ranks 26 flags per voxel, the hex mesh 8 corners per voxel, in 32 bits (compact.cuh: fewer than 2^31 rows);
// voxel_grid_geometry's int32 faces index 8 n vertices.
constexpr long long kSvgMaxDilate = (0x7ffffffeLL) / 26;   // 82 595 524
constexpr long long kSvgMaxHex = (0x7ffffffeLL) / 8;       // 2^28 - 1
constexpr long long kVgMaxVoxels = 1LL << 28;

int svg_overflow() {
    return fail(PCU_B200_INVALID_ARGUMENT, "Invalid vertex leads to an overflow integer. Perhaps grid_size is too small.");
}

// The handle's block for `recs` records: sort scratch, run heads (unless the records are distinct), block offsets, the
// count record.  The caller writes the records into sort.a.
int svg_alloc(pcu_b200_sparse_grid* h, long long recs, bool heads, SortScratch<McRec>& sort, cudaStream_t stream) {
    h->recs = recs;
    const auto carve = [&](Carver& cv) {
        sort.carve(cv, recs);
        h->head = heads ? cv.take<unsigned char>((size_t)recs) : nullptr;
        h->offsets = cv.take<unsigned>(keep_count_words(recs));
        h->counts = cv.take<SvgCounts>(1);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "sparse voxel grid"));
    carve_at(h->block, carve);
    PCU_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(SvgCounts), stream));
    return PCU_B200_OK;
}

// Sorts the records, numbers their runs (the count of distinct codes into h->counts->rows) and, when read, reads the
// count record: one synchronisation of `stream`.
int svg_sort_runs(pcu_b200_sparse_grid* h, const SortScratch<McRec>& sort, bool read, cudaStream_t stream) {
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sort, h->recs, 1, stream, &sorted));
    h->sorted = sorted;
    if (h->head) {
        PCU_LAUNCH(mc_heads_kernel, blocks_for(h->recs), kThreads, stream, (const McRec*)sorted, h->recs, h->head);
        PCU_TRY(enqueue_keep_offsets(h->head, h->recs, h->offsets, &h->counts->rows, stream));
    }
    if (!read) return PCU_B200_OK;
    SvgCounts c;
    PCU_TRY(read_record(h->counts, &c, stream));
    if (c.bad) return svg_overflow();
    h->rows = c.rows;
    return PCU_B200_OK;
}

// A grid argument of the sparse-grid entry points: int32 or int64 (unsigned grids fail the reference's range check).
int svg_check_grid(const void* g, long long n, int kind, long long most, const char* what) {
    if (!g || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid grid_coordinates has zero rows!");
    if (n > most) return fail(PCU_B200_INVALID_ARGUMENT, "%s: at most %lld voxels are supported, got %lld", what, most, n);
    if (kind != kIdxI32 && kind != kIdxI64) return svg_overflow();
    return PCU_B200_OK;
}

template <typename T>
int svg_points_prepare(pcu_b200_workspace* ws, const T* p, long long n, const double size[3], const double origin[3],
                       pcu_b200_sparse_grid** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!p || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid points has zero rows!");
    if (n >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "sparse_voxel_grid_from_pointcloud: at most 2^31 - 2 points are supported, got %lld", n);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgPoints; h->n = n;
        for (int a = 0; a < 3; ++a) { h->place.g[a] = size[a]; h->place.o[a] = origin[a]; }
        SortScratch<McRec> sort;
        PCU_TRY(svg_alloc(h, n, true, sort, stream));
        PCU_LAUNCH((svg_point_codes_kernel<T>), blocks_for(n), kThreads, stream, p, n, h->place, sort.a, &h->counts->bad);
        return svg_sort_runs(h, sort, true, stream);
    }));
    out_counts[0] = (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

// One dilation round: the input's codes and their sort, the owned missing neighbours' flags and their count (read:
// one synchronisation), then the owned codes, compacted and sorted.
template <typename I>
int svg_dilate_build(pcu_b200_workspace* ws, pcu_b200_sparse_grid* h, const I* g, long long n, cudaStream_t stream) {
    const long long slots = 26 * n;
    struct { SortScratch<McRec> sort; unsigned char* flag; unsigned* counts; SvgCounts* rec; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.flag = cv.take<unsigned char>((size_t)slots);
        sc.counts = cv.take<unsigned>(keep_count_words(slots));
        sc.rec = cv.take<SvgCounts>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(SvgCounts), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, &sc.rec->bad);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH(svg_dilate_flag_kernel, blocks_for(n), kThreads, stream, (const McRec*)sorted, n, sc.flag);
    PCU_TRY(enqueue_keep_offsets(sc.flag, slots, sc.counts, &sc.rec->rows, stream));
    SvgCounts c;
    PCU_TRY(read_record(sc.rec, &c, stream));
    if (c.bad) return svg_overflow();
    h->rows = c.rows;
    if (c.rows == 0) return PCU_B200_OK;
    SortScratch<McRec> sort;
    PCU_TRY(svg_alloc(h, c.rows, false, sort, stream));
    PCU_LAUNCH(svg_dilate_write_kernel, blocks_for(slots), kThreads, stream, (const McRec*)sorted, n, (const unsigned char*)sc.flag,
               (const unsigned*)sc.counts, sort.a);
    return svg_sort_runs(h, sort, false, stream);
}

int svg_dilate_prepare(pcu_b200_workspace* ws, const void* g, long long n, int kind, pcu_b200_sparse_grid** out, long long* out_counts,
                       cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(svg_check_grid(g, n, kind, kSvgMaxDilate, "dilate_sparse_voxel_grid"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgDilate; h->n = n; h->grid = g; h->out_kind = kind;
        return kind == kIdxI64 ? svg_dilate_build<long long>(ws, h, (const long long*)g, n, stream)
                               : svg_dilate_build<int>(ws, h, (const int*)g, n, stream);
    }));
    out_counts[0] = n + (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

int svg_hex_prepare(pcu_b200_workspace* ws, const void* g, long long n, int kind, const double size[3], const double origin[3], int v_f64,
                    pcu_b200_sparse_grid** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    PCU_TRY(svg_check_grid(g, n, kind, kSvgMaxHex, "sparse_voxel_grid_to_hex_mesh"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_sparse_grid* h) -> int {
        h->mode = kSvgHex; h->n = n; h->out_kind = v_f64 != 0;
        for (int a = 0; a < 3; ++a) { h->place.g[a] = size[a]; h->place.o[a] = origin[a]; }
        SortScratch<McRec> sort;
        PCU_TRY(svg_alloc(h, 8 * n, true, sort, stream));
        if (kind == kIdxI64) PCU_LAUNCH((svg_corners_kernel<long long>), blocks_for(n), kThreads, stream, (const long long*)g, n, sort.a, &h->counts->bad);
        else PCU_LAUNCH((svg_corners_kernel<int>), blocks_for(n), kThreads, stream, (const int*)g, n, sort.a, &h->counts->bad);
        return svg_sort_runs(h, sort, true, stream);
    }));
    out_counts[0] = (*out)->rows;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

template <typename O>
int svg_decode_launch(const pcu_b200_sparse_grid* h, void* out, cudaStream_t stream) {
    PCU_LAUNCH(svg_decode_kernel<O>, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, h->place, (O*)out);
    return PCU_B200_OK;
}

// From points: out_rows (rows, 3) int32, out_index (n) int64 point_to_vox.  Dilation: out_rows (n + rows, 3) of the
// grid's kind, the input rows then the new ones.  Hex mesh: out_rows (rows, 3) vertices, out_index (n, 8) int64 cubes.
int svg_emit(pcu_b200_workspace* ws, const pcu_b200_sparse_grid* h, void* out_rows, int64_t* out_index, cudaStream_t stream) {
    if (!ws || !h || !out_rows || (h->mode != kSvgDilate && !out_index)) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "sparse voxel grid"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    if (h->mode == kSvgDilate) {
        const size_t width = h->out_kind == kIdxI64 ? 8 : 4;
        PCU_CUDA(cudaMemcpyAsync(out_rows, h->grid, (size_t)h->n * 3 * width, cudaMemcpyDeviceToDevice, stream));
        if (h->rows == 0) return PCU_B200_OK;
        unsigned char* tail = (unsigned char*)out_rows + (size_t)h->n * 3 * width;
        return h->out_kind == kIdxI64 ? svg_decode_launch<long long>(h, tail, stream) : svg_decode_launch<int>(h, tail, stream);
    }
    if (h->mode == kSvgPoints) PCU_TRY(svg_decode_launch<int>(h, out_rows, stream));
    else PCU_TRY(h->out_kind ? svg_decode_launch<double>(h, out_rows, stream) : svg_decode_launch<float>(h, out_rows, stream));
    PCU_LAUNCH(svg_rank_kernel, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, (long long*)out_index);
    return PCU_B200_OK;
}

// Erosion: codes, their sort, the 26-neighbour test, the ordered copy of the kept rows.  out_counts (device):
// {kept rows, rows out of range}.
template <typename I>
int svg_erode_device(pcu_b200_workspace* ws, const I* g, long long n, I* out, long long* out_counts, cudaStream_t stream) {
    struct { SortScratch<McRec> sort; unsigned char* keep; unsigned* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.keep = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 2 * sizeof(long long), stream));
    PCU_LAUNCH((svb_codes_kernel<I>), blocks_for(n), kThreads, stream, g, n, sc.sort.a, (unsigned long long*)(out_counts + 1));
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 1, stream, &sorted));
    PCU_LAUNCH((svg_erode_flag_kernel<I>), blocks_for(n), kThreads, stream, g, n, (const McRec*)sorted, sc.keep);
    PCU_TRY(enqueue_keep_offsets(sc.keep, n, sc.counts, out_counts, stream));
    PCU_LAUNCH((svg_keep_voxels_kernel<I>), blocks_for(n), kThreads, stream, g, (const unsigned char*)sc.keep, n, (const unsigned*)sc.counts, out);
    return PCU_B200_OK;
}

int svg_erode(pcu_b200_workspace* ws, const void* g, long long n, int kind, void* out, long long* out_counts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(svg_check_grid(g, n, kind, 0x7ffffffeLL, "erode_sparse_voxel_grid"));
    if (!out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    return kind == kIdxI64 ? svg_erode_device<long long>(ws, (const long long*)g, n, (long long*)out, out_counts, stream)
                           : svg_erode_device<int>(ws, (const int*)g, n, (int*)out, out_counts, stream);
}

int voxel_grid_geometry_device(pcu_b200_workspace* ws, const void* ijk, long long n, int kind, const double size[3], const double origin[3],
                               double gap, float* out_v, int32_t* out_f, cudaStream_t stream) {
    if (!ws || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (!ijk || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input point cloud with zero points");
    if (n > kVgMaxVoxels) return fail(PCU_B200_INVALID_ARGUMENT, "voxel_grid_geometry: at most 2^28 voxels are supported, got %lld", n);
    if (kind < kIdxI32 || kind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind %d", kind);
    // as in the reference, a NaN size passes here
    if (size[0] <= 0.0 || size[1] <= 0.0 || size[2] <= 0.0) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size must be positive");
    if (!out_v || !out_f) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    VgGeom g;
    for (int k = 0; k < 3; ++k) { g.s[k] = size[k]; g.o[k] = origin[k]; }
    g.keep = 1.0 - gap;
    g.shift = 0.5 * gap;
    const unsigned blocks = blocks_for(12 * n);
    switch (kind) {
        case kIdxI32: PCU_LAUNCH(vg_geometry_kernel<int>, blocks, kThreads, stream, (const int*)ijk, n, g, out_v, out_f); break;
        case kIdxI64: PCU_LAUNCH(vg_geometry_kernel<long long>, blocks, kThreads, stream, (const long long*)ijk, n, g, out_v, out_f); break;
        case kIdxU32: PCU_LAUNCH(vg_geometry_kernel<unsigned>, blocks, kThreads, stream, (const unsigned*)ijk, n, g, out_v, out_f); break;
        default: PCU_LAUNCH(vg_geometry_kernel<unsigned long long>, blocks, kThreads, stream, (const unsigned long long*)ijk, n, g, out_v, out_f);
    }
    return PCU_B200_OK;
}

// ---- triangle-mesh voxelization and 3-D flood fill (voxelize.cuh) ------------------------------------------------
// Persistent CTAs of vx_test_kernel: enough to fill every SM (the kernel holds 16-32 KB of shared memory per CTA).
inline unsigned vx_test_blocks(const pcu_b200_workspace* ws) { return (unsigned)ws->sm_count * 6u; }

// Bounds, scan and the counting pass; read the counts (first synchronisation); the code records, sized by the accepted
// count, their sort and run heads; read the number of distinct codes (second synchronisation).
template <typename T>
int vx_build(pcu_b200_workspace* ws, pcu_b200_voxelize* h, const T* v, long long nv, const void* f, long long m, int fkind,
             const VxGeom& g, cudaStream_t stream) {
    const long long tiles = (m + kThreads - 1) / kThreads;
    struct { VxFace* faces; unsigned long long* local; unsigned long long* tile; VxCounts* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.faces = cv.take<VxFace>((size_t)m);
        sc.local = cv.take<unsigned long long>((size_t)m);
        sc.tile = cv.take<unsigned long long>((size_t)tiles);
        sc.counts = cv.take<VxCounts>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.counts, 0, sizeof(VxCounts), stream));
    PCU_LAUNCH((vx_bounds_kernel<T>), (unsigned)tiles, kThreads, stream, v, nv, f, fkind, m, g, sc.faces, sc.local, sc.tile, sc.counts);
    PCU_LAUNCH(vx_tiles_kernel, 1, 1024, stream, sc.tile, tiles, sc.counts);
    PCU_LAUNCH((vx_test_kernel<T, kVxCount>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
               (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr);
    VxCounts c;
    PCU_TRY(read_record(sc.counts, &c, stream));
    if (c.bad_corner) return bad_corners(c.bad_corner);
    if (c.bad_bounds)
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: %llu faces have a non-finite vertex or voxel index bounds outside "
                    "[-2^31, 2^31 - 2]", c.bad_bounds);
    if (!(c.cand_d < kVxMaxCandidates))
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: %.6g candidate voxels overflow a 64-bit count", c.cand_d);
    if (c.accepted >= 0x7fffffffull)
        return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: at most 2^31 - 2 (face, voxel) overlaps are supported, got %llu",
                    c.accepted);
    const long long na = (long long)c.accepted;
    h->recs = na;
    if (na == 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    struct { SortScratch<McRec> sort; unsigned char* head; unsigned* counts; } hb;
    const auto carve = [&](Carver& cv) {
        hb.sort.carve(cv, na);
        hb.head = cv.take<unsigned char>((size_t)na);
        hb.counts = cv.take<unsigned>(keep_count_words(na));
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "voxelization"));
    carve_at(h->block, carve);
    PCU_LAUNCH((vx_test_kernel<T, kVxCodes>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
               (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, hb.sort.a);
    McRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(hb.sort, na, 1, stream, &sorted));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(na), kThreads, stream, (const McRec*)sorted, na, hb.head);
    PCU_TRY(enqueue_keep_offsets(hb.head, na, hb.counts, &sc.counts->unique, stream));
    PCU_TRY(read_record(sc.counts, &c, stream));
    h->n = c.unique;
    h->sorted = sorted;
    h->head = hb.head;
    h->offsets = hb.counts;
    return PCU_B200_OK;
}

template <typename T>
int voxelize_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, const double size[3],
                            const double origin[3], pcu_b200_voxelize** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts || !size || !origin) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (m >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "voxelize_triangle_mesh: at most 2^31 - 2 faces are supported, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    // as in the reference, a NaN size passes here (it makes every face's bounds non-finite)
    if (size[0] <= 0.0 || size[1] <= 0.0 || size[2] <= 0.0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid voxel size");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    VxGeom g;
    for (int k = 0; k < 3; ++k) { g.o[k] = origin[k]; g.s[k] = size[k]; g.h[k] = size[k] / 2; }
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_voxelize* h) { return vx_build<T>(ws, h, v, nv, f, m, fkind, g, stream); }));
    out_counts[0] = (*out)->n;
    out_counts[1] = (*out)->recs;
    return PCU_B200_OK;
}

int voxelize_emit_device(pcu_b200_workspace* ws, const pcu_b200_voxelize* h, int32_t* out_ijk, cudaStream_t stream) {
    if (!ws || !h || !out_ijk) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "voxelization"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_LAUNCH(vx_decode_kernel, blocks_for(h->recs), kThreads, stream, h->sorted, h->recs, (const unsigned char*)h->head,
               (const unsigned*)h->offsets, (int*)out_ijk);
    return PCU_B200_OK;
}

// (T)fill_value as the reference's x86 build converts a double: cvttsd2si for the integers (truncation toward zero; NaN
// and values whose truncation is out of range give the "integer indefinite" INT_MIN), round to nearest for float.
template <typename T>
T ff_cast(double x) {
    if constexpr (std::is_same<T, int>::value) return (x > -2147483649.0 && x < 2147483648.0) ? (int)x : INT32_MIN;
    else if constexpr (std::is_same<T, long long>::value) return (x >= -0x1p63 && x < 0x1p63) ? (long long)x : LLONG_MIN;
    else return (T)x;
}

// Tiles of at most kFfTileMax voxels, sides powers of two: up to 32 along z, then up to 256 / tz along y, the rest along
// x, each no larger than the grid needs.
inline int ff_log2_cover(long long n, int cap_log2) {
    int l = 0;
    while (l < cap_log2 && (1ll << l) < n) ++l;
    return l;
}

template <typename T>
int ff_device(pcu_b200_workspace* ws, const T* grid, long long w, long long h, long long d, long long seed, double fill, T* out,
              cudaStream_t stream) {
    FfShape s;
    s.w = w; s.h = h; s.d = d; s.n = w * h * d; s.seed = seed;
    s.lz = ff_log2_cover(d, 5);
    s.ly = ff_log2_cover(h, 8 - s.lz);
    s.lx = ff_log2_cover(w, 10 - s.lz - s.ly);
    s.tz_n = (unsigned)((d + (1ll << s.lz) - 1) >> s.lz);
    s.ty_n = (unsigned)((h + (1ll << s.ly) - 1) >> s.ly);
    const long long tx_n = (w + (1ll << s.lx) - 1) >> s.lx;
    const long long tiles = tx_n * s.ty_n * s.tz_n;
    int* P = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { P = cv.take<int>((size_t)s.n); }));
    PCU_LAUNCH((ff_tile_kernel<T>), (unsigned)tiles, kThreads, stream, grid, s, P);
    PCU_LAUNCH((ff_cross_kernel<T>), (unsigned)tiles, kThreads, stream, grid, s, P);
    PCU_LAUNCH((ff_out_kernel<T>), blocks_for(s.n), kThreads, stream, grid, s.n, seed, ff_cast<T>(fill), P, out);
    return PCU_B200_OK;
}

int flood_fill_3d_device(pcu_b200_workspace* ws, const void* grid, int kind, long long w, long long h, long long d, long long sx,
                         long long sy, long long sz, double fill, void* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!grid || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (sx < 0 || sx >= w || sy < 0 || sy >= h || sz < 0 || sz >= d) return fail(PCU_B200_INVALID_ARGUMENT, "seed point must be inside grid");
    if (w > 0x7fffffffLL || h > 0x7fffffffLL || d > 0x7fffffffLL || w * h > 0x7fffffffLL || w * h * d > 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "flood_fill_3d: grids of at most 2^31 - 1 voxels are supported, got %lld x %lld x %lld", w, h, d);
    PCU_ON_DEVICE(ws);
    const long long seed = (sx * h + sy) * d + sz;
    switch (kind) {
        case PCU_B200_GRID_I32: return ff_device<int>(ws, (const int*)grid, w, h, d, seed, fill, (int*)out, stream);
        case PCU_B200_GRID_I64: return ff_device<long long>(ws, (const long long*)grid, w, h, d, seed, fill, (long long*)out, stream);
        case PCU_B200_GRID_F32: return ff_device<float>(ws, (const float*)grid, w, h, d, seed, fill, (float*)out, stream);
        case PCU_B200_GRID_F64: return ff_device<double>(ws, (const double*)grid, w, h, d, seed, fill, (double*)out, stream);
        default: return fail(PCU_B200_INVALID_ARGUMENT, "unknown grid kind %d", kind);
    }
}

// ---- watertight manifold remeshing (watertight.cuh) ---------------------------------------------------------------
// The grid of DESIGN.md §3: c = (lo + hi) / 2, L = 1.4 max_a (hi_a - lo_a), o = c - L / 2, every operation rounded.
struct WtFrame { double o[3], L; };

// Bounds of v (first synchronisation), then per depth the counting pass (one synchronisation) and, where its pair
// count reaches the resolution, the grid pass (one more): the depth, the occupancy bytes of its grid in *grid.
template <typename T>
int wt_depth_search(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, double resolution,
                    CallBlock& grid, WtFrame& fr, int& depth, cudaStream_t stream) {
    const long long tiles = (m + kThreads - 1) / kThreads;
    struct { VxFace* faces; unsigned long long* local; unsigned long long* tile; VxCounts* counts; WtBounds* bounds; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.faces = cv.take<VxFace>((size_t)m);
        sc.local = cv.take<unsigned long long>((size_t)m);
        sc.tile = cv.take<unsigned long long>((size_t)tiles);
        sc.counts = cv.take<VxCounts>(1);
        sc.bounds = cv.take<WtBounds>(1);
    }));
    WtBounds b;
    for (int k = 0; k < 3; ++k) { b.lo[k] = LLONG_MAX; b.hi[k] = LLONG_MIN; }
    b.bad = 0;
    PCU_CUDA(cudaMemcpyAsync(sc.bounds, &b, sizeof b, cudaMemcpyHostToDevice, stream));
    PCU_LAUNCH((wt_bounds_kernel<T>), (unsigned)std::min<long long>(blocks_for(nv), (long long)ws->sm_count * 8), kThreads, stream, v, nv,
               sc.bounds);
    PCU_TRY(read_record(sc.bounds, &b, stream));
    if (b.bad) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: v has %llu non-finite coordinates", b.bad);
    double ext = 0.0, c[3];
    for (int k = 0; k < 3; ++k) {
        const auto unord = [](long long x) { x = x >= 0 ? x : x ^ 0x7fffffffffffffffll; double d; std::memcpy(&d, &x, 8); return d; };
        const double lo = unord(b.lo[k]), hi = unord(b.hi[k]);
        const volatile double sum = lo + hi, width = hi - lo;
        c[k] = sum / 2.0;
        ext = std::max(ext, (double)width);
    }
    if (!(ext > 0.0)) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: the mesh has zero extent (every vertex is the same point)");
    const volatile double L = 1.4 * ext;
    fr.L = L;
    if (!std::isfinite(fr.L)) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: the mesh's extent %g overflows fp64", ext);
    for (int k = 0; k < 3; ++k) { const volatile double h = fr.L / 2.0; fr.o[k] = c[k] - h; }
    for (depth = kWtMinDepth;; ++depth) {
        const double s = std::ldexp(fr.L, -depth);
        VxGeom g;
        for (int k = 0; k < 3; ++k) { const volatile double hs = s / 2.0, ok = fr.o[k] + hs; g.o[k] = ok; g.s[k] = s; g.h[k] = hs; }
        PCU_CUDA(cudaMemsetAsync(sc.counts, 0, sizeof(VxCounts), stream));
        PCU_LAUNCH((vx_bounds_kernel<T>), (unsigned)tiles, kThreads, stream, v, nv, f, fkind, m, g, sc.faces, sc.local, sc.tile, sc.counts);
        PCU_LAUNCH(vx_tiles_kernel, 1, 1024, stream, sc.tile, tiles, sc.counts);
        PCU_LAUNCH((vx_test_kernel<T, kVxCount>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
                   (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr, (unsigned*)nullptr, 0);
        VxCounts cnt;
        PCU_TRY(read_record(sc.counts, &cnt, stream));
        if (cnt.bad_corner) return bad_corners(cnt.bad_corner);
        if (cnt.bad_bounds || !(cnt.cand_d < kVxMaxCandidates))   // not reached: the mesh lies inside the grid
            return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: voxel bounds out of range at depth %d", depth);
        if ((double)cnt.accepted < resolution && depth < kWtMaxDepth) continue;   // occupied <= accepted pairs
        const size_t bytes = (size_t)1 << (3 * depth);
        grid.reset();
        PCU_TRY(alloc_block(grid.p, bytes, stream, "make_mesh_watertight's occupancy grid"));
        PCU_CUDA(cudaMemsetAsync(grid.p, 0, bytes, stream));
        PCU_LAUNCH((vx_test_kernel<T, kVxGrid>), vx_test_blocks(ws), kThreads, stream, v, nv, f, fkind, m, g, (const VxFace*)sc.faces,
                   (const unsigned long long*)sc.local, (const unsigned long long*)sc.tile, sc.counts, (McRec*)nullptr, (unsigned*)grid.p, depth);
        PCU_TRY(read_record(sc.counts, &cnt, stream));
        if ((double)cnt.occupied >= resolution || depth == kWtMaxDepth) return PCU_B200_OK;
    }
}

// The exterior and the surface of the occupancy grid (two synchronisations: the counts, then nothing until the
// projection), into the handle's block: x (nv, 3) fp64 pre-projection vertices, faces (nf, 3) int32.
int wt_surface(pcu_b200_workspace* ws, pcu_b200_watertight* h, unsigned char* grid, int lg, const WtFrame& fr, CallBlock& dense,
               cudaStream_t stream) {
    const long long N = 1ll << lg, n = N * N * N;
    PCU_TRY(alloc_block(dense.p, sizeof(int) * (size_t)n, stream, "make_mesh_watertight's voxel labels"));
    int* P = (int*)dense.p;
    FfShape sh;
    sh.w = sh.h = sh.d = N; sh.n = n; sh.seed = 0;
    sh.lz = ff_log2_cover(N, 5);
    sh.ly = ff_log2_cover(N, 8 - sh.lz);
    sh.lx = ff_log2_cover(N, 10 - sh.lz - sh.ly);
    sh.tz_n = (unsigned)((N + (1ll << sh.lz) - 1) >> sh.lz);
    sh.ty_n = (unsigned)((N + (1ll << sh.ly) - 1) >> sh.ly);
    const long long ftiles = ((N + (1ll << sh.lx) - 1) >> sh.lx) * sh.ty_n * sh.tz_n;
    PCU_LAUNCH((ff_tile_kernel<unsigned char>), (unsigned)ftiles, kThreads, stream, (const unsigned char*)grid, sh, P);
    PCU_LAUNCH((ff_cross_kernel<unsigned char>), (unsigned)ftiles, kThreads, stream, (const unsigned char*)grid, sh, P);
    PCU_LAUNCH(wt_exterior_kernel, blocks_for(n), kThreads, stream, grid, n, P);
    const unsigned tiles = blocks_for(n);
    struct { unsigned* sum; unsigned long long* v0; unsigned long long* f0; McCounts* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sum = cv.take<unsigned>(tiles);
        sc.v0 = cv.take<unsigned long long>(tiles);
        sc.f0 = cv.take<unsigned long long>(tiles);
        sc.counts = cv.take<McCounts>(1);
    }));
    PCU_LAUNCH(wt_count_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, sc.sum);
    PCU_LAUNCH(mc_tiles_kernel, 1, 1024, stream, (const unsigned*)sc.sum, (long long)tiles, sc.v0, sc.f0, sc.counts);
    McCounts c;
    PCU_TRY(read_record(sc.counts, &c, stream));
    if (c.slots >= 0x7fffffffull || c.faces >= 0x7fffffffull)
        return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: at most 2^31 - 2 vertices and faces are supported, got %llu and %llu",
                    c.slots, c.faces);
    h->nv = (long long)c.slots;
    h->nf = (long long)c.faces;
    const auto carve = [&](Carver& cv) {
        h->x = cv.take<double>(3 * (size_t)h->nv);
        h->faces = cv.take<int>(3 * (size_t)h->nf);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "make_mesh_watertight"));
    carve_at(h->block, carve);
    WtPlace pl;
    for (int k = 0; k < 3; ++k) pl.o[k] = fr.o[k];
    pl.s = std::ldexp(fr.L, -lg);
    PCU_LAUNCH(wt_verts_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, (const unsigned long long*)sc.v0,
               (const unsigned long long*)sc.f0, pl, P, const_cast<double*>(h->x));
    PCU_LAUNCH(wt_faces_kernel, tiles, kThreads, stream, (const unsigned char*)grid, lg, n, (const unsigned long long*)sc.v0,
               (const unsigned long long*)sc.f0, (const int*)P, const_cast<int*>(h->faces));
    return PCU_B200_OK;
}

constexpr int kWtRounds = 10;

// The projection rounds of DESIGN.md §3 on h->x: the input's fp64 tree once, then per round the closest points, the
// proposals, flip passes until none is flipped (one synchronisation each) and the commit.
template <typename T>
int wt_project(pcu_b200_workspace* ws, pcu_b200_watertight* h, const T* v, long long nv, const void* f, long long m, int fkind,
               cudaStream_t stream) {
    const long long n = h->nv, nf = h->nf;
    if (n == 0) return PCU_B200_OK;
    struct { unsigned char* tree; double* v64; double* x0; double* y; double* alpha; int* rev; double* d; long long* fidx; double* bc;
             unsigned long long* flipped; } sc;
    MeshTree<Pt<double>> t;
    const auto carve = [&](Carver& cv) {
        sc.tree = cv.take<unsigned char>(carve_at(nullptr, [&](Carver& c2) { carve_mesh_tree<Pt<double>>(c2, m, false, t); }));
        sc.v64 = sizeof(T) == 8 ? nullptr : cv.take<double>(3 * (size_t)nv);
        sc.x0 = cv.take<double>(3 * (size_t)n);
        sc.y = cv.take<double>(3 * (size_t)n);
        sc.alpha = cv.take<double>((size_t)n);
        sc.rev = cv.take<int>((size_t)n);
        sc.d = cv.take<double>((size_t)n);
        sc.fidx = cv.take<long long>((size_t)n);
        sc.bc = cv.take<double>(3 * (size_t)n);
        sc.flipped = cv.take<unsigned long long>(2);
    };
    CallBlock blk(stream);
    PCU_TRY(alloc_block(blk.p, carve_at(nullptr, carve), stream, "make_mesh_watertight's projection"));
    carve_at(blk.p, carve);
    const double* v64 = (const double*)v;
    if (sizeof(T) != 8) {
        PCU_LAUNCH((wt_widen_kernel<T>), blocks_for(3 * nv), kThreads, stream, v, 3 * nv, sc.v64);
        v64 = sc.v64;
    }
    PCU_TRY(build_mesh_tree<double>(ws, v64, nv, f, m, fkind, false, sc.flipped + 1, stream, t, sc.tree));
    double* x = const_cast<double*>(h->x);
    const unsigned vb = blocks_for(n), fb = blocks_for(nf);
    PCU_LAUNCH(wt_start_kernel, vb, kThreads, stream, (const double*)x, n, sc.x0, sc.alpha);
    for (int round = 0; round < kWtRounds; ++round) {
        PCU_LAUNCH((mq_query_kernel<double>), query_blocks(ws, n), kThreads, stream, (const double*)x, n, m, (const MqScratch*)t.sc,
                   (const MqNode*)t.nodes, (const Pt<double>*)t.leaves, sc.d, (void*)sc.fidx, 1, sc.bc);
        PCU_LAUNCH(wt_propose_kernel, vb, kThreads, stream, v64, nv, f, fkind, (const long long*)sc.fidx, (const double*)sc.bc,
                   (const double*)x, (const double*)sc.alpha, n, sc.y);
        PCU_CUDA(cudaMemsetAsync(sc.rev, 0, sizeof(int) * (size_t)n, stream));
        for (int pass = 1;; ++pass) {
            PCU_CUDA(cudaMemsetAsync(sc.flipped, 0, sizeof(unsigned long long), stream));
            PCU_LAUNCH(wt_flip_kernel, fb, kThreads, stream, h->faces, nf, (const double*)sc.x0, (const double*)x, (const double*)sc.y,
                       sc.rev, pass, sc.flipped);
            unsigned long long flipped = 0;
            PCU_TRY(read_record(sc.flipped, &flipped, stream));
            if (flipped == 0) break;
        }
        PCU_LAUNCH(wt_commit_kernel, vb, kThreads, stream, (const double*)sc.y, (const int*)sc.rev, n, x, sc.alpha);
    }
    return PCU_B200_OK;
}

template <typename T>
int make_mesh_watertight_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind,
                                        double resolution, pcu_b200_watertight** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: at most 2^31 - 2 vertices and faces are supported");
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_watertight* h) -> int {
        h->t_f64 = sizeof(T) == 8;
        h->fkind = fkind;
        CallBlock grid(stream), dense(stream);
        WtFrame fr;
        PCU_TRY(wt_depth_search<T>(ws, v, nv, f, m, fkind, resolution, grid, fr, h->depth, stream));
        PCU_TRY(wt_surface(ws, h, grid.p, h->depth, fr, dense, stream));
        grid.reset();
        dense.reset();
        const long long most = fkind == kIdxI32 ? (1ll << 31) : fkind == kIdxU32 ? (1ll << 32) : LLONG_MAX;
        if (h->nv > most) return fail(PCU_B200_INVALID_ARGUMENT, "make_mesh_watertight: %lld vertices cannot be indexed by f's dtype", h->nv);
        return wt_project<T>(ws, h, v, nv, f, m, fkind, stream);
    }));
    out_counts[0] = (*out)->nv;
    out_counts[1] = (*out)->nf;
    out_counts[2] = (*out)->depth;
    return PCU_B200_OK;
}

int make_mesh_watertight_emit_device(pcu_b200_workspace* ws, const pcu_b200_watertight* h, void* out_v, void* out_f, cudaStream_t stream) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "watertight"));
    if (h->nv == 0 && h->nf == 0) return PCU_B200_OK;
    if (!out_v || !out_f) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(3 * std::max(h->nv, h->nf));
    if (h->t_f64) PCU_LAUNCH(wt_emit_kernel<double>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->nf, (int)wide_index(h->fkind), (double*)out_v, out_f);
    else PCU_LAUNCH(wt_emit_kernel<float>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->nf, (int)wide_index(h->fkind), (float*)out_v, out_f);
    return PCU_B200_OK;
}

// ---- mesh connected components and vertex removal (mesh_topology.cuh) ----------------------------------------------
// Persistent CTAs of cc_validate_kernel.
inline unsigned cc_validate_blocks(const pcu_b200_workspace* ws, long long total) {
    return (unsigned)std::max(1ll, std::min((long long)ws->sm_count * 8, (total + kThreads - 1) / kThreads));
}

// Validate f and read max(f) (first synchronisation); the labels and counts in the handle's block; read the component
// count (second synchronisation).
int cc_build(pcu_b200_workspace* ws, pcu_b200_components* h, const void* f, long long m, int c, int fkind, cudaStream_t stream) {
    CcCounts* rec = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { rec = cv.take<CcCounts>(1); }));
    PCU_CUDA(cudaMemsetAsync(rec, 0, sizeof(CcCounts), stream));
    const long long total = m * c;
    PCU_LAUNCH(cc_validate_kernel, cc_validate_blocks(ws, total), kThreads, stream, f, fkind, total, rec);
    CcCounts hc;
    PCU_TRY(read_record(rec, &hc, stream));
    if (hc.bad)
        return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: %llu face indices are negative or above 2^31 - 2", hc.bad);
    const long long n = (long long)hc.max_index + 1;
    struct { int *P, *root, *rank, *nv, *nf, *cf; unsigned char* is_root; unsigned* counts; } b;
    const auto carve = [&](Carver& cv) {
        b.P = cv.take<int>((size_t)n);
        b.root = cv.take<int>((size_t)n);
        b.rank = cv.take<int>((size_t)n);
        b.nv = cv.take<int>((size_t)n);
        b.nf = cv.take<int>((size_t)n);
        b.cf = cv.take<int>((size_t)m);
        b.is_root = cv.take<unsigned char>((size_t)n);
        b.counts = cv.take<unsigned>(keep_count_words(n));
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "connected components"));
    carve_at(h->block, carve);
    PCU_CUDA(cudaMemsetAsync(b.nv, 0, sizeof(int) * (size_t)n, stream));
    PCU_CUDA(cudaMemsetAsync(b.nf, 0, sizeof(int) * (size_t)n, stream));
    PCU_LAUNCH(cc_init_kernel, blocks_for(n), kThreads, stream, b.P, n);
    PCU_LAUNCH(cc_hook_kernel, blocks_for(m), kThreads, stream, f, fkind, m, c, b.P);
    PCU_LAUNCH(cc_flatten_kernel, blocks_for(n), kThreads, stream, b.P, n, b.root, b.is_root);
    PCU_TRY(enqueue_keep_offsets(b.is_root, n, b.counts, &rec->ncomp, stream));
    PCU_LAUNCH(cc_rank_kernel, blocks_for(n), kThreads, stream, (const unsigned char*)b.is_root, n, (const unsigned*)b.counts, b.rank);
    PCU_LAUNCH(cc_label_kernel, blocks_for(n), kThreads, stream, b.root, n, (const int*)b.rank, b.nv);
    PCU_LAUNCH(cc_face_kernel, blocks_for(m), kThreads, stream, f, fkind, m, c, (const int*)b.root, b.cf, b.nf);
    PCU_TRY(read_record(rec, &hc, stream));
    h->n = n;
    h->m = m;
    h->k = hc.ncomp;
    h->cv = b.root;
    h->cf = b.cf;
    h->nv = b.nv;
    h->nf = b.nf;
    return PCU_B200_OK;
}

int connected_components_prepare_device(pcu_b200_workspace* ws, const void* f, long long m, int c, int fkind, pcu_b200_components** out,
                                        long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (m <= 0 || c <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: f must have at least one row and one column");
    if (m >= 0x7fffffffLL || m * c >= (1ll << 40))
        return fail(PCU_B200_INVALID_ARGUMENT, "connected_components: at most 2^31 - 2 faces are supported, got %lld x %d", m, c);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_components* h) {
        h->fkind = fkind;
        return cc_build(ws, h, f, m, c, fkind, stream);
    }));
    out_counts[0] = (*out)->n;
    out_counts[1] = (*out)->k;
    return PCU_B200_OK;
}

int connected_components_emit_device(pcu_b200_workspace* ws, const pcu_b200_components* h, void* out_cv, void* out_nv, void* out_cf,
                                     void* out_nf, cudaStream_t stream) {
    if (!ws || !h || !out_cv || !out_nv || !out_cf || !out_nf) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "components"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(std::max(h->n, h->m));
    if (wide_index(h->fkind))
        PCU_LAUNCH(cc_emit_kernel<long long>, blocks, kThreads, stream, h->cv, h->n, h->cf, h->m, h->nv, h->nf, h->k, (long long*)out_cv,
                   (long long*)out_cf, (long long*)out_nv, (long long*)out_nf);
    else
        PCU_LAUNCH(cc_emit_kernel<int>, blocks, kThreads, stream, h->cv, h->n, h->cf, h->m, h->nv, h->nf, h->k, (int*)out_cv, (int*)out_cf,
                   (int*)out_nv, (int*)out_nf);
    return PCU_B200_OK;
}

// Arguments shared by the two removals.
int mt_check(const pcu_b200_workspace* ws, const void* v, long long nv, const void* f, long long m, int fkind) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m >= 0x7fffffffLL)
        return fail(PCU_B200_INVALID_ARGUMENT, "at most 2^31 - 2 vertices and faces are supported, got %lld and %lld", nv, m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

template <typename T>
int remove_mesh_vertices_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind,
                                const unsigned char* mask, T* out_v, void* out_f, long long* out_counts, cudaStream_t stream) {
    PCU_TRY(mt_check(ws, v, nv, f, m, fkind));
    if (fkind != kIdxI32 && fkind != kIdxI64) return fail(PCU_B200_INVALID_ARGUMENT, "remove_mesh_vertices: f must be int32 or int64");
    if (!mask || !out_v || !out_f || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    struct { MtCounts* rec; int* remap; unsigned* vcounts; unsigned char* keep; unsigned* fcounts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MtCounts>(1);
        sc.remap = cv.take<int>((size_t)nv);
        sc.vcounts = cv.take<unsigned>(keep_count_words(nv));
        sc.keep = cv.take<unsigned char>((size_t)m);
        sc.fcounts = cv.take<unsigned>(keep_count_words(m));
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MtCounts), stream));
    PCU_TRY(enqueue_keep_offsets(mask, nv, sc.vcounts, &sc.rec->kept_v, stream));
    PCU_LAUNCH(rmv_vertex_kernel<T>, blocks_for(nv), kThreads, stream, v, nv, mask, (const unsigned*)sc.vcounts, out_v, sc.remap);
    PCU_LAUNCH(rmv_face_flag_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const int*)sc.remap, sc.keep, sc.rec);
    PCU_TRY(enqueue_keep_offsets(sc.keep, m, sc.fcounts, &sc.rec->kept_f, stream));
    if (wide_index(fkind))
        PCU_LAUNCH(rmv_face_emit_kernel<long long>, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const unsigned char*)sc.keep,
                   (const unsigned*)sc.fcounts, (const int*)sc.remap, (long long*)out_f);
    else
        PCU_LAUNCH(rmv_face_emit_kernel<int>, blocks_for(m), kThreads, stream, f, fkind, m, nv, (const unsigned char*)sc.keep,
                   (const unsigned*)sc.fcounts, (const int*)sc.remap, (int*)out_f);
    MtCounts hc;
    PCU_TRY(read_record(sc.rec, &hc, stream));
    if (hc.bad) return bad_corners(hc.bad);
    out_counts[0] = hc.kept_v;
    out_counts[1] = hc.kept_f;
    return PCU_B200_OK;
}

template <typename T, typename I>
int rur_launch(const T* v, long long nv, const void* f, long long m, int fkind, const unsigned char* used, const unsigned* vcounts,
               T* out_v, void* out_f, void* out_j, void* out_i, cudaStream_t stream) {
    PCU_LAUNCH((rur_vertex_kernel<T, I>), blocks_for(nv), kThreads, stream, v, nv, used, vcounts, out_v, (I*)out_j, (I*)out_i);
    PCU_LAUNCH(rur_face_kernel<I>, blocks_for(3 * m), kThreads, stream, f, fkind, 3 * m, nv, (const I*)out_i, (I*)out_f);
    return PCU_B200_OK;
}

template <typename T>
int remove_unreferenced_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, T* out_v,
                               void* out_f, void* out_j, void* out_i, long long* out_count, cudaStream_t stream) {
    PCU_TRY(mt_check(ws, v, nv, f, m, fkind));
    if (!out_v || !out_f || !out_j || !out_i || !out_count) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    struct { MtCounts* rec; unsigned char* used; unsigned* vcounts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MtCounts>(1);
        sc.used = cv.take<unsigned char>((size_t)nv);
        sc.vcounts = cv.take<unsigned>(keep_count_words(nv));
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MtCounts), stream));
    PCU_CUDA(cudaMemsetAsync(sc.used, 0, (size_t)nv, stream));
    PCU_LAUNCH(rur_mark_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, sc.used, sc.rec);
    PCU_TRY(enqueue_keep_offsets(sc.used, nv, sc.vcounts, &sc.rec->kept_v, stream));
    if (wide_index(fkind))
        PCU_TRY((rur_launch<T, long long>(v, nv, f, m, fkind, sc.used, sc.vcounts, out_v, out_f, out_j, out_i, stream)));
    else
        PCU_TRY((rur_launch<T, int>(v, nv, f, m, fkind, sc.used, sc.vcounts, out_v, out_f, out_j, out_i, stream)));
    MtCounts hc;
    PCU_TRY(read_record(sc.rec, &hc, stream));
    if (hc.bad) return bad_corners(hc.bad);
    *out_count = hc.kept_v;
    return PCU_B200_OK;
}

// ---- consistent face orientation (orient.cuh) ----------------------------------------------------------------------
// K = the half-edge records' word, I = f's width.  Every buffer is sized by m: no synchronisation.
template <typename K, typename I>
int orient_launch(pcu_b200_workspace* ws, const void* f, long long m, int fkind, I* out_f, I* out_c, cudaStream_t stream) {
    using Rec = OmRec<K>;
    const long long n = 3 * m;
    struct { SortScratch<Rec> sort; int *P, *nb, *root, *rank, *next; unsigned char *flag, *enq; unsigned* counts; long long* seeds; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.P = cv.take<int>(2 * (size_t)m);
        sc.nb = cv.take<int>((size_t)n);
        sc.root = cv.take<int>((size_t)m);
        sc.rank = cv.take<int>((size_t)m);
        sc.next = cv.take<int>((size_t)m);
        sc.flag = cv.take<unsigned char>((size_t)m);
        sc.enq = cv.take<unsigned char>((size_t)m);
        sc.counts = cv.take<unsigned>(keep_count_words(m));
        sc.seeds = cv.take<long long>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.nb, 0xff, sizeof(int) * (size_t)n, stream));
    PCU_CUDA(cudaMemsetAsync(sc.enq, 0, (size_t)m, stream));
    PCU_LAUNCH(om_records_kernel<K>, blocks_for(m), kThreads, stream, f, fkind, m, sc.sort.a, sc.P);
    Rec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 2, stream, &sorted));
    PCU_LAUNCH(om_runs_kernel<K>, blocks_for(n), kThreads, stream, (const Rec*)sorted, n, m, f, fkind, sc.nb, sc.P);
    PCU_LAUNCH(om_flatten_kernel, blocks_for(m), kThreads, stream, sc.P, m, sc.root, sc.flag);
    PCU_TRY(enqueue_keep_offsets(sc.flag, m, sc.counts, sc.seeds, stream));
    PCU_LAUNCH(cc_rank_kernel, blocks_for(m), kThreads, stream, (const unsigned char*)sc.flag, m, (const unsigned*)sc.counts, sc.rank);
    PCU_LAUNCH(om_emit_kernel<I>, blocks_for(m), kThreads, stream, (const I*)f, m, (const int*)sc.root, (const int*)sc.rank, out_f, out_c);
    PCU_LAUNCH(om_replay_kernel<I>, blocks_for(m), kThreads, stream, (const unsigned char*)sc.flag, m, (const int*)sc.nb, sc.enq, sc.next,
               out_f);
    return PCU_B200_OK;
}

int orient_mesh_faces_device(pcu_b200_workspace* ws, const void* f, long long m, int fkind, void* out_f, void* out_c, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!f || !out_f || !out_c) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (m <= 0 || m > kOmMaxFaces)
        return fail(PCU_B200_INVALID_ARGUMENT, "orient_mesh_faces: between 1 and 2^30 - 1 faces are supported, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    return wide_index(fkind) ? orient_launch<unsigned long long, long long>(ws, f, m, fkind, (long long*)out_f, (long long*)out_c, stream)
                             : orient_launch<unsigned, int>(ws, f, m, fkind, (int*)out_f, (int*)out_c, stream);
}

// ---- mesh normals, face areas and Laplacian smoothing (mesh_geometry.cuh, laplacian.cuh) ---------------------------
// Arguments shared by the four entry points.  6 m records must fit int32 positions.
int mg_check(const pcu_b200_workspace* ws, const void* v, long long nv, const void* f, long long m, int fkind, const void* out) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!v || !f || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv >= 0x7fffffffLL || m > 0x7fffffffLL / 6)
        return fail(PCU_B200_INVALID_ARGUMENT, "at most 2^31 - 2 vertices and 357913941 faces are supported, got %lld and %lld", nv, m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    return PCU_B200_OK;
}

// CTAs of the kernels that reduce (reduce_grid): a function of the row count alone, so the sums' order is too.
inline unsigned mg_blocks(long long n) { return std::min<unsigned>(kMgBlocks, blocks_for(n)); }

// Bits of the largest vertex index n - 1 (at least 1).
inline int mg_index_bits(long long n) {
    int b = 1;
    while (b < 31 && ((n - 1) >> b) != 0) ++b;
    return b;
}

// One face pass over v (T = the type of v; double for the smoothing's fp64 iterate).
template <typename T>
int mg_face_pass(const T* v, long long nv, const void* f, int fkind, long long m, const FaceOut<T>& out, MgRecord* rec, cudaStream_t stream) {
    PCU_LAUNCH(mg_face_kernel<T>, mg_blocks(m), kThreads, stream, v, nv, f, fkind, m, out, rec);
    return PCU_B200_OK;
}

// The corner CSR of the nv vertices: first (nv + 1) and corner (3 m), through the stable sort of the corner records
// (sort: scratch for at least 3 m records).
int enqueue_incidence(const SortScratch<MgRec>& sort, const void* f, int fkind, long long m, long long nv, int* first, int* corner,
                      cudaStream_t stream) {
    const long long n = 3 * m;
    PCU_LAUNCH(mg_corner_kernel, blocks_for(n), kThreads, stream, f, fkind, n, nv, sort.a);
    MgRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sort, n, 1, stream, &sorted, mg_index_bits(nv)));
    PCU_LAUNCH(mg_rows_kernel, blocks_for(n + 1), kThreads, stream, (const MgRec*)sorted, n, nv, first, corner, 0);
    return PCU_B200_OK;
}

// mesh_face_areas (normal == false) or estimate_mesh_face_normals (normal == true): one face pass, one synchronisation.
template <typename T>
int mesh_face_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, bool normal, T* out,
                     cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    PCU_ON_DEVICE(ws);
    MgRecord* rec = nullptr;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { rec = cv.take<MgRecord>(1); }));
    PCU_CUDA(cudaMemsetAsync(rec, 0, sizeof(MgRecord), stream));
    FaceOut<T> o = {};
    if (normal) o.normal = out; else o.area = out;
    PCU_TRY(mg_face_pass<T>(v, nv, f, fkind, m, o, rec, stream));
    MgRecord host;
    PCU_TRY(read_record(rec, &host, stream));
    return host.bad ? bad_corners(host.bad) : PCU_B200_OK;
}

// estimate_mesh_vertex_normals, weighting 0 uniform, 1 area, 2 angle: face pass, corner CSR, vertex pass; one
// synchronisation.
template <typename T>
int vertex_normals_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, int weighting, T* out,
                          cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    if (weighting < 0 || weighting > 2) return fail(PCU_B200_INVALID_ARGUMENT, "unknown weighting %d", weighting);
    PCU_ON_DEVICE(ws);
    struct { MgRecord* rec; double *unit, *weight; SortScratch<MgRec> sort; int *first, *corner; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<MgRecord>(1);
        sc.unit = cv.take<double>(3 * (size_t)m);
        sc.weight = weighting ? cv.take<double>(3 * (size_t)m) : nullptr;
        sc.sort.carve(cv, 3 * m);
        sc.first = cv.take<int>((size_t)nv + 1);
        sc.corner = cv.take<int>(3 * (size_t)m);
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(MgRecord), stream));
    FaceOut<T> o = {};
    o.unit = sc.unit;
    o.weight = sc.weight;
    o.weighting = weighting;
    PCU_TRY(mg_face_pass<T>(v, nv, f, fkind, m, o, sc.rec, stream));
    PCU_TRY(enqueue_incidence(sc.sort, f, fkind, m, nv, sc.first, sc.corner, stream));
    PCU_LAUNCH(mg_vertex_normal_kernel<T>, blocks_for(nv), kThreads, stream, (const int*)sc.first, (const int*)sc.corner, nv,
               (const double*)sc.unit, (const double*)sc.weight, out);
    MgRecord host;
    PCU_TRY(read_record(sc.rec, &host, stream));
    return host.bad ? bad_corners(host.bad) : PCU_B200_OK;
}

constexpr int kCgWindow = 16;   // CG iterations enqueued between two reads of the solver's record

// The buffers of one smoothing call.
struct LapScratch {
    LapRecord* rec;
    double *u, *r, *z, *p, *q, *mass, *halfcot, *dbla, *partial, *val, *diag;
    SortScratch<MgRec> sort;
    MgRec* rows;
    unsigned char *head, *lone;
    unsigned* counts;
    int *col, *rowptr, *first, *corner;
    void carve(Carver& cv, long long nv, long long m, bool cotan) {
        const size_t n3 = 3 * (size_t)nv, e = 6 * (size_t)m;
        rec = cv.take<LapRecord>(1);
        u = cv.take<double>(n3); r = cv.take<double>(n3); z = cv.take<double>(n3); p = cv.take<double>(n3); q = cv.take<double>(n3);
        mass = cotan ? cv.take<double>((size_t)nv) : nullptr;
        halfcot = cv.take<double>(3 * (size_t)m);
        dbla = cotan ? cv.take<double>((size_t)m) : nullptr;
        partial = cv.take<double>((size_t)kMgBlocks * 9);
        sort.carve(cv, (long long)e);
        rows = cv.take<MgRec>(e);
        head = cv.take<unsigned char>(e);
        counts = cv.take<unsigned>(keep_count_words((long long)e));
        col = cv.take<int>(e);
        val = cv.take<double>(e);
        rowptr = cv.take<int>((size_t)nv + 1);
        diag = cv.take<double>((size_t)nv);
        lone = cv.take<unsigned char>((size_t)nv);
        first = cotan ? cv.take<int>((size_t)nv + 1) : nullptr;
        corner = cotan ? cv.take<int>(3 * (size_t)m) : nullptr;
    }
};

// Reads the record (one synchronisation) and fails on a mesh of zero total area.
int lap_read(const LapRecord* rec, LapRecord* host, cudaStream_t stream) {
    PCU_TRY(read_record(rec, host, stream));
    if (host->mesh.zero_area) return fail(PCU_B200_INVALID_ARGUMENT, "laplacian_smooth_mesh: the mesh has zero total area");
    return PCU_B200_OK;
}

// The cotangent Laplacian of u in the scratch's CSR; reads the record once (corners, finiteness, entries).
int lap_assemble(LapScratch& s, const void* f, int fkind, long long m, long long nv, bool cotan, cudaStream_t stream) {
    const long long e = 6 * m;
    const int bits = mg_index_bits(nv);
    FaceOut<double> o = {};
    o.halfcot = s.halfcot;
    PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
    PCU_LAUNCH(lap_edge_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, bits, s.sort.a);
    MgRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(s.sort, e, 1, stream, &sorted, 2 * bits));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(e), kThreads, stream, (const McRec*)sorted, e, s.head);
    PCU_TRY(enqueue_keep_offsets(s.head, e, s.counts, &s.rec->mesh.nnz, stream));
    PCU_LAUNCH(lap_entries_kernel, blocks_for(e), kThreads, stream, (const MgRec*)sorted, e, (const unsigned char*)s.head,
               (const unsigned*)s.counts, (const double*)s.halfcot, bits, s.rows, s.col, s.val);
    if (cotan) PCU_TRY(enqueue_incidence(s.sort, f, fkind, m, nv, s.first, s.corner, stream));
    LapRecord host;
    PCU_TRY(lap_read(s.rec, &host, stream));
    if (host.mesh.bad) return bad_corners(host.mesh.bad);
    if (host.mesh.nonfinite)
        return fail(PCU_B200_INVALID_ARGUMENT, "laplacian_smooth_mesh: v has %llu coordinates that are not finite", host.mesh.nonfinite);
    PCU_LAUNCH(mg_rows_kernel, blocks_for(host.mesh.nnz + 1), kThreads, stream, (const MgRec*)s.rows, host.mesh.nnz, nv, s.rowptr,
               (int*)nullptr, 0);
    PCU_LAUNCH(lap_diag_kernel, blocks_for(nv), kThreads, stream, (const int*)s.rowptr, (const double*)s.val, nv, s.diag, s.lone);
    return PCU_B200_OK;
}

// One CG solve of S u' = M u in place; reads the record once per window of kCgWindow iterations.  Returns the
// iterations and the largest |r| / |b| of the three columns at exit.
int lap_solve(const LapScratch& s, const LapSystem& sys, int max_iters, int* out_iters, double* out_residual, cudaStream_t stream) {
    const long long n = sys.n;
    const unsigned blocks = mg_blocks(n);
    PCU_CUDA(cudaMemsetAsync(&s.rec->cg, 0, sizeof(CgState), stream));
    PCU_LAUNCH(lap_cg_init_kernel, blocks, kThreads, stream, sys, (const double*)s.u, s.r, s.z, s.p, s.partial, s.rec);
    LapRecord host;
    for (;;) {
        for (int k = 0; k < kCgWindow; ++k) {
            PCU_LAUNCH(lap_cg_spmv_kernel, blocks, kThreads, stream, sys, (const double*)s.p, s.q, s.partial, s.rec);
            PCU_LAUNCH(lap_cg_update_kernel, blocks, kThreads, stream, sys, s.u, s.r, s.z, (const double*)s.p, (const double*)s.q, s.partial,
                       max_iters, s.rec);
            PCU_LAUNCH(lap_cg_direction_kernel, blocks_for(3 * n), kThreads, stream, n, (const double*)s.z, s.p, (const LapRecord*)s.rec);
        }
        PCU_TRY(lap_read(s.rec, &host, stream));
        if (host.cg.done) break;
    }
    double worst = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double rr = host.cg.rr[c], bb = host.cg.bb[c];
        const double rel = bb > 0.0 ? std::sqrt(rr / bb) : (rr > 0.0 ? HUGE_VAL : 0.0);
        worst = std::max(worst, rel);
    }
    *out_iters = host.cg.iters;
    *out_residual = worst;
    return PCU_B200_OK;
}

// laplacian_smooth_mesh (src/smooth.cpp): out_iters / out_residual (host, num_iters entries) receive every step's CG
// iterations and its largest relative residual at exit.
template <typename T>
int laplacian_smooth_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, int num_iters,
                            double step_size, bool cotan, int max_cg_iters, T* out, int* out_iters, double* out_residual, cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out));
    if (num_iters < 0)
        return fail(PCU_B200_INVALID_ARGUMENT, "Invalid value for argument num_iters in smooth_mesh_laplacian. Must be a positive integer or 0.");
    if (max_cg_iters <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_cg_iters must be positive, got %d", max_cg_iters);
    if (num_iters > 0 && (!out_iters || !out_residual)) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_ON_DEVICE(ws);
    if (num_iters == 0) {
        PCU_TRY(adopt_stream(ws, stream));
        PCU_CUDA(cudaMemcpyAsync(out, v, 3 * (size_t)nv * sizeof(T), cudaMemcpyDeviceToDevice, stream));
        return PCU_B200_OK;
    }
    LapScratch s;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) { s.carve(cv, nv, m, cotan); }));
    PCU_CUDA(cudaMemsetAsync(s.rec, 0, sizeof(LapRecord), stream));
    PCU_LAUNCH(lap_load_kernel<T>, blocks_for(3 * nv), kThreads, stream, v, 3 * nv, s.u, &s.rec->mesh);
    PCU_TRY(lap_assemble(s, f, fkind, m, nv, cotan, stream));
    const LapSystem sys = {s.rowptr, s.col, s.val, s.diag, s.mass, cotan ? step_size * 1e-3 : step_size, nv};
    for (int it = 0; it < num_iters; ++it) {
        if (cotan) {
            FaceOut<double> o = {};
            o.dbla = s.dbla;
            o.partial = s.partial;
            PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
            PCU_LAUNCH(lap_mass_kernel, blocks_for(nv), kThreads, stream, (const int*)s.first, (const int*)s.corner, nv, (const double*)s.dbla,
                       (const unsigned char*)s.lone, s.mass);
        }
        PCU_TRY(lap_solve(s, sys, max_cg_iters, out_iters + it, out_residual + it, stream));
        if (cotan) {
            FaceOut<double> o = {};
            o.partial = s.partial;
            PCU_TRY(mg_face_pass<double>(s.u, nv, f, fkind, m, o, &s.rec->mesh, stream));
            PCU_LAUNCH(lap_rescale_kernel, blocks_for(3 * nv), kThreads, stream, s.u, nv, (const MgRecord*)&s.rec->mesh);
        }
    }
    PCU_LAUNCH(lap_store_kernel<T>, blocks_for(3 * nv), kThreads, stream, (const double*)s.u, 3 * nv, out);
    if (cotan) {
        LapRecord host;
        PCU_TRY(lap_read(s.rec, &host, stream));
    }
    return PCU_B200_OK;
}

}  // namespace

// =================================================================================================
extern "C" {

int pcu_b200_voronoi_centroids(pcu_b200_workspace* ws, const double* centers, int64_t n, int dim, double* out_centroids,
                               double* out_moments, int64_t* out_passes, void* stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(vor_check(n, dim));
    if (n <= 0 || !centers || !out_centroids) return fail(PCU_B200_INVALID_ARGUMENT, "voronoi: n >= 1 seeds and non-null pointers required");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    const int rs = dim == 3 ? voronoi_centroids_device<3>(ws, centers, n, out_centroids, out_moments, passes, (cudaStream_t)stream)
                            : voronoi_centroids_device<2>(ws, centers, n, out_centroids, out_moments, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    return rs;
}
int pcu_b200_lloyd(pcu_b200_workspace* ws, int64_t n, int dim, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                   double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    PCU_TRY(vor_check(n, dim));
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "n must be a positive integer. Got n = %lld", (long long)n);
    if (!out_points) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    int steps = 0;
    const int rs = dim == 3 ? lloyd_device<3>(ws, n, seed, num_lloyd, num_newton, out_points, out_energy, &steps, passes, (cudaStream_t)stream)
                            : lloyd_device<2>(ws, n, seed, num_lloyd, num_newton, out_points, out_energy, &steps, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    if (out_newton_steps) *out_newton_steps = steps;
    return rs;
}

int pcu_b200_restricted_voronoi_moments(pcu_b200_workspace* ws, const double* seeds, int64_t n, const double* v, int64_t nv,
                                        const void* f, int64_t nf, int f_kind, double* out_moments, int64_t* out_passes, void* stream) {
    PCU_TRY(rv_check(ws, v, nv, f, nf, f_kind, n));
    if (!seeds || !out_moments) return fail(PCU_B200_INVALID_ARGUMENT, "null seeds or output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    const int rs = restricted_moments_device(ws, seeds, n, v, nv, f, nf, f_kind, out_moments, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    return rs;
}
int pcu_b200_sample_mesh_lloyd(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                               int64_t num_samples, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                               double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream) {
    PCU_TRY(rv_check(ws, v, nv, f, nf, f_kind, num_samples));
    if (!out_points) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    long long passes[3] = {0, 0, 0};
    int steps = 0;
    const int rs = sample_mesh_lloyd_device(ws, v, nv, f, nf, f_kind, num_samples, seed, num_lloyd, num_newton, out_points, out_energy,
                                            &steps, passes, (cudaStream_t)stream);
    if (out_passes) for (int i = 0; i < 3; ++i) out_passes[i] = passes[i];
    if (out_newton_steps) *out_newton_steps = steps;
    return rs;
}

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

int pcu_b200_marching_cubes_prepare_f32(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const float* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream) {
    return marching_cubes_prepare_device<float>(ws, scalars, scalars_f64, coords, n, cube_idx, m, idx_kind, isovalue, out_mc,
                                                (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_prepare_f64(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const double* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream) {
    return marching_cubes_prepare_device<double>(ws, scalars, scalars_f64, coords, n, cube_idx, m, idx_kind, isovalue, out_mc,
                                                 (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_emit(pcu_b200_workspace* ws, const pcu_b200_marching_cubes* mc, void* out_v, void* out_f, void* stream) {
    return marching_cubes_emit_device(ws, mc, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_marching_cubes_destroy(pcu_b200_marching_cubes* mc) {
    if (!mc) return PCU_B200_OK;
    DeviceGuard guard(mc->device);
    delete mc;
    return PCU_B200_OK;
}
int pcu_b200_sparse_voxel_grid_boundary(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, int64_t* out_idx,
                                        int64_t* out_counts, void* stream) {
    return sparse_voxel_grid_boundary_device(ws, grid, n, idx_kind, (long long*)out_idx, (long long*)out_counts, (cudaStream_t)stream);
}

int pcu_b200_sparse_grid_from_points_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream) {
    return svg_points_prepare<float>(ws, points, n, voxel_size, origin, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_from_points_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream) {
    return svg_points_prepare<double>(ws, points, n, voxel_size, origin, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_dilate_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, pcu_b200_sparse_grid** out_grid,
                                        int64_t out_counts[2], void* stream) {
    return svg_dilate_prepare(ws, grid, n, idx_kind, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_hex_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, const double voxel_size[3],
                                     const double origin[3], int vertices_f64, pcu_b200_sparse_grid** out_grid, int64_t out_counts[2],
                                     void* stream) {
    return svg_hex_prepare(ws, grid, n, idx_kind, voxel_size, origin, vertices_f64, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_emit(pcu_b200_workspace* ws, const pcu_b200_sparse_grid* sg, void* out_rows, int64_t* out_index, void* stream) {
    return svg_emit(ws, sg, out_rows, out_index, (cudaStream_t)stream);
}
int pcu_b200_sparse_grid_destroy(pcu_b200_sparse_grid* sg) {
    if (!sg) return PCU_B200_OK;
    DeviceGuard guard(sg->device);
    delete sg;
    return PCU_B200_OK;
}
int pcu_b200_sparse_grid_erode(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, void* out_grid, int64_t* out_counts,
                               void* stream) {
    return svg_erode(ws, grid, n, idx_kind, out_grid, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_voxel_grid_geometry(pcu_b200_workspace* ws, const void* ijk, int64_t n, int idx_kind, const double voxel_size[3],
                                 const double voxel_origin[3], double gap_fraction, float* out_v, int32_t* out_f, void* stream) {
    return voxel_grid_geometry_device(ws, ijk, n, idx_kind, voxel_size, voxel_origin, gap_fraction, out_v, out_f, (cudaStream_t)stream);
}

int pcu_b200_voxelize_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream) {
    return voxelize_prepare_device<float>(ws, v, nv, f, nf, f_kind, voxel_size, voxel_origin, out_vx, (long long*)out_counts,
                                          (cudaStream_t)stream);
}
int pcu_b200_voxelize_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream) {
    return voxelize_prepare_device<double>(ws, v, nv, f, nf, f_kind, voxel_size, voxel_origin, out_vx, (long long*)out_counts,
                                           (cudaStream_t)stream);
}
int pcu_b200_voxelize_emit(pcu_b200_workspace* ws, const pcu_b200_voxelize* vx, int32_t* out_ijk, void* stream) {
    return voxelize_emit_device(ws, vx, out_ijk, (cudaStream_t)stream);
}
int pcu_b200_voxelize_destroy(pcu_b200_voxelize* vx) {
    if (!vx) return PCU_B200_OK;
    DeviceGuard guard(vx->device);
    delete vx;
    return PCU_B200_OK;
}
int pcu_b200_flood_fill_3d(pcu_b200_workspace* ws, const void* grid, int grid_kind, int64_t w, int64_t h, int64_t d, int64_t seed_x,
                           int64_t seed_y, int64_t seed_z, double fill_value, void* out, void* stream) {
    return flood_fill_3d_device(ws, grid, grid_kind, w, h, d, seed_x, seed_y, seed_z, fill_value, out, (cudaStream_t)stream);
}

int pcu_b200_make_mesh_watertight_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream) {
    return make_mesh_watertight_prepare_device<float>(ws, v, nv, f, nf, f_kind, resolution, out_wt, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream) {
    return make_mesh_watertight_prepare_device<double>(ws, v, nv, f, nf, f_kind, resolution, out_wt, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_emit(pcu_b200_workspace* ws, const pcu_b200_watertight* wt, void* out_v, void* out_f, void* stream) {
    return make_mesh_watertight_emit_device(ws, wt, out_v, out_f, (cudaStream_t)stream);
}
int pcu_b200_make_mesh_watertight_destroy(pcu_b200_watertight* wt) {
    if (!wt) return PCU_B200_OK;
    DeviceGuard guard(wt->device);
    delete wt;
    return PCU_B200_OK;
}

int pcu_b200_connected_components_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_cols, int f_kind,
                                           pcu_b200_components** out_cc, int64_t out_counts[2], void* stream) {
    return connected_components_prepare_device(ws, f, nf, f_cols, f_kind, out_cc, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_connected_components_emit(pcu_b200_workspace* ws, const pcu_b200_components* cc, void* out_cv, void* out_nv, void* out_cf,
                                        void* out_nf, void* stream) {
    return connected_components_emit_device(ws, cc, out_cv, out_nv, out_cf, out_nf, (cudaStream_t)stream);
}
int pcu_b200_connected_components_destroy(pcu_b200_components* cc) {
    if (!cc) return PCU_B200_OK;
    DeviceGuard guard(cc->device);
    delete cc;
    return PCU_B200_OK;
}
int pcu_b200_remove_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, float* out_v, void* out_f, int64_t out_counts[2], void* stream) {
    return remove_mesh_vertices_device<float>(ws, v, nv, f, nf, f_kind, mask, out_v, out_f, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_remove_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, double* out_v, void* out_f, int64_t out_counts[2], void* stream) {
    return remove_mesh_vertices_device<double>(ws, v, nv, f, nf, f_kind, mask, out_v, out_f, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_remove_unreferenced_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   float* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream) {
    return remove_unreferenced_device<float>(ws, v, nv, f, nf, f_kind, out_v, out_f, out_corr_v, out_corr_f, (long long*)out_count,
                                             (cudaStream_t)stream);
}
int pcu_b200_remove_unreferenced_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   double* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream) {
    return remove_unreferenced_device<double>(ws, v, nv, f, nf, f_kind, out_v, out_f, out_corr_v, out_corr_f, (long long*)out_count,
                                              (cudaStream_t)stream);
}
int pcu_b200_orient_mesh_faces(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, void* out_f, void* out_components,
                               void* stream) {
    return orient_mesh_faces_device(ws, f, nf, f_kind, out_f, out_components, (cudaStream_t)stream);
}

int pcu_b200_mesh_face_areas_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_areas,
                                 void* stream) {
    return mesh_face_device<float>(ws, v, nv, f, nf, f_kind, false, out_areas, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_areas_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_areas,
                                 void* stream) {
    return mesh_face_device<double>(ws, v, nv, f, nf, f_kind, false, out_areas, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_n,
                                   void* stream) {
    return mesh_face_device<float>(ws, v, nv, f, nf, f_kind, true, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_face_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_n,
                                   void* stream) {
    return mesh_face_device<double>(ws, v, nv, f, nf, f_kind, true, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_vertex_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     float* out_n, void* stream) {
    return vertex_normals_device<float>(ws, v, nv, f, nf, f_kind, weighting, out_n, (cudaStream_t)stream);
}
int pcu_b200_mesh_vertex_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     double* out_n, void* stream) {
    return vertex_normals_device<double>(ws, v, nv, f, nf, f_kind, weighting, out_n, (cudaStream_t)stream);
}
int pcu_b200_laplacian_smooth_mesh_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, float* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream) {
    return laplacian_smooth_device<float>(ws, v, nv, f, nf, f_kind, num_iters, step_size, use_cotan_weights != 0, max_cg_iters, out_v,
                                          out_cg_iters, out_residual, (cudaStream_t)stream);
}
int pcu_b200_laplacian_smooth_mesh_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, double* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream) {
    return laplacian_smooth_device<double>(ws, v, nv, f, nf, f_kind, num_iters, step_size, use_cotan_weights != 0, max_cg_iters, out_v,
                                           out_cg_iters, out_residual, (cudaStream_t)stream);
}

}  // extern "C"
