// mesh_topology.cu -- connected components and vertex removal, adjacency lists, consistent face orientation, face areas
// and normals, vertex normals, principal curvatures and Laplacian smoothing (mesh_topology.cuh, orient.cuh,
// mesh_geometry.cuh, curvature.cuh, laplacian.cuh): launch sequencing and C entry points.
#include "runtime.cuh"
#include "mesh_topology.cuh"
#include "orient.cuh"
#include "laplacian.cuh"
#include "curvature.cuh"

using namespace pcu;
using namespace pcu_internal;

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

// Adjacency lists between pcu_b200_adjacency_list_prepare and _emit: the int32 CSR in one block (rowptr over the n + 1
// row boundaries, col over the nnz entries).
struct pcu_b200_adjacency : StreamHandle {
    int fkind = 0;
    long long n = 0, nnz = 0;
    unsigned char* block = nullptr;
    const int* rowptr = nullptr;
    const int* col = nullptr;
    ~pcu_b200_adjacency() { release(block); }
};

namespace {

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

// mesh_principal_curvatures (curvature.cuh): face pass (unit normals, Max's weights and, for the one-ring mode, dblA
// and half-cotangents), corner CSR, fp64 vertex normals; then the one-ring kernels (r <= 0) or the ball pass of
// nearest.cu (r > 0).  The normals and the record live in kMesh, which the ball pass's binning does not re-carve.  One
// synchronisation.
template <typename T>
int mesh_curvatures_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, double r, T* out_k1,
                           T* out_k2, T* out_d1, T* out_d2, cudaStream_t stream) {
    PCU_TRY(mg_check(ws, v, nv, f, m, fkind, out_k1));
    if (!out_k2 || !out_d1 || !out_d2) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    if (!std::isfinite(r)) return fail(PCU_B200_INVALID_ARGUMENT, "mesh_principal_curvatures: r must be finite, got %g", r);
    PCU_ON_DEVICE(ws);
    const bool ring = !(r > 0.0);
    struct { MgRecord* rec; double* normal; } keep;
    PCU_TRY(carve_scratch(ws, kMesh, stream, [&](Carver& cv) {
        keep.rec = cv.take<MgRecord>(1);
        keep.normal = cv.take<double>(3 * (size_t)nv);
    }));
    struct { double *unit, *weight, *dbla, *halfcot, *frame_u, *efg; SortScratch<MgRec> sort; int *first, *corner; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.unit = cv.take<double>(3 * (size_t)m);
        sc.weight = cv.take<double>(3 * (size_t)m);
        sc.dbla = ring ? cv.take<double>((size_t)m) : nullptr;
        sc.halfcot = ring ? cv.take<double>(3 * (size_t)m) : nullptr;
        sc.frame_u = ring ? cv.take<double>(3 * (size_t)m) : nullptr;
        sc.efg = ring ? cv.take<double>(3 * (size_t)m) : nullptr;
        sc.sort.carve(cv, 3 * m);
        sc.first = cv.take<int>((size_t)nv + 1);
        sc.corner = cv.take<int>(3 * (size_t)m);
    }));
    PCU_CUDA(cudaMemsetAsync(keep.rec, 0, sizeof(MgRecord), stream));
    FaceOut<T> o = {};
    o.unit = sc.unit;
    o.weight = sc.weight;
    o.weighting = 3;
    o.dbla = sc.dbla;
    o.halfcot = sc.halfcot;
    PCU_TRY(mg_face_pass<T>(v, nv, f, fkind, m, o, keep.rec, stream));
    PCU_TRY(enqueue_incidence(sc.sort, f, fkind, m, nv, sc.first, sc.corner, stream));
    PCU_LAUNCH(mg_vertex_normal_kernel<double>, blocks_for(nv), kThreads, stream, (const int*)sc.first, (const int*)sc.corner, nv,
               (const double*)sc.unit, (const double*)sc.weight, keep.normal);
    if (ring) {
        // the corner areas overwrite Max's weights, which the vertex normals no longer need
        PCU_LAUNCH(curv_face_kernel<T>, blocks_for(m), kThreads, stream, v, nv, f, fkind, m, (const double*)keep.normal,
                   (const double*)sc.unit, (const double*)sc.dbla, (const double*)sc.halfcot, sc.frame_u, sc.efg, sc.weight);
        PCU_LAUNCH(curv_vertex_kernel<T>, blocks_for(nv), kThreads, stream, (const int*)sc.first, (const int*)sc.corner, nv,
                   (const double*)keep.normal, (const double*)sc.unit, (const double*)sc.frame_u, (const double*)sc.efg,
                   (const double*)sc.weight, out_k1, out_k2, out_d1, out_d2);
    } else {
        PCU_TRY(curvature_ball_device<T>(ws, v, nv, keep.normal, r, out_k1, out_k2, out_d1, out_d2, stream));
    }
    MgRecord host;
    PCU_TRY(read_record(keep.rec, &host, stream));
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
    PCU_LAUNCH(mc_heads_kernel, blocks_for(e), kThreads, stream, (const MgRec*)sorted, e, s.head);
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

// ---- adjacency lists (mesh_topology.cuh, on the Laplacian's assembly) -----------------------------------------------
// Validate f and read max(f) (first synchronisation); the Laplacian's sorted directed-edge records over the rows [0, n)
// and their run heads, and read the entry count (second synchronisation); then the CSR in the handle's block.  The sort's
// second buffer, free once the sort is done, holds the entries' row records.
int adj_build(pcu_b200_workspace* ws, pcu_b200_adjacency* h, const void* f, long long m, int fkind, cudaStream_t stream) {
    const long long e = 6 * m;
    struct { AdjCounts* rec; SortScratch<MgRec> sort; unsigned char* head; unsigned* counts; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.rec = cv.take<AdjCounts>(1);
        sc.sort.carve(cv, e);
        sc.head = cv.take<unsigned char>((size_t)e);
        sc.counts = cv.take<unsigned>(keep_count_words(e));
    }));
    PCU_CUDA(cudaMemsetAsync(sc.rec, 0, sizeof(AdjCounts), stream));
    PCU_LAUNCH(cc_validate_kernel, cc_validate_blocks(ws, 3 * m), kThreads, stream, f, fkind, 3 * m, &sc.rec->valid);
    AdjCounts hc;
    PCU_TRY(read_record(sc.rec, &hc, stream));
    if (hc.valid.bad)
        return fail(PCU_B200_INVALID_ARGUMENT, "adjacency_list: %llu face indices are negative or above 2^31 - 2", hc.valid.bad);
    const long long n = (long long)hc.valid.max_index + 1;
    const int bits = mg_index_bits(n);
    PCU_LAUNCH(lap_edge_kernel, blocks_for(m), kThreads, stream, f, fkind, m, n, bits, sc.sort.a);
    MgRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, e, 1, stream, &sorted, 2 * bits));
    PCU_LAUNCH(mc_heads_kernel, blocks_for(e), kThreads, stream, (const MgRec*)sorted, e, sc.head);
    PCU_TRY(enqueue_keep_offsets(sc.head, e, sc.counts, &sc.rec->nnz, stream));
    PCU_TRY(read_record(sc.rec, &hc, stream));
    const long long nnz = hc.nnz;
    struct { int *rowptr, *col; } b;
    const auto carve = [&](Carver& cv) {
        b.rowptr = cv.take<int>((size_t)n + 1);
        b.col = cv.take<int>((size_t)nnz);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "adjacency lists"));
    carve_at(h->block, carve);
    MgRec* rows = sorted == sc.sort.a ? sc.sort.b : sc.sort.a;
    PCU_LAUNCH(adj_entries_kernel, blocks_for(e), kThreads, stream, (const MgRec*)sorted, e, (const unsigned char*)sc.head,
               (const unsigned*)sc.counts, bits, rows, b.col);
    PCU_LAUNCH(mg_rows_kernel, blocks_for(nnz + 1), kThreads, stream, (const MgRec*)rows, nnz, n, b.rowptr, (int*)nullptr, 0);
    h->n = n;
    h->nnz = nnz;
    h->rowptr = b.rowptr;
    h->col = b.col;
    return PCU_B200_OK;
}

int adjacency_list_prepare_device(pcu_b200_workspace* ws, const void* f, long long m, int fkind, pcu_b200_adjacency** out,
                                  long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (m <= 0 || m > 0x7fffffffLL / 6)
        return fail(PCU_B200_INVALID_ARGUMENT, "adjacency_list: between 1 and 357913941 faces are supported, got %lld", m);
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_adjacency* h) {
        h->fkind = fkind;
        return adj_build(ws, h, f, m, fkind, stream);
    }));
    out_counts[0] = (*out)->n;
    out_counts[1] = (*out)->nnz;
    return PCU_B200_OK;
}

int adjacency_list_emit_device(pcu_b200_workspace* ws, const pcu_b200_adjacency* h, void* out_offsets, void* out_neighbors,
                               cudaStream_t stream) {
    if (!ws || !h || !out_offsets || !out_neighbors) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "adjacency"));
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(std::max(h->n + 1, h->nnz));
    if (wide_index(h->fkind))
        PCU_LAUNCH(adj_emit_kernel<long long>, blocks, kThreads, stream, h->rowptr, h->n, h->col, h->nnz, (long long*)out_offsets,
                   (long long*)out_neighbors);
    else
        PCU_LAUNCH(adj_emit_kernel<int>, blocks, kThreads, stream, h->rowptr, h->n, h->col, h->nnz, (int*)out_offsets, (int*)out_neighbors);
    return PCU_B200_OK;
}

}  // namespace

extern "C" {

int pcu_b200_connected_components_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_cols, int f_kind,
                                           pcu_b200_components** out_cc, int64_t out_counts[2], void* stream) {
    return connected_components_prepare_device(ws, f, nf, f_cols, f_kind, out_cc, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_connected_components_emit(pcu_b200_workspace* ws, const pcu_b200_components* cc, void* out_cv, void* out_nv, void* out_cf,
                                        void* out_nf, void* stream) {
    return connected_components_emit_device(ws, cc, out_cv, out_nv, out_cf, out_nf, (cudaStream_t)stream);
}
int pcu_b200_connected_components_destroy(pcu_b200_components* cc) { return destroy_handle(cc); }
int pcu_b200_adjacency_list_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, pcu_b200_adjacency** out_adj,
                                    int64_t out_counts[2], void* stream) {
    return adjacency_list_prepare_device(ws, f, nf, f_kind, out_adj, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_adjacency_list_emit(pcu_b200_workspace* ws, const pcu_b200_adjacency* adj, void* out_offsets, void* out_neighbors, void* stream) {
    return adjacency_list_emit_device(ws, adj, out_offsets, out_neighbors, (cudaStream_t)stream);
}
int pcu_b200_adjacency_list_destroy(pcu_b200_adjacency* adj) { return destroy_handle(adj); }
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
int pcu_b200_mesh_principal_curvatures_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, double r,
                                           float* out_k1, float* out_k2, float* out_d1, float* out_d2, void* stream) {
    return mesh_curvatures_device<float>(ws, v, nv, f, nf, f_kind, r, out_k1, out_k2, out_d1, out_d2, (cudaStream_t)stream);
}
int pcu_b200_mesh_principal_curvatures_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double r,
                                           double* out_k1, double* out_k2, double* out_d1, double* out_d2, void* stream) {
    return mesh_curvatures_device<double>(ws, v, nv, f, nf, f_kind, r, out_k1, out_k2, out_d1, out_d2, (cudaStream_t)stream);
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
