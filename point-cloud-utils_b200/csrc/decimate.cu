// decimate.cu -- shortest-edge decimation of triangle meshes (decimate.cuh): launch sequencing and C entry points.
#include "runtime.cuh"
#include "decimate.cuh"

using namespace pcu;
using namespace pcu_internal;

// Decimation between pcu_b200_decimate_triangle_mesh_prepare_* and _emit: the result in one block, vertices in fp64 and
// indices in int32, which emit converts to the input's types.
struct pcu_b200_decimate : StreamHandle {
    int t_f64 = 0, fkind = 0;
    long long nv = 0, nf = 0, rounds = 0;
    unsigned char* block = nullptr;
    const double* x = nullptr;
    const int* faces = nullptr;
    const int* vcorr = nullptr;
    const int* fcorr = nullptr;
    ~pcu_b200_decimate() { release(block); }
};

namespace {

const char* const kDcRejected = "decimate_triangle_mesh_doc produced an empty mesh. This can happen if the input is non-manifold.";

// The buffers of one call, sized by the input: m faces give at most 6 m directed-edge records and runs.
struct DcScratch {
    long long nv = 0, m = 0;
    int id_bits = 1;               // vertex ids < 2^id_bits: the adjacency sort's key bits
    double* x;
    int *F, *live, *next, *map, *beg, *end, *nb, *label;
    unsigned* stamp;
    int *rs, *rd, *o0, *o1;
    unsigned char *flag, *alive, *used;
    unsigned* offsets;
    DcCounts* counts;
    SortScratch<DcRec> sort;
    void carve(Carver& cv) {
        const long long n = 6 * m;
        x = cv.take<double>(3 * (size_t)nv);
        F = cv.take<int>(3 * (size_t)m);
        live = cv.take<int>((size_t)m);
        next = cv.take<int>((size_t)m);
        map = cv.take<int>((size_t)nv);
        beg = cv.take<int>((size_t)nv);
        end = cv.take<int>((size_t)nv);
        nb = cv.take<int>((size_t)nv);
        label = cv.take<int>((size_t)nv);
        stamp = cv.take<unsigned>((size_t)nv);
        rs = cv.take<int>((size_t)n);
        rd = cv.take<int>((size_t)n);
        o0 = cv.take<int>((size_t)n);
        o1 = cv.take<int>((size_t)n);
        flag = cv.take<unsigned char>((size_t)n);
        alive = cv.take<unsigned char>((size_t)m);
        used = cv.take<unsigned char>((size_t)nv);
        offsets = cv.take<unsigned>(keep_count_words(std::max(n, nv)));
        counts = cv.take<DcCounts>(1);
        sort.carve(cv, n);
    }
};

// The adjacency of the A live faces: the records sorted by (src, dst), their runs, every vertex's neighbour list and
// boundary edges.
int dc_adjacency(DcScratch& s, long long A, cudaStream_t stream) {
    const long long n = 6 * A;
    PCU_LAUNCH(dc_records_kernel, blocks_for(A), kThreads, stream, (const int*)s.F, (const int*)s.live, A, s.sort.a);
    DcRec* sorted = nullptr;
    PCU_TRY(radix_sort_records(s.sort, n, 2, stream, &sorted, s.id_bits));
    PCU_LAUNCH(dc_heads_kernel, blocks_for(n), kThreads, stream, (const DcRec*)sorted, n, s.flag);
    PCU_TRY(enqueue_keep_offsets(s.flag, n, s.offsets, &s.counts->runs, stream));
    PCU_CUDA(cudaMemsetAsync(s.nb, 0, sizeof(int) * (size_t)s.nv, stream));
    PCU_LAUNCH(dc_runs_kernel, blocks_for(n), kThreads, stream, (const DcRec*)sorted, n, (const unsigned char*)s.flag,
               (const unsigned*)s.offsets, s.rs, s.rd, s.o0, s.o1, s.beg, s.end, s.nb, s.counts);
    return PCU_B200_OK;
}

// One round on the A > max_faces live faces whose adjacency is built: validity, ranking, selection, trim and collapse,
// then the new live list (in s.next) and the count record read back into *hc (the round's synchronisation).
int dc_round(DcScratch& s, long long A, long long max_faces, DcCounts* hc, cudaStream_t stream) {
    const long long n = 6 * A, K = A - max_faces, P = std::min(K, 3 * A);
    PCU_LAUNCH(dc_valid_kernel, blocks_for(n), kThreads, stream, n, (const DcCounts*)s.counts, (const int*)s.rs, (const int*)s.rd,
               (const int*)s.o0, (const int*)s.o1, (const int*)s.beg, (const int*)s.end, (const int*)s.nb, s.flag);
    PCU_TRY(enqueue_keep_offsets(s.flag, n, s.offsets, &s.counts->valid, stream));
    PCU_LAUNCH(dc_keys_kernel, blocks_for(n), kThreads, stream, n, 3 * A, (const unsigned char*)s.flag, (const unsigned*)s.offsets,
               (const DcCounts*)s.counts, (const int*)s.rs, (const int*)s.rd, (const double*)s.x, s.sort.a);
    DcRec* ranked = nullptr;
    PCU_TRY(radix_sort_records(s.sort, 3 * A, 2, stream, &ranked));
    PCU_CUDA(cudaMemsetAsync(s.stamp, 0xff, sizeof(unsigned) * (size_t)s.nv, stream));
    PCU_CUDA(cudaMemsetAsync(&s.counts->applied, 0, 2 * sizeof(unsigned long long), stream));
    PCU_LAUNCH(dc_stamp_kernel, blocks_for(P), kThreads, stream, P, (const DcRec*)ranked, (const DcCounts*)s.counts, (const int*)s.rs,
               (const int*)s.rd, (const int*)s.beg, (const int*)s.end, s.stamp);
    PCU_LAUNCH(dc_select_kernel, blocks_for(P), kThreads, stream, P, (const DcRec*)ranked, (const DcCounts*)s.counts, (const int*)s.rs,
               (const int*)s.rd, (const int*)s.o1, (const int*)s.beg, (const int*)s.end, (const unsigned*)s.stamp, s.flag);
    PCU_TRY(enqueue_keep_offsets(s.flag, 2 * P, s.offsets, &s.counts->removable, stream));
    PCU_LAUNCH(dc_apply_kernel, blocks_for(2 * P), kThreads, stream, 2 * P, K, (const unsigned char*)s.flag, (const unsigned*)s.offsets,
               (const DcRec*)ranked, (const int*)s.rs, (const int*)s.rd, s.x, s.map, s.counts);
    PCU_LAUNCH(dc_faces_kernel, blocks_for(A), kThreads, stream, s.F, (const int*)s.live, A, (const int*)s.map, s.flag);
    PCU_TRY(enqueue_keep_offsets(s.flag, A, s.offsets, &s.counts->alive, stream));
    PCU_LAUNCH(dc_live_kernel, blocks_for(A), kThreads, stream, (const int*)s.live, A, (const unsigned char*)s.flag,
               (const unsigned*)s.offsets, s.next);
    return read_record(s.counts, hc, stream);
}

// The live faces in ascending input order relabelled to the used vertices in ascending id, into the handle's block.
int dc_output(DcScratch& s, pcu_b200_decimate* h, long long A, cudaStream_t stream) {
    const auto carve = [&](Carver& cv) {
        h->x = cv.take<double>(3 * (size_t)s.nv);
        h->faces = cv.take<int>(3 * (size_t)s.m);
        h->vcorr = cv.take<int>((size_t)s.nv);
        h->fcorr = cv.take<int>((size_t)s.m);
    };
    PCU_TRY(alloc_block(h->block, carve_at(nullptr, carve), stream, "decimate_triangle_mesh"));
    carve_at(h->block, carve);
    PCU_CUDA(cudaMemsetAsync(s.alive, 0, (size_t)s.m, stream));
    PCU_CUDA(cudaMemsetAsync(s.used, 0, (size_t)s.nv, stream));
    PCU_LAUNCH(dc_mark_kernel, blocks_for(A), kThreads, stream, (const int*)s.F, (const int*)s.live, A, s.alive, s.used);
    PCU_TRY(enqueue_keep_offsets(s.used, s.nv, s.offsets, &s.counts->nv_out, stream));
    PCU_LAUNCH(dc_vrank_kernel, blocks_for(s.nv), kThreads, stream, s.nv, (const unsigned char*)s.used, (const unsigned*)s.offsets,
               (const double*)s.x, s.label, const_cast<int*>(h->vcorr), const_cast<double*>(h->x));
    PCU_TRY(enqueue_keep_offsets(s.alive, s.m, s.offsets, &s.counts->nf_out, stream));
    PCU_LAUNCH(dc_fout_kernel, blocks_for(s.m), kThreads, stream, s.m, (const unsigned char*)s.alive, (const unsigned*)s.offsets,
               (const int*)s.F, (const int*)s.label, const_cast<int*>(h->fcorr), const_cast<int*>(h->faces));
    DcCounts hc;
    PCU_TRY(read_record(s.counts, &hc, stream));
    h->nv = hc.nv_out;
    h->nf = hc.nf_out;
    if (h->nv == 0) return fail(PCU_B200_INVALID_ARGUMENT, "%s", kDcRejected);
    return PCU_B200_OK;
}

// Input check (first synchronisation), the first adjacency and its acceptance test (second), the rounds (one each),
// the output (one more).
template <typename T>
int dc_build(pcu_b200_decimate* h, const T* v, long long nv, const void* f, long long m, int fkind, long long max_faces, cudaStream_t stream) {
    DcScratch s;
    s.nv = nv;
    s.m = m;
    while ((1ll << s.id_bits) < nv) ++s.id_bits;
    CallBlock blk(stream);
    PCU_TRY(alloc_block(blk.p, carve_at(nullptr, [&](Carver& cv) { s.carve(cv); }), stream, "decimate_triangle_mesh's scratch"));
    carve_at(blk.p, [&](Carver& cv) { s.carve(cv); });
    PCU_CUDA(cudaMemsetAsync(s.counts, 0, sizeof(DcCounts), stream));
    PCU_LAUNCH(dc_faces_in_kernel, blocks_for(m), kThreads, stream, f, fkind, m, nv, s.F, s.live, s.counts);
    PCU_LAUNCH((dc_verts_in_kernel<T>), blocks_for(nv), kThreads, stream, v, nv, s.x, s.map, s.counts);
    DcCounts hc;
    PCU_TRY(read_record(s.counts, &hc, stream));
    if (hc.bad_corner) return bad_corners(hc.bad_corner);
    if (hc.non_finite) return fail(PCU_B200_INVALID_ARGUMENT, "decimate_triangle_mesh: v has %llu non-finite vertices", hc.non_finite);
    if (hc.rejected) return fail(PCU_B200_INVALID_ARGUMENT, "%s", kDcRejected);
    long long A = m;
    PCU_TRY(dc_adjacency(s, A, stream));
    PCU_LAUNCH(dc_accept_kernel, blocks_for(nv), kThreads, stream, (const int*)s.nb, nv, s.counts);
    PCU_TRY(read_record(s.counts, &hc, stream));
    if (hc.rejected) return fail(PCU_B200_INVALID_ARGUMENT, "%s", kDcRejected);
    while (A > max_faces) {
        PCU_TRY(dc_round(s, A, max_faces, &hc, stream));
        if (hc.valid == 0) break;            // nothing collapsed: the mesh has stalled
        ++h->rounds;
        A = hc.alive;
        std::swap(s.live, s.next);
        if (A > max_faces) PCU_TRY(dc_adjacency(s, A, stream));
    }
    return dc_output(s, h, A, stream);
}

template <typename T>
int decimate_prepare_device(pcu_b200_workspace* ws, const T* v, long long nv, const void* f, long long m, int fkind, long long max_faces,
                            pcu_b200_decimate** out, long long* out_counts, cudaStream_t stream) {
    if (!ws || !out || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!v || !f) return fail(PCU_B200_INVALID_ARGUMENT, "null input pointer");
    if (nv <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid input mesh with zero elements");
    if (nv > kDcMaxIds || m > kDcMaxIds / 6)
        return fail(PCU_B200_INVALID_ARGUMENT, "decimate_triangle_mesh: at most 2^31 - 2 vertices and (2^31 - 2) / 6 faces are supported");
    if (fkind < kIdxI32 || fkind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown face index kind %d", fkind);
    if (max_faces <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_faces must be greater than 0, got %lld.", max_faces);
    if (max_faces > m)
        return fail(PCU_B200_INVALID_ARGUMENT, "max_faces must be less than or equal to the number of input faces (%lld), got %lld.", m, max_faces);
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    PCU_TRY(prepare_handle(ws, stream, out, [&](pcu_b200_decimate* h) -> int {
        h->t_f64 = sizeof(T) == 8;
        h->fkind = fkind;
        return dc_build<T>(h, v, nv, f, m, fkind, max_faces, stream);
    }));
    out_counts[0] = (*out)->nv;
    out_counts[1] = (*out)->nf;
    out_counts[2] = (*out)->rounds;
    return PCU_B200_OK;
}

int decimate_emit_device(pcu_b200_workspace* ws, const pcu_b200_decimate* h, void* out_v, void* out_f, void* out_vc, void* out_fc,
                         cudaStream_t stream) {
    if (!ws || !h) return fail(PCU_B200_INVALID_ARGUMENT, "null argument");
    PCU_TRY(check_handle_device(ws, h, "decimation"));
    if (!out_v || !out_f || !out_vc || !out_fc) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_TRY(adopt_stream(ws, stream));
    const unsigned blocks = blocks_for(3 * std::max(h->nv, h->nf));
    const int wide = (int)wide_index(h->fkind);
    if (h->t_f64)
        PCU_LAUNCH(dc_emit_kernel<double>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->vcorr, h->fcorr, h->nf, wide, (double*)out_v, out_f,
                   out_vc, out_fc);
    else
        PCU_LAUNCH(dc_emit_kernel<float>, blocks, kThreads, stream, h->x, h->nv, h->faces, h->vcorr, h->fcorr, h->nf, wide, (float*)out_v, out_f,
                   out_vc, out_fc);
    return PCU_B200_OK;
}

}  // namespace

extern "C" {

int pcu_b200_decimate_triangle_mesh_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                int64_t max_faces, pcu_b200_decimate** out_dc, int64_t out_counts[3], void* stream) {
    return decimate_prepare_device<float>(ws, v, nv, f, nf, f_kind, max_faces, out_dc, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_decimate_triangle_mesh_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                int64_t max_faces, pcu_b200_decimate** out_dc, int64_t out_counts[3], void* stream) {
    return decimate_prepare_device<double>(ws, v, nv, f, nf, f_kind, max_faces, out_dc, (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_decimate_triangle_mesh_emit(pcu_b200_workspace* ws, const pcu_b200_decimate* dc, void* out_v, void* out_f, void* out_v_corr,
                                         void* out_f_corr, void* stream) {
    return decimate_emit_device(ws, dc, out_v, out_f, out_v_corr, out_f_corr, (cudaStream_t)stream);
}
int pcu_b200_decimate_triangle_mesh_destroy(pcu_b200_decimate* dc) { return destroy_handle(dc); }

}  // extern "C"
