// voxels.cu -- marching cubes and the boundary of a sparse voxel grid, sparse voxel grids and voxel cube meshes,
// triangle-mesh voxelization, 3-D flood fill and watertight remeshing (sparse_voxels.cuh, voxelize.cuh,
// watertight.cuh): launch sequencing and C entry points.
#include "runtime.cuh"
#include "sparse_voxels.cuh"
#include "voxelize.cuh"
#include "watertight.cuh"

using namespace pcu;
using namespace pcu_internal;

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
        sc.tree = cv.take<unsigned char>(closest_tree_bytes(m));
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
    PCU_TRY(build_closest_tree(ws, v64, nv, f, m, fkind, sc.flipped + 1, sc.tree, t, stream));
    double* x = const_cast<double*>(h->x);
    const unsigned vb = blocks_for(n), fb = blocks_for(nf);
    PCU_LAUNCH(wt_start_kernel, vb, kThreads, stream, (const double*)x, n, sc.x0, sc.alpha);
    for (int round = 0; round < kWtRounds; ++round) {
        PCU_TRY(enqueue_closest_points(ws, t, m, x, n, sc.d, sc.fidx, sc.bc, stream));
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

}  // namespace

extern "C" {

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
int pcu_b200_marching_cubes_destroy(pcu_b200_marching_cubes* mc) { return destroy_handle(mc); }
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
int pcu_b200_sparse_grid_destroy(pcu_b200_sparse_grid* sg) { return destroy_handle(sg); }
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
int pcu_b200_voxelize_destroy(pcu_b200_voxelize* vx) { return destroy_handle(vx); }
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
int pcu_b200_make_mesh_watertight_destroy(pcu_b200_watertight* wt) { return destroy_handle(wt); }

}  // extern "C"
