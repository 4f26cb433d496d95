// point_ops.cu -- point-cloud operations that share nothing with the nearest-neighbour sweep: duplicate removal, Morton
// codes, voxel-grid downsampling, dense pairwise distances and Sinkhorn, point areas from given neighbour rows, and
// their device and host C entry points.
#include "runtime.cuh"
#include "dedup.cuh"
#include "morton.cuh"
#include "point_areas.cuh"
#include "sinkhorn.cuh"
#include "voxel.cuh"

namespace pcu {

// pts: (n, 3) int32 or int64 (truncated to int32 like the reference's `int32_t px = pts(i, 0)`, morton.cpp:229)
template <typename I>
__global__ void morton_encode_kernel(const I* __restrict__ pts, long long n, unsigned long long* __restrict__ codes) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    codes[i] = morton_encode3((int)pts[3 * i], (int)pts[3 * i + 1], (int)pts[3 * i + 2]);
}
__global__ void morton_decode_kernel(const unsigned long long* __restrict__ codes, long long n, int* __restrict__ pts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int x, y, z;
    morton_decode3(codes[i], x, y, z);
    pts[3 * i] = x; pts[3 * i + 1] = y; pts[3 * i + 2] = z;
}
// op 0: a + b; op 1: a - b = a + negate(b)  (morton_code.cpp:160-163)
__global__ void morton_addsub_kernel(const unsigned long long* __restrict__ a, const unsigned long long* __restrict__ b,
                                     long long n, int op, unsigned long long* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = morton_add2(a[i], op ? morton_negate(b[i]) : b[i]);
}

// morton_knn (morton.cpp:324-414): lower_bound of the query code in the SORTED codes, then the window of k
// consecutive positions around it (k / 2 above, the rest below, shifted back inside the array at the ends).
// k has already been clamped to n by the caller (:351).  sort_dist: order the window by squared distance to the
// query point (ties by position) -- the reference's comparator reads three uninitialised locals there (:381-398),
// so that ORDER is undefined in the reference; the window itself is exactly the reference's.
__global__ void morton_knn_kernel(const unsigned long long* __restrict__ codes, long long n,
                                  const unsigned long long* __restrict__ qcodes, long long m, int k, int sort_dist,
                                  long long* __restrict__ out_idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const unsigned long long q = qcodes[i];
    long long lo = 0, hi = n;                 // std::lower_bound
    while (lo < hi) {
        const long long mid = lo + (hi - lo) / 2;
        if (codes[mid] < q) lo = mid + 1; else hi = mid;
    }
    const int half_up = k / 2, half_down = k - half_up;
    long long upper = lo + half_up, lower = lo - half_down;
    if (upper >= n) { lower -= (upper - n); upper = n; }
    if (lower < 0) { upper += -lower; lower = 0; }
    long long* row = out_idx + i * k;
    const int count = (int)(upper - lower);
    if (!sort_dist) {
        for (int j = 0; j < count; ++j) row[j] = lower + j;
        return;
    }
    int qx, qy, qz;
    morton_decode3(q, qx, qy, qz);
    for (int j = 0; j < count; ++j) {         // insertion sort by (distance, position)
        const long long pos = lower + j;
        int x, y, z;
        morton_decode3(codes[pos], x, y, z);
        const double dx = (double)qx - x, dy = (double)qy - y, dz = (double)qz - z;
        const double d = dx * dx + dy * dy + dz * dz;
        int s = j;
        while (s > 0) {
            int px, py, pz;
            morton_decode3(codes[row[s - 1]], px, py, pz);
            const double ex = (double)qx - px, ey = (double)qy - py, ez = (double)qz - pz;
            if (ex * ex + ey * ey + ez * ez <= d) break;
            row[s] = row[s - 1];
            --s;
        }
        row[s] = pos;
    }
}

}  // namespace pcu

using namespace pcu;
using namespace pcu_internal;

namespace {

// ---- duplicate removal (SURVEY.md 8f N2, src/remove_duplicates.cpp) ----------------------------------------
// faces == nullptr: points only.  out_pts (n, 3), out_svi (n) and out_faces (nf, cols) are sized for the worst case;
// out_counts[0] = unique points, [1] = surviving faces, [2] = faces with a corner out of range (an error for the caller).
template <typename T, typename I>
int dedup_device(pcu_b200_workspace* ws, const T* pts, long long n, double epsilon, const I* faces, long long nf, int cols,
                 T* out_pts, int* out_svi, int* out_svj, I* out_faces, long long* out_counts, cudaStream_t stream) {
    using Rec = typename DedupRec<T>::type;
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld rows)", n);
    if (!out_pts || !out_svi || !out_svj || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    if (faces != nullptr && (nf < 0 || cols <= 0 || cols > 16 || (nf > 0 && !out_faces)))
        return fail(PCU_B200_INVALID_ARGUMENT, "faces must be an (m, c) array with 1 <= c <= 16");
    if (nf >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "too many faces (%lld)", nf);
    PCU_ON_DEVICE(ws);
    struct { SortScratch<Rec> sort; unsigned char* head; unsigned* counts; unsigned char* fkeep; unsigned* fcounts; unsigned* bad; } sc;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        sc.sort.carve(cv, n);
        sc.head = cv.take<unsigned char>((size_t)n);
        sc.counts = cv.take<unsigned>(keep_count_words(n));
        sc.fkeep = cv.take<unsigned char>((size_t)std::max<long long>(1, nf));
        sc.fcounts = cv.take<unsigned>(std::max<size_t>(1, faces ? keep_count_words(nf) : 0));
        sc.bad = cv.take<unsigned>(1);
    }));
    PCU_CUDA(cudaMemsetAsync(out_counts, 0, 3 * sizeof(long long), stream));
    PCU_LAUNCH((dedup_keys_kernel<T>), blocks_for(n), kThreads, stream, pts, n, (T)epsilon, sc.sort.a);
    Rec* sorted = nullptr;
    PCU_TRY(radix_sort_records(sc.sort, n, 3, stream, &sorted));
    PCU_LAUNCH((dedup_heads_kernel<Rec>), blocks_for(n), kThreads, stream, (const Rec*)sorted, n, sc.head);
    PCU_TRY(enqueue_keep_offsets(sc.head, n, sc.counts, out_counts, stream));
    PCU_LAUNCH((dedup_emit_kernel<T, Rec>), blocks_for(n), kThreads, stream, (const Rec*)sorted, n, (const unsigned char*)sc.head,
               (const unsigned*)sc.counts, pts, out_pts, out_svi, out_svj);
    if (faces != nullptr && nf > 0) {
        PCU_CUDA(cudaMemsetAsync(sc.bad, 0, sizeof(unsigned), stream));
        PCU_LAUNCH((dedup_faces_flag_kernel<I>), blocks_for(nf), kThreads, stream, faces, nf, cols, n, (const int*)out_svj, sc.fkeep, sc.bad);
        PCU_TRY(enqueue_keep_offsets(sc.fkeep, nf, sc.fcounts, out_counts + 1, stream));
        PCU_LAUNCH((dedup_faces_emit_kernel<I>), blocks_for(nf), kThreads, stream, faces, nf, cols, (const int*)out_svj,
                   (const unsigned char*)sc.fkeep, (const unsigned*)sc.fcounts, out_faces);
        PCU_LAUNCH(widen_counter_kernel, 1, 1, stream, sc.bad, out_counts + 2);
    }
    return PCU_B200_OK;
}

template <typename T>
int dedup_dispatch(pcu_b200_workspace* ws, const T* pts, long long n, double epsilon, const void* faces, long long nf, int cols,
                   int faces_are_i64, T* out_pts, int* out_svi, int* out_svj, void* out_faces, long long* out_counts, cudaStream_t stream) {
    if (faces_are_i64)
        return dedup_device<T, long long>(ws, pts, n, epsilon, (const long long*)faces, nf, cols, out_pts, out_svi, out_svj,
                                          (long long*)out_faces, out_counts, stream);
    return dedup_device<T, int>(ws, pts, n, epsilon, (const int*)faces, nf, cols, out_pts, out_svi, out_svj, (int*)out_faces, out_counts, stream);
}

// ---- Morton codes (SURVEY.md 8f N3) -------------------------------------------------------------------

template <typename I>
int morton_encode_device(pcu_b200_workspace* ws, const I* pts, long long n, unsigned long long* out_codes, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    if (!out_codes) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH((morton_encode_kernel<I>), blocks_for(n), kThreads, stream, pts, n, out_codes);
    return PCU_B200_OK;
}

int morton_decode_device(pcu_b200_workspace* ws, const unsigned long long* codes, long long n, int* out_pts, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!codes || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    if (!out_pts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_decode_kernel, blocks_for(n), kThreads, stream, codes, n, out_pts);
    return PCU_B200_OK;
}

int morton_addsub_device(pcu_b200_workspace* ws, const unsigned long long* a, const unsigned long long* b, long long n, int op,
                         unsigned long long* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes_1 and codes_2 must be arrays of shape [n,] but got an empty array");
    if (!out) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_addsub_kernel, blocks_for(n), kThreads, stream, a, b, n, op, out);
    return PCU_B200_OK;
}

int morton_knn_device(pcu_b200_workspace* ws, const unsigned long long* codes, long long n, const unsigned long long* qcodes,
                      long long m, int k, int sort_dist, long long* out_idx, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "k must be greater than 0");
    if (!codes || n <= 0 || !qcodes || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    if ((long long)k > n) return fail(PCU_B200_INVALID_ARGUMENT, "k (%d) exceeds the number of codes (%lld): clamp it first (morton.cpp:351)", k, n);
    if (!out_idx) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    PCU_LAUNCH(morton_knn_kernel, blocks_for(m), kThreads, stream, codes, n, qcodes, m, k, sort_dist, out_idx);
    return PCU_B200_OK;
}

// ---- voxel-grid down-sampling (SURVEY.md 8f N2) -----------------------------------------------------------
template <typename T, typename A>
int voxel_downsample_device(pcu_b200_workspace* ws, const T* pts, long long n, const A* attr, int attr_cols, const double size[3],
                            const double min_bound[3], const double max_bound[3], int min_points, T* out_pts, A* out_attr,
                            int* out_counts, long long* out_rows, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!pts || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld rows)", n);
    if (!out_pts || !out_rows || attr_cols < 0 || (attr_cols > 0 && (!attr || !out_attr)))
        return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    VoxelGrid<T> g;
    for (int a = 0; a < 3; ++a) {   // src/sample_point_cloud.cpp:175-182, in the cloud's precision like the reference's casts (:346-354)
        g.size[a] = (T)size[a];
        g.min_bound[a] = (T)min_bound[a];
        if (g.size[a] <= (T)0) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size is negative");
        if (g.size[a] * (T)2147483647 < (T)max_bound[a] - g.min_bound[a]) return fail(PCU_B200_INVALID_ARGUMENT, "Voxel size is too small");
    }
    PCU_ON_DEVICE(ws);
    unsigned slots = 64;
    while ((long long)slots < 2 * n) slots <<= 1;     // load factor <= 1/2
    int *table, *slot_of; VoxelAcc* acc; double* attr_sum; unsigned char* keep; unsigned* counts;
    PCU_TRY(carve_scratch(ws, kArena, stream, [&](Carver& cv) {
        table = cv.take<int>(slots);
        acc = cv.take<VoxelAcc>(slots);
        slot_of = cv.take<int>((size_t)n);
        attr_sum = cv.take<double>((size_t)slots * (attr_cols > 0 ? attr_cols : 0) + 1);
        keep = cv.take<unsigned char>((size_t)n);
        counts = cv.take<unsigned>(keep_count_words(n));
    }));
    PCU_LAUNCH(voxel_init_kernel, blocks_for(slots), kThreads, stream, table, acc, slots);
    if (attr_cols > 0) PCU_CUDA(cudaMemsetAsync(attr_sum, 0, sizeof(double) * (size_t)slots * attr_cols, stream));
    PCU_LAUNCH((voxel_insert_kernel<T, A>), blocks_for(n), kThreads, stream, pts, n, g, table, slots, acc, slot_of, attr, attr_cols, attr_sum);
    PCU_LAUNCH(voxel_flag_kernel, blocks_for(n), kThreads, stream, slot_of, acc, n, min_points, keep);
    PCU_TRY(enqueue_keep_offsets(keep, n, counts, out_rows, stream));
    PCU_LAUNCH((voxel_emit_kernel<T, A>), blocks_for(n), kThreads, stream, keep, n, counts, slot_of, acc, attr_sum, attr_cols, out_pts, out_attr, out_counts);
    return PCU_B200_OK;
}

template <typename T>
int voxel_downsample_dispatch(pcu_b200_workspace* ws, const T* pts, long long n, const void* attr, int attr_cols, int attr_is_f64,
                              const double size[3], const double min_bound[3], const double max_bound[3], int min_points, T* out_pts,
                              void* out_attr, int* out_counts, long long* out_rows, cudaStream_t stream) {
    if (attr_is_f64)
        return voxel_downsample_device<T, double>(ws, pts, n, (const double*)attr, attr_cols, size, min_bound, max_bound, min_points,
                                                  out_pts, (double*)out_attr, out_counts, out_rows, stream);
    return voxel_downsample_device<T, float>(ws, pts, n, (const float*)attr, attr_cols, size, min_bound, max_bound, min_points, out_pts,
                                             (float*)out_attr, out_counts, out_rows, stream);
}

// ---- dense pairwise distances, Sinkhorn (SURVEY.md 8f N4) ------------------------------------------------
// gridDim.y and gridDim.z stop at 65535: the dense kernels take rows and batches there, so larger problems are
// launched in chunks of that many, the pointers offset to each chunk's first row or batch.
constexpr long long kMaxGridYZ = 65535;

template <typename T>
int pairwise_device(pcu_b200_workspace* ws, const T* a, const T* b, long long nb, long long n, long long m, int d, int norm_kind,
                    double p, T* out, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || !out) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (nb <= 0 || n <= 0 || m <= 0 || d <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Invalid shape: a and b must be [m, n, d] or [n, d] with positive sizes");
    if (norm_kind < kNorm2 || norm_kind > kNormP) return fail(PCU_B200_INVALID_ARGUMENT, "unknown norm");
    PCU_ON_DEVICE(ws);
    for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ)
        for (long long i0 = 0; i0 < n; i0 += kMaxGridYZ) {
            const dim3 grid(blocks_for(m), (unsigned)std::min(n - i0, kMaxGridYZ), (unsigned)std::min(nb - b0, kMaxGridYZ));
            PCU_LAUNCH((pairwise_kernel<T>), grid, kThreads, stream, a + (b0 * n + i0) * d, b + b0 * m * d, n, m, d, norm_kind, p,
                       out + (b0 * n + i0) * m);
        }
    return PCU_B200_OK;
}

// a: (nb, n) weights, b: (nb, m) weights, M: (nb, n, m) costs -> P: (nb, n, m); out_cost (nb) fp64 = sum P * M, or null;
// out_iters: device int32, iterations run (or null).  No host synchronisation: the iteration's three kernels are
// enqueued max_iters times and return at once after the convergence test has passed on the device.
template <typename T>
int sinkhorn_device(pcu_b200_workspace* ws, const T* a, const T* b, const T* M, long long nb, long long n, long long m, double eps,
                    int max_iters, double stop_thresh, T* out_P, double* out_cost, int* out_iters, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!a || !b || !M || !out_P) return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    if (nb <= 0 || n <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "Got unexpected shape for M, should be [nb, m, n] with positive sizes");
    if (max_iters < 0) return fail(PCU_B200_INVALID_ARGUMENT, "max_iters must be >= 0");
    PCU_ON_DEVICE(ws);
    T *u, *v; double *eu, *ev; int* flags;
    auto carve = [&](Carver& cv) {
        u = cv.take<T>((size_t)nb * n);
        v = cv.take<T>((size_t)nb * m);
        eu = cv.take<double>((size_t)nb);
        ev = cv.take<double>((size_t)nb);
        flags = cv.take<int>(2);   // [0] done, [1] iterations
    };
    const size_t bytes = carve_at(nullptr, carve);
    PCU_TRY(carve_scratch(ws, kArena, stream, carve));
    PCU_CUDA(cudaMemsetAsync(u, 0, bytes, stream));   // u = v = 0 (:101-102), accumulators, flags
    if (out_cost) PCU_CUDA(cudaMemsetAsync(out_cost, 0, sizeof(double) * nb, stream));
    const T e = (T)eps;
    for (int it = 0; it < max_iters; ++it) {
        for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ) {
            const unsigned nbc = (unsigned)std::min(nb - b0, kMaxGridYZ);
            PCU_LAUNCH((sinkhorn_half_kernel<T, false>), dim3((unsigned)n, nbc), kThreads, stream, M + b0 * n * m, a + b0 * n, v + b0 * m,
                       u + b0 * n, n, m, e, eu + b0, flags);
        }
        for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ) {
            const unsigned nbc = (unsigned)std::min(nb - b0, kMaxGridYZ);
            PCU_LAUNCH((sinkhorn_half_kernel<T, true>), dim3((unsigned)((m + 31) / 32), nbc), kThreads, stream, M + b0 * n * m, b + b0 * m,
                       u + b0 * n, v + b0 * m, m, n, e, ev + b0, flags);
        }
        PCU_LAUNCH(sinkhorn_check_kernel, 1, kThreads, stream, eu, ev, nb, stop_thresh, flags, flags + 1);
    }
    for (long long b0 = 0; b0 < nb; b0 += kMaxGridYZ)
        for (long long i0 = 0; i0 < n; i0 += kMaxGridYZ) {
            const dim3 grid(blocks_for(m), (unsigned)std::min(n - i0, kMaxGridYZ), (unsigned)std::min(nb - b0, kMaxGridYZ));
            PCU_LAUNCH((sinkhorn_plan_kernel<T>), grid, kThreads, stream, M + (b0 * n + i0) * m, u + b0 * n + i0, v + b0 * m, n, m, e,
                       out_P + (b0 * n + i0) * m, out_cost ? out_cost + b0 : nullptr);
        }
    if (out_iters) PCU_CUDA(cudaMemcpyAsync(out_iters, flags + 1, sizeof(int), cudaMemcpyDeviceToDevice, stream));
    return PCU_B200_OK;
}

// ---- point areas (estimate_point_cloud_areas, src/point_areas.cpp) -------------------------------------------
template <typename T>
int point_areas_device(pcu_b200_workspace* ws, const T* points, long long n, const T* normals, const void* idx, int k, int kind,
                       T* out_areas, unsigned long long* out_bad, cudaStream_t stream) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (n < 0 || (n > 0 && (!points || !normals || (k > 0 && !idx) || !out_areas)) || !out_bad)
        return fail(PCU_B200_INVALID_ARGUMENT, "points, normals, idx and the outputs must be non-null");
    if (n >= 0x7fffffffLL) return fail(PCU_B200_INVALID_ARGUMENT, "point cloud too large (%lld rows)", n);
    if (k < 0 || k > kAreaMaxK)
        return fail(PCU_B200_INVALID_ARGUMENT, "estimate_point_cloud_areas: i may have at most %d columns, got %d", kAreaMaxK, k);
    if (kind < kIdxI32 || kind > kIdxU64) return fail(PCU_B200_INVALID_ARGUMENT, "unknown index kind %d", kind);
    PCU_ON_DEVICE(ws);
    PCU_CUDA(cudaMemsetAsync(out_bad, 0, sizeof(unsigned long long), stream));
    if (n == 0) return PCU_B200_OK;
    const int cap = std::max(32, (k + 31) / 32 * 32);
    return launch_pdl(point_areas_kernel<T>, dim3((unsigned)((n + kAreaWarps - 1) / kAreaWarps)), dim3(kAreaWarps * 32),
                      point_area_smem<T>(cap), stream, points, normals, n, idx, k, kind, cap, out_areas, out_bad);
}

// voxel-grid down-sampling on HOST arrays: stage, run, fetch the row count, then exactly the rows that exist
template <typename T>
int voxel_downsample_host(pcu_b200_workspace* ws, const T* points, long long n, const void* attrib, int attrib_cols, int attrib_is_f64,
                          const double size[3], const double min_bound[3], const double max_bound[3], int min_points, T* out_points,
                          void* out_attrib, int32_t* out_counts, long long* out_rows) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!points || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (!out_points || !out_rows || attrib_cols < 0 || (attrib_cols > 0 && (!attrib || !out_attrib)))
        return fail(PCU_B200_INVALID_ARGUMENT, "null pointer");
    PCU_ON_DEVICE(ws);
    const size_t abytes = (size_t)(attrib_is_f64 ? 8 : 4) * (size_t)attrib_cols;      // per row
    cudaStream_t st = ws->own_stream;
    T *dp, *op; unsigned char *da, *oa; int* oc; long long* orows;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        dp = cv.take<T>((size_t)3 * n);
        da = cv.take<unsigned char>(abytes * (size_t)n + 1);
        op = cv.take<T>((size_t)3 * n);
        oa = cv.take<unsigned char>(abytes * (size_t)n + 1);
        oc = cv.take<int>((size_t)n);
        orows = cv.take<long long>(1);
    }));
    PCU_TRY(h2d(ws, dp, points, sizeof(T) * 3 * n, st));
    if (attrib_cols > 0) PCU_TRY(h2d(ws, da, attrib, abytes * (size_t)n, st));
    PCU_TRY(voxel_downsample_dispatch<T>(ws, dp, n, attrib_cols > 0 ? da : nullptr, attrib_cols, attrib_is_f64, size, min_bound, max_bound,
                                         min_points, op, attrib_cols > 0 ? oa : nullptr, out_counts ? oc : nullptr, orows, st));
    long long* hr = reinterpret_cast<long long*>(ws->host_slot);
    PCU_CUDA(cudaMemcpyAsync(hr, orows, sizeof(long long), cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    const long long rows = *hr;
    if (rows > 0) {
        PCU_CUDA(cudaMemcpyAsync(out_points, op, sizeof(T) * 3 * rows, cudaMemcpyDeviceToHost, st));
        if (attrib_cols > 0) PCU_CUDA(cudaMemcpyAsync(out_attrib, oa, abytes * (size_t)rows, cudaMemcpyDeviceToHost, st));
        if (out_counts) PCU_CUDA(cudaMemcpyAsync(out_counts, oc, sizeof(int) * rows, cudaMemcpyDeviceToHost, st));
        PCU_CUDA(cudaStreamSynchronize(st));
    }
    *out_rows = rows;
    return PCU_B200_OK;
}

// duplicate removal on HOST arrays (faces may be null)
template <typename T>
int deduplicate_host(pcu_b200_workspace* ws, const T* points, long long n, double epsilon, const void* faces, long long nf, int cols,
                     int faces_are_i64, T* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces, long long* out_counts) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!points || n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "points must be a non-empty (n, 3) array");
    if (!out_points || !out_svi || !out_svj || !out_counts) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    if (faces != nullptr && (nf < 0 || cols <= 0 || cols > 16 || (nf > 0 && !out_faces)))
        return fail(PCU_B200_INVALID_ARGUMENT, "faces must be an (m, c) array with 1 <= c <= 16");
    PCU_ON_DEVICE(ws);
    const bool with_faces = faces != nullptr && nf > 0;
    const size_t fbytes = with_faces ? (size_t)(faces_are_i64 ? 8 : 4) * (size_t)cols * (size_t)nf : 0;
    cudaStream_t st = ws->own_stream;
    T *dp, *op; unsigned char *df, *of; int *svi, *svj; long long* oc;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        dp = cv.take<T>((size_t)3 * n);
        df = cv.take<unsigned char>(fbytes + 1);
        op = cv.take<T>((size_t)3 * n);
        svi = cv.take<int>((size_t)n);
        svj = cv.take<int>((size_t)n);
        of = cv.take<unsigned char>(fbytes + 1);
        oc = cv.take<long long>(3);
    }));
    PCU_TRY(h2d(ws, dp, points, sizeof(T) * 3 * n, st));
    if (with_faces) PCU_TRY(h2d(ws, df, faces, fbytes, st));
    PCU_TRY(dedup_dispatch<T>(ws, dp, n, epsilon, with_faces ? df : nullptr, with_faces ? nf : 0, cols, faces_are_i64, op, svi, svj,
                              with_faces ? of : nullptr, oc, st));
    long long* hc = reinterpret_cast<long long*>(ws->host_slot);
    PCU_CUDA(cudaMemcpyAsync(hc, oc, 3 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    const long long unique = hc[0], kept = hc[1];
    PCU_CUDA(cudaMemcpyAsync(out_points, op, sizeof(T) * 3 * unique, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaMemcpyAsync(out_svi, svi, sizeof(int) * unique, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaMemcpyAsync(out_svj, svj, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    if (with_faces && kept > 0)
        PCU_CUDA(cudaMemcpyAsync(out_faces, of, (size_t)(faces_are_i64 ? 8 : 4) * (size_t)cols * (size_t)kept, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < 3; ++i) out_counts[i] = hc[i];
    return PCU_B200_OK;
}

// Morton entry points on HOST arrays: up to two inputs, one output, copies either side of one device call.
template <typename Call>
int morton_host(pcu_b200_workspace* ws, const void* in_a, size_t bytes_a, const void* in_b, size_t bytes_b, void* out,
                size_t bytes_out, Call&& call) {
    if (!ws) return fail(PCU_B200_INVALID_ARGUMENT, "null workspace");
    if (!in_a || bytes_a == 0 || (bytes_b != 0 && !in_b)) return fail(PCU_B200_INVALID_ARGUMENT, "codes / pts must be non-empty arrays but got an empty array");
    if (!out) return fail(PCU_B200_INVALID_ARGUMENT, "null output pointer");
    PCU_ON_DEVICE(ws);
    cudaStream_t st = ws->own_stream;
    unsigned char *da, *db, *dout;
    PCU_TRY(carve_scratch(ws, kIo, st, [&](Carver& cv) {
        da = cv.take<unsigned char>(bytes_a);
        db = cv.take<unsigned char>(bytes_b ? bytes_b : 1);
        dout = cv.take<unsigned char>(bytes_out);
    }));
    PCU_TRY(h2d(ws, da, in_a, bytes_a, st));
    if (bytes_b) PCU_TRY(h2d(ws, db, in_b, bytes_b, st));
    PCU_TRY(call(da, db, dout, st));
    PCU_CUDA(cudaMemcpyAsync(out, dout, bytes_out, cudaMemcpyDeviceToHost, st));
    PCU_CUDA(cudaStreamSynchronize(st));
    return PCU_B200_OK;
}

}  // namespace

// =================================================================================================
extern "C" {

int pcu_b200_voxel_downsample_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, float* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream) {
    return voxel_downsample_dispatch<float>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                            min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows, (cudaStream_t)stream);
}
int pcu_b200_voxel_downsample_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, double* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream) {
    return voxel_downsample_dispatch<double>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                             min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows, (cudaStream_t)stream);
}

int pcu_b200_pairwise_distances_f32(pcu_b200_workspace* ws, const float* a, const float* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, float* out, void* stream) {
    return pairwise_device<float>(ws, a, b, nb, n, m, d, norm_kind, p, out, (cudaStream_t)stream);
}
int pcu_b200_pairwise_distances_f64(pcu_b200_workspace* ws, const double* a, const double* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, double* out, void* stream) {
    return pairwise_device<double>(ws, a, b, nb, n, m, d, norm_kind, p, out, (cudaStream_t)stream);
}
int pcu_b200_sinkhorn_f32(pcu_b200_workspace* ws, const float* a, const float* b, const float* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, float* out_P, double* out_cost, int32_t* out_iters, void* stream) {
    return sinkhorn_device<float>(ws, a, b, M, nb, n, m, eps, max_iters, stop_thresh, out_P, out_cost, out_iters, (cudaStream_t)stream);
}
int pcu_b200_sinkhorn_f64(pcu_b200_workspace* ws, const double* a, const double* b, const double* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, double* out_P, double* out_cost, int32_t* out_iters, void* stream) {
    return sinkhorn_device<double>(ws, a, b, M, nb, n, m, eps, max_iters, stop_thresh, out_P, out_cost, out_iters, (cudaStream_t)stream);
}

int pcu_b200_estimate_point_cloud_areas_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* normals, const void* idx,
                                            int k, int idx_kind, float* out_areas, uint64_t* out_bad, void* stream) {
    return point_areas_device<float>(ws, points, n, normals, idx, k, idx_kind, out_areas, (unsigned long long*)out_bad, (cudaStream_t)stream);
}
int pcu_b200_estimate_point_cloud_areas_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* normals,
                                            const void* idx, int k, int idx_kind, double* out_areas, uint64_t* out_bad, void* stream) {
    return point_areas_device<double>(ws, points, n, normals, idx, k, idx_kind, out_areas, (unsigned long long*)out_bad,
                                      (cudaStream_t)stream);
}

int pcu_b200_morton_encode_i32(pcu_b200_workspace* ws, const int32_t* pts, int64_t n, uint64_t* out_codes, void* stream) {
    return morton_encode_device<int32_t>(ws, pts, n, (unsigned long long*)out_codes, (cudaStream_t)stream);
}
int pcu_b200_morton_encode_i64(pcu_b200_workspace* ws, const int64_t* pts, int64_t n, uint64_t* out_codes, void* stream) {
    return morton_encode_device<long long>(ws, (const long long*)pts, n, (unsigned long long*)out_codes, (cudaStream_t)stream);
}
int pcu_b200_morton_decode(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, int32_t* out_pts, void* stream) {
    return morton_decode_device(ws, (const unsigned long long*)codes, n, out_pts, (cudaStream_t)stream);
}
int pcu_b200_morton_add(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream) {
    return morton_addsub_device(ws, (const unsigned long long*)a, (const unsigned long long*)b, n, 0, (unsigned long long*)out, (cudaStream_t)stream);
}
int pcu_b200_morton_subtract(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream) {
    return morton_addsub_device(ws, (const unsigned long long*)a, (const unsigned long long*)b, n, 1, (unsigned long long*)out, (cudaStream_t)stream);
}
int pcu_b200_morton_knn(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, const uint64_t* qcodes, int64_t m, int k,
                        int sort_dist, int64_t* out_idx, void* stream) {
    return morton_knn_device(ws, (const unsigned long long*)codes, n, (const unsigned long long*)qcodes, m, k, sort_dist,
                             (long long*)out_idx, (cudaStream_t)stream);
}
int pcu_b200_deduplicate_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, float* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream) {
    return dedup_dispatch<float>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                 (long long*)out_counts, (cudaStream_t)stream);
}
int pcu_b200_deduplicate_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, double* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream) {
    return dedup_dispatch<double>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                  (long long*)out_counts, (cudaStream_t)stream);
}

int pcu_b200_voxel_downsample_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const void* attrib, int attrib_cols,
                                       int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                       int min_points_per_voxel, float* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows) {
    return voxel_downsample_host<float>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                        min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows);
}
int pcu_b200_voxel_downsample_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const void* attrib, int attrib_cols,
                                       int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                       int min_points_per_voxel, double* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows) {
    return voxel_downsample_host<double>(ws, points, n, attrib, attrib_cols, attrib_is_f64, voxel_size, min_bound, max_bound,
                                         min_points_per_voxel, out_points, out_attrib, out_counts, (long long*)out_rows);
}
int pcu_b200_deduplicate_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                                  int face_cols, int faces_are_i64, float* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                                  int64_t* out_counts) {
    return deduplicate_host<float>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                   (long long*)out_counts);
}
int pcu_b200_deduplicate_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                                  int face_cols, int faces_are_i64, double* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                                  int64_t* out_counts) {
    return deduplicate_host<double>(ws, points, n, epsilon, faces, n_faces, face_cols, faces_are_i64, out_points, out_svi, out_svj, out_faces,
                                    (long long*)out_counts);
}

int pcu_b200_morton_encode_host_i32(pcu_b200_workspace* ws, const int32_t* pts, int64_t n, uint64_t* out_codes) {
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    return morton_host(ws, pts, sizeof(int32_t) * 3 * n, nullptr, 0, out_codes, sizeof(uint64_t) * n,
                       [&](unsigned char* a, unsigned char*, unsigned char* o, cudaStream_t st) {
                           return morton_encode_device<int32_t>(ws, (const int32_t*)a, n, (unsigned long long*)o, st); });
}
int pcu_b200_morton_encode_host_i64(pcu_b200_workspace* ws, const int64_t* pts, int64_t n, uint64_t* out_codes) {
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "pts must be an array of shape [n, 3] but got an empty array");
    return morton_host(ws, pts, sizeof(int64_t) * 3 * n, nullptr, 0, out_codes, sizeof(uint64_t) * n,
                       [&](unsigned char* a, unsigned char*, unsigned char* o, cudaStream_t st) {
                           return morton_encode_device<long long>(ws, (const long long*)a, n, (unsigned long long*)o, st); });
}
int pcu_b200_morton_decode_host(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, int32_t* out_pts) {
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    return morton_host(ws, codes, sizeof(uint64_t) * n, nullptr, 0, out_pts, sizeof(int32_t) * 3 * n,
                       [&](unsigned char* a, unsigned char*, unsigned char* o, cudaStream_t st) {
                           return morton_decode_device(ws, (const unsigned long long*)a, n, (int*)o, st); });
}
int pcu_b200_morton_add_host(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out) {
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes_1 must be an array of shape [n,] but got an empty array");
    return morton_host(ws, a, sizeof(uint64_t) * n, b, sizeof(uint64_t) * n, out, sizeof(uint64_t) * n,
                       [&](unsigned char* da, unsigned char* db, unsigned char* o, cudaStream_t st) {
                           return morton_addsub_device(ws, (const unsigned long long*)da, (const unsigned long long*)db, n, 0, (unsigned long long*)o, st); });
}
int pcu_b200_morton_subtract_host(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out) {
    if (n <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes_1 must be an array of shape [n,] but got an empty array");
    return morton_host(ws, a, sizeof(uint64_t) * n, b, sizeof(uint64_t) * n, out, sizeof(uint64_t) * n,
                       [&](unsigned char* da, unsigned char* db, unsigned char* o, cudaStream_t st) {
                           return morton_addsub_device(ws, (const unsigned long long*)da, (const unsigned long long*)db, n, 1, (unsigned long long*)o, st); });
}
int pcu_b200_morton_knn_host(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, const uint64_t* qcodes, int64_t m, int k,
                             int sort_dist, int64_t* out_idx) {
    if (k <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "k must be greater than 0");
    if (n <= 0 || m <= 0) return fail(PCU_B200_INVALID_ARGUMENT, "codes must be an array of shape [n] but got an empty array");
    if ((int64_t)k > n) return fail(PCU_B200_INVALID_ARGUMENT, "k (%d) exceeds the number of codes (%lld): clamp it first (morton.cpp:351)", k, (long long)n);
    return morton_host(ws, codes, sizeof(uint64_t) * n, qcodes, sizeof(uint64_t) * m, out_idx, sizeof(int64_t) * m * k,
                       [&](unsigned char* da, unsigned char* db, unsigned char* o, cudaStream_t st) {
                           return morton_knn_device(ws, (const unsigned long long*)da, n, (const unsigned long long*)db, m, k, sort_dist, (long long*)o, st); });
}

}  // extern "C"
