/*
 * pcu_b200.h -- C ABI of the GPU-native (H100, sm_90a) nearest-neighbour path (libpcu_b200.so).
 *
 * This is the drop-in boundary for the ONE hot path of fwilliams/point-cloud-utils that this
 * repository replaces: exact L2 k-nearest-neighbour search between two 3-D point clouds and the
 * Chamfer / Hausdorff scalars built on it.  Each entry point names the reference interface it
 * stands in for (paths relative to /root/reference):
 *
 *   pcu_b200_knn_*                   shortest_distances_nanoflann<>      src/point_cloud_distance.cpp:21-99
 *                                    as called by k_nearest_neighbors    src/point_cloud_distance.cpp:123-164
 *   pcu_b200_nn_stats_*              the k = 1 sweep + dists.maxCoeff    src/point_cloud_distance.cpp:219-225
 *                                    (one_sided_hausdorff_distance       src/point_cloud_distance.cpp:186-234)
 *                                    and norm(...).mean() of chamfer     point_cloud_utils/__init__.py:112-113
 *   pcu_b200_chamfer_*               chamfer_distance, p_norm = 2        point_cloud_utils/__init__.py:84-120
 *   pcu_b200_batched_chamfer_*       a Python loop of chamfer_distance over pairs (the docstring's
 *                                    "[m, n, d] minibatch", __init__.py:89-90, which the 2-D-only
 *                                    binding never implemented)
 *
 * Conventions
 *   - Plain C: raw pointers, sizes, an opaque workspace handle and a CUDA stream passed as void*.
 *     No C++ / torch / numpy types cross this boundary and no exception does either.
 *   - Every function returns a pcu_b200_status; the message of the last failure on the calling
 *     thread is available from pcu_b200_last_error().
 *   - Point clouds are dense row-major (n, 3) arrays of float (…_f32) or double (…_f64).
 *   - The caller owns every input and output buffer.  The library never allocates user-visible
 *     memory; scratch lives in the workspace (grown on demand, reused across calls).  One
 *     workspace serves one stream at a time.
 *   - "device" entry points take DEVICE pointers, enqueue work on `stream` and return without
 *     synchronising; results are valid once the stream reaches that point.  "host" entry points
 *     take HOST pointers (pinned or pageable), copy them to device staging owned by the workspace
 *     on the workspace's own streams -- the copy of the second cloud overlaps the first kernels --
 *     and return after the results have landed in the caller's buffers.  Page-locked inputs are
 *     DMA'd as they are; pageable inputs of 4 MB and more go through a 32 MB page-locked ring of
 *     the workspace, filled by eight copy threads in 512 KB chunks and drained in transfers of up
 *     to 4 MB (pcu_b200_options::host_staging; the threads start with the first such copy).
 *   - Scratch grows with stream-ordered allocation (cudaMallocAsync): no entry point synchronises
 *     the device.  A workspace serves one stream at a time; a call on another stream than the
 *     previous one is ordered after it on the device.
 *   - Results follow the reference bit for bit: squared distance is ((qx-px)^2+(qy-py)^2)+(qz-pz)^2,
 *     every operation rounded in the input precision, no FMA (nanoflann.hpp:496-507); indices are
 *     int64 (ptrdiff_t in the reference); rows are ascending by distance; queries whose answer
 *     depends on how equal distances are ordered are re-answered on the GPU by a replica of the
 *     reference's kd-tree traversal (visit order decides, nanoflann.hpp:194-227) built with the
 *     caller's max_points_per_leaf; fewer than k neighbours (k > m) pads with -1 / -1.0
 *     (src/point_cloud_distance.cpp:90-93).
 */
#ifndef PCU_B200_H
#define PCU_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCU_B200_ABI_VERSION 3

typedef enum pcu_b200_status {
    PCU_B200_OK = 0,
    PCU_B200_INVALID_ARGUMENT = 1, /* maps to ValueError in the Python layer (pybind11::value_error in the reference) */
    PCU_B200_CUDA_ERROR = 2,       /* maps to RuntimeError */
    PCU_B200_OUT_OF_MEMORY = 3,    /* maps to MemoryError */
    PCU_B200_NO_DEVICE = 4,        /* no usable sm_90 (H100) device: the product has no CPU fallback */
    PCU_B200_INTERNAL = 5
} pcu_b200_status;

typedef struct pcu_b200_workspace pcu_b200_workspace;

/* Per-direction result of the fused k = 1 sweep (no per-point distance buffer is written). */
typedef struct pcu_b200_nn_stats {
    /* A query has a neighbour when some point's rounded d2 is below FLT_MAX / DBL_MAX (nanoflann's admission   */
    /* rule); a query without one counts as d2_min = -1 in max_sq_dist and makes both sums +inf.                */
    double sum_dist;      /* sum over queries of sqrt(d2_min), accumulated in fp64                */
    double sum_sq_dist;   /* sum over queries of d2_min, accumulated in fp64                      */
    double max_sq_dist;   /* largest d2_min (exact: the input-precision value widened to double); */
                          /* -1 when no query has a neighbour                                      */
    int64_t argmax_query; /* first (lowest-index) query attaining it (Eigen maxCoeff, :221-223)   */
    int64_t argmax_data;  /* its nearest neighbour in the dataset (:225); -1 when it has none     */
    int64_t n_queries;    /* n                                                                    */
    int64_t n_tied;       /* -1: the fused sweeps track distances only (ties only matter to witness_tied) */
    int64_t n_far;        /* queries that needed the ring-expansion slow path (diagnostic)        */
    int64_t witness_tied; /* 1: argmax_query had several equally near neighbours, so argmax_data  */
                          /* is the lowest such index, not necessarily the reference's pick; the  */
                          /* host entry points resolve this themselves, device callers use        */
                          /* pcu_b200_resolve_witness_* (value, sums and argmax_query are final)   */
    double pair_value;    /* bidirectional calls (pcu_b200_chamfer_*): the pair's Chamfer value in fp64,  */
                          /* sum_dist[x->y] / n + sum_dist[y->x] / m, written to BOTH records by the sweep */
                          /* that finishes second (what a multi-GPU caller sums across ranks);            */
                          /* one-directional calls: sum_dist / n_queries                                  */
} pcu_b200_nn_stats;

/* Tunables; zero-initialise and override what you need.  0 always means "library default". */
typedef struct pcu_b200_options {
    int max_points_per_leaf; /* reference kwarg; only influences how exact-distance ties are ordered (default 10) */
    float cell_occupancy;    /* target dataset points per grid cell (0 = default: 1.5 for k = 1; 3 / 4 / 7 / 12  */
                             /* at k = 4 / 8 / 16 / 32, interpolated in between -- measured, DESIGN.md section 4) */
    int disable_tie_replay;  /* diagnostic only.  1: keep the (distance, lowest index) order for tied queries;        */
                             /* 2: replay on full reference trees only (no pruned build); 3: pruned build with    */
                             /* zero slack (every walk hits a stub, which exercises the full-rebuild path)        */
    int binning;             /* 0: automatic (one CTA per cloud up to 8192 points, the cell-wise passes for a    */
                             /* single pair up to 65536, else the slab build); 1: always the cell-wise          */
                             /* passes; 2: the one-CTA-per-cloud build whenever a cloud's cell counters fit in   */
                             /* shared memory; 3: the slab build above 8192 points, batches included             */
                             /* (1 .. 3 are diagnostic only)                                                      */
    int host_staging;        /* host entry points, inputs of >= 4 MB: 0 pageable memory goes through the          */
                             /* workspace's pinned ring filled by copy threads, pinned memory is DMA'd as it is;  */
                             /* 1 always the ring; 2 never (plain cudaMemcpyAsync: the driver stages)             */
} pcu_b200_options;

/* ---- library / error plumbing ------------------------------------------------------------ */
int pcu_b200_abi_version(void);
const char* pcu_b200_last_error(void);
/* Number of CUDA devices this build can run on (compute capability 10.x); 0 if none. */
int pcu_b200_device_count(void);
/* The device a call that names none runs on.  The reference's interface (src/point_cloud_distance.cpp:123-131,
 * :186-193) has no device argument, so the replacement has to pick one: the environment variable
 * PCU_B200_DEVICE if set; else the CUDA runtime's current device of the calling thread when that is not 0
 * (torch.cuda.set_device / `with torch.cuda.device(i)`); else LOCAL_RANK when a launcher (torchrun) set it
 * and that many devices are visible; else 0. */
int pcu_b200_current_device(void);
/* Kernels launched by this library on the calling process since load (bench.py's gpu_launches). */
int64_t pcu_b200_launch_count(void);

/* Page-locked host memory (cudaHostAlloc / cudaFreeHost), for callers that want their big result buffers to
 * be copy targets the DMA engines can write directly: the numpy-facing binding backs k-NN results of 1 MiB and
 * more with such blocks (recycled through a small pool), because a device-to-host copy into freshly allocated
 * pageable memory runs at ~3 GB/s -- the page faults, not PCIe -- against ~50 GB/s into pinned memory.
 * The block is placed on the NUMA node of the calling thread's current GPU (the PCI device's numa_node in sysfs):
 * on two-socket hosts a page-locked buffer on the other node is copied at half the rate or less. */
int pcu_b200_host_alloc(void** out_ptr, int64_t bytes);
int pcu_b200_host_free(void* ptr);

/* ---- workspace ---------------------------------------------------------------------------- */
int pcu_b200_workspace_create(int device, pcu_b200_workspace** out_ws);
int pcu_b200_workspace_destroy(pcu_b200_workspace* ws);
/* The device the workspace was created on (-1 for NULL).  Every entry point runs there and leaves the
 * calling thread's current device as it found it. */
int pcu_b200_workspace_device(const pcu_b200_workspace* ws);
/* Bytes of device scratch currently held. */
int64_t pcu_b200_workspace_bytes(const pcu_b200_workspace* ws);
int pcu_b200_workspace_set_options(pcu_b200_workspace* ws, const pcu_b200_options* opts);
/* Diagnostic: how much finer than the default the two clouds' grids of the NEXT call with the last call's
 * shapes will be (1 = default cells per point).  The library learns this from the fill statistics each
 * call leaves behind: surfaces and other thin point sets get finer grids from the second call on.  It
 * changes speed only, never results. */
int pcu_b200_workspace_grid_refinement(const pcu_b200_workspace* ws, float out_mult[2]);
/* Per-stage device timing (diagnostic; bench.py's roofline pass).  When enabled, every device entry
 * point records CUDA events on the launching stream between its stages; after that stream has been
 * synchronised, last_profile() returns the milliseconds of the LAST call's 8 stages (descriptors,
 * bbox+grid, slab_count, partition, cell_sort, search, search_far, finalize) and their count (0 if none);
 * the three grid-build slots after bbox+grid hold the slab build's kernels, or cell_count, scan_lookback
 * and scatter where the cell-wise passes run, or nothing where one CTA bins a whole cloud; after a
 * host entry point and with capacity >= 10, two more: the host-to-device copies in front of the first stage
 * and the device-to-host copies behind the last ("h2d", "d2h"). */
int pcu_b200_workspace_set_profiling(pcu_b200_workspace* ws, int enabled);
int pcu_b200_workspace_last_profile(pcu_b200_workspace* ws, float* out_ms, int capacity);
const char* pcu_b200_profile_stage_name(int stage);

/* ---- k nearest neighbours, DEVICE pointers -------------------------------------------------
 * out_dist : (n, k) row-major, input precision; sqrt(d2) unless squared != 0
 * out_idx  : (n, k) row-major int64 indices into dataset
 * out_n_tied (may be NULL): device int64 that receives the number of queries that went through
 *            the tie replay.
 * The call never synchronises: the kd-tree replay is one cooperative launch gated, on the device, on
 * the number of flagged queries (it returns at once when that number is zero).
 * Replaces shortest_distances_nanoflann (src/point_cloud_distance.cpp:21-99).                    */
int pcu_b200_knn_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m, int k,
                     int squared, float* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream);
int pcu_b200_knn_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m, int k,
                     int squared, double* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream);

/* ---- fused k = 1 sweep + reductions, DEVICE pointers ---------------------------------------
 * out_stats : device pointer to ONE pcu_b200_nn_stats (query -> dataset direction).
 * Replaces the k = 1 sweep, dists.maxCoeff and corrs(i, 0) of one_sided_hausdorff_distance
 * (src/point_cloud_distance.cpp:219-225).                                                        */
int pcu_b200_nn_stats_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m,
                          pcu_b200_nn_stats* out_stats, void* stream);
int pcu_b200_nn_stats_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m,
                          pcu_b200_nn_stats* out_stats, void* stream);

/* Re-answers stats->argmax_query with the reference's tie order (kd-tree replay built with
 * max_points_per_leaf) and stores the result in stats->argmax_data; clears witness_tied.
 * `stats` is a DEVICE pointer to one record produced by the calls above for (query, dataset).
 * Synchronises the stream once (the workspace scratch is re-carved for the replay).              */
int pcu_b200_resolve_witness_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset,
                                 int64_t m, pcu_b200_nn_stats* stats, void* stream);
int pcu_b200_resolve_witness_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset,
                                 int64_t m, pcu_b200_nn_stats* stats, void* stream);

/* ---- fused bidirectional Chamfer (+ Hausdorff), DEVICE pointers ----------------------------
 * out_stats : device pointer to TWO pcu_b200_nn_stats: [0] = x -> y, [1] = y -> x.
 * out_value : device pointer to one scalar of the input precision:
 *             chamfer = stats[0].sum_dist / n + stats[1].sum_dist / m   (no 1/2, not squared;
 *             point_cloud_utils/__init__.py:112-115).  May be NULL.
 * Both clouds are binned once and swept in one launch; no distance buffer is materialised.       */
int pcu_b200_chamfer_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const float* y, int64_t m,
                         pcu_b200_nn_stats* out_stats, float* out_value, void* stream);
int pcu_b200_chamfer_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const double* y, int64_t m,
                         pcu_b200_nn_stats* out_stats, double* out_value, void* stream);

/* ---- prepared clouds: bin a fixed cloud ONCE, use it as one side of many calls ---------------
 * The reference rebuilds its kd-tree on every call -- three times per direction (src/point_cloud_distance.cpp:41-42,
 * nanoflann.hpp:1357, 2288) -- even when one cloud never changes (a loss against a fixed target evaluated every
 * iteration).  pcu_b200_cloud_prepare_* copies the points into a private device block and bins them there; the
 * *_prepared_* calls take the handle as the SECOND cloud (y / target / dataset), bin only the first cloud and run
 * the same fused sweeps: results are those of the unprepared calls bit for bit.  Host variants copy only the first
 * cloud over PCIe.  A handle may serve calls on several workspaces / streams of its device at once (it is
 * read-only after preparation, apart from an occupancy pyramid every user would write identically).
 * pcu_b200_cloud_destroy synchronises the device. */
typedef struct pcu_b200_cloud pcu_b200_cloud;
int pcu_b200_cloud_prepare_f32(pcu_b200_workspace* ws, const float* points, int64_t n, pcu_b200_cloud** out_cloud, void* stream);
int pcu_b200_cloud_prepare_f64(pcu_b200_workspace* ws, const double* points, int64_t n, pcu_b200_cloud** out_cloud, void* stream);
int pcu_b200_cloud_prepare_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, pcu_b200_cloud** out_cloud);
int pcu_b200_cloud_prepare_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, pcu_b200_cloud** out_cloud);
/* The same for k-NN calls: the cell size is chosen for searches with this k, and the reference's kd-tree replica (leaf
 * size max_points_per_leaf, 0 = 10) is built once into the handle, so that pcu_b200_knn_prepared_* neither bins the
 * dataset nor builds the tree -- it only replays its tied rows on it (the reference builds its tree in every call,
 * src/point_cloud_distance.cpp:41-42).  A call whose options name another leaf size builds its own tree as usual.
 * The handle's tree counters and pyramid are shared state: one k-NN call at a time per handle. */
int pcu_b200_cloud_prepare_knn_f32(pcu_b200_workspace* ws, const float* points, int64_t n, int k, int max_points_per_leaf,
                                   pcu_b200_cloud** out_cloud, void* stream);
int pcu_b200_cloud_prepare_knn_f64(pcu_b200_workspace* ws, const double* points, int64_t n, int k, int max_points_per_leaf,
                                   pcu_b200_cloud** out_cloud, void* stream);
int pcu_b200_cloud_prepare_knn_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, int k, int max_points_per_leaf,
                                        pcu_b200_cloud** out_cloud);
int pcu_b200_cloud_prepare_knn_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, int k, int max_points_per_leaf,
                                        pcu_b200_cloud** out_cloud);
/* k nearest neighbours of `query` in a prepared cloud: outputs as pcu_b200_knn_* (same results, bit for bit). */
int pcu_b200_knn_prepared_f32(pcu_b200_workspace* ws, const float* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                              float* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream);
int pcu_b200_knn_prepared_f64(pcu_b200_workspace* ws, const double* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                              double* out_dist, int64_t* out_idx, int64_t* out_n_tied, void* stream);
int pcu_b200_knn_prepared_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                                   float* out_dist, int64_t* out_idx, int64_t* out_n_tied);
int pcu_b200_knn_prepared_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, pcu_b200_cloud* dataset, int k, int squared,
                                   double* out_dist, int64_t* out_idx, int64_t* out_n_tied);
int pcu_b200_cloud_destroy(pcu_b200_cloud* cloud);
int64_t pcu_b200_cloud_size(const pcu_b200_cloud* cloud);
/* DEVICE pointer to the handle's private (n, 3) copy of the points (what pcu_b200_resolve_witness_* wants as the
 * prepared side's array). */
const void* pcu_b200_cloud_points(const pcu_b200_cloud* cloud);
/* out_stats: TWO records ([0] = x -> y, [1] = y -> x) as for pcu_b200_chamfer_*; out_value may be NULL */
int pcu_b200_chamfer_prepared_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const pcu_b200_cloud* y,
                                  pcu_b200_nn_stats* out_stats, float* out_value, void* stream);
int pcu_b200_chamfer_prepared_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const pcu_b200_cloud* y,
                                  pcu_b200_nn_stats* out_stats, double* out_value, void* stream);
/* out_stats: ONE record (query -> dataset) as for pcu_b200_nn_stats_* */
int pcu_b200_nn_stats_prepared_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const pcu_b200_cloud* dataset,
                                   pcu_b200_nn_stats* out_stats, void* stream);
int pcu_b200_nn_stats_prepared_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const pcu_b200_cloud* dataset,
                                   pcu_b200_nn_stats* out_stats, void* stream);
int pcu_b200_chamfer_prepared_host_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const pcu_b200_cloud* y,
                                       pcu_b200_nn_stats* out_stats, float* out_value);
int pcu_b200_chamfer_prepared_host_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const pcu_b200_cloud* y,
                                       pcu_b200_nn_stats* out_stats, double* out_value);
int pcu_b200_nn_stats_prepared_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const pcu_b200_cloud* dataset,
                                        pcu_b200_nn_stats* out_stats);
int pcu_b200_nn_stats_prepared_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const pcu_b200_cloud* dataset,
                                        pcu_b200_nn_stats* out_stats);

/* ---- batched Chamfer over independent pairs, DEVICE pointers -------------------------------
 * x : (B, n, 3), y : (B, m, 3) dense; out_per_pair : (B) scalars of the input precision;
 * out_sum (may be NULL): device double = sum of the B per-pair values (the quantity a multi-GPU
 * caller all-reduces).                                                                            */
int pcu_b200_batched_chamfer_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch, int64_t n,
                                 int64_t m, float* out_per_pair, double* out_sum, void* stream);

/* ---- point-cloud normals from k nearest neighbours (SURVEY.md 8f, N1) ----------------------
 * Replaces estimate_point_cloud_normals_knn_internal (src/point_cloud_normals.cpp:375-411, estimator :115-173):
 * for every point its k nearest points of the same cloud (itself included), the unit normal of the plane
 * fitted to them, and -- when view_dirs (n, 3) is not NULL -- orientation towards the view direction and
 * dropping of points whose normal makes an angle above drop_angle_threshold (radians) with it.
 * out_idx (capacity n) / out_normals (capacity n x 3): the kept points in ascending row order; out_count: how
 * many.  The neighbour sets are the reference's bit for bit (same exact k-NN, same tie order); the plane fit is
 * the smallest eigenvector of the fp64 scatter matrix, equal to the reference's JacobiSVD vector up to rounding
 * and, without view directions, up to sign.  DEVICE pointers; out_count is a device int64. */
int pcu_b200_normals_knn_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs, int k,
                             double drop_angle_threshold, int64_t* out_idx, float* out_normals, int64_t* out_count, void* stream);
int pcu_b200_normals_knn_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs, int k,
                             double drop_angle_threshold, int64_t* out_idx, double* out_normals, int64_t* out_count, void* stream);

/* ---- duplicate removal (SURVEY.md 8f, N2) ---------------------------------------------------
 * Replaces deduplicate_point_cloud / deduplicate_mesh_vertices (src/remove_duplicates.cpp:108-176, helpers :11-79;
 * libigl's round + unique_rows underneath).  epsilon > 0: rows are compared after round(p / epsilon) (division in the
 * cloud's precision, halves away from zero); otherwise as they are.  Unique rows come in ascending lexicographic
 * order of the compared values.
 *   out_points (capacity n x 3): points[out_svi];  out_svi (capacity n): for every unique row the FIRST input row of its
 *   cluster (libigl returns an unspecified member: its row sort is not stable);  out_svj (n): unique row of every input
 *   row;  faces (may be NULL): (n_faces, face_cols) int32 or int64 vertex indices -> out_faces (capacity n_faces x
 *   face_cols) holds the re-indexed faces whose corners stay distinct, in their original order.
 *   out_counts: 3 device int64 = { unique points, surviving faces, faces with a corner outside [0, n) (dropped) }.
 * DEVICE pointers. */
int pcu_b200_deduplicate_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, float* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream);
int pcu_b200_deduplicate_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                             int face_cols, int faces_are_i64, double* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                             int64_t* out_counts, void* stream);

/* ---- point-cloud normals from all points in a ball (SURVEY.md 8f, N1) -----------------------
 * Replaces estimate_point_cloud_normals_ball_internal (src/point_cloud_normals.cpp:303-370, estimator :48-113).
 * The neighbourhood of a point is what the reference's call nanoflann radiusSearch(query, ball_radius) returns:
 * every point (itself included) whose SQUARED distance, rounded like the reference's metric, is below
 * (scalar)radius -- nanoflann's radius is in squared units and the reference passes ball_radius as it is -- while
 * the weight function sees the true distance: 1 ("constant") or (1 - d/r)^4 (4 d/r + 1) ("rbf").  Points with
 * fewer than min_pts_per_ball neighbours are dropped; with max_pts_per_ball > 0 a uniformly random subset of that
 * size is fitted (the reference shuffles with rand(); here selection sampling from a hash of seed, row, position:
 * same distribution, reproducible for a given seed, not the same subset).  Outputs as for the k-NN variant. */
typedef struct pcu_b200_ball_options {
    double radius;                 /* > 0 */
    double drop_angle_threshold;   /* radians; only used with view directions */
    int32_t min_pts_per_ball;      /* >= 3 */
    int32_t max_pts_per_ball;      /* <= 0: no limit, else >= 3 */
    int32_t weight_function;       /* 0 "constant", 1 "rbf" */
    uint32_t seed;                 /* subset selection when max_pts_per_ball > 0 */
} pcu_b200_ball_options;
int pcu_b200_normals_ball_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs,
                              const pcu_b200_ball_options* options, int64_t* out_idx, float* out_normals, int64_t* out_count, void* stream);
int pcu_b200_normals_ball_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs,
                              const pcu_b200_ball_options* options, int64_t* out_idx, double* out_normals, int64_t* out_count, void* stream);

/* ---- Poisson-disk down-sampling ---------------------------------------------------------------
 * Replaces blue_noise_downsample as called by downsample_point_cloud_poisson_disk (src/sample_point_cloud.cpp:14-109,
 * :328) for one radius; the target-count search around it (:278-326) stays with the caller, one call per radius.
 * The reference's subset (libigl blue_noise + std::mt19937 over an unordered_map) cannot be reproduced; the sample
 * here is a pure function of (points, radius, seed):
 *   r = (scalar)radius, rr = r * r rounded in the scalar type (:16, :72);  rows p, q conflict iff d2(p, q) < rr, d2
 *   rounded like the library's metric (the boundary d2 == rr is unpinned against the reference);  every row has the
 *   key (mix32(seed ^ mix32(row * 0x9e3779b9 + 0x85ebca6b)), row), 32-bit wrap-around, compared lexicographically;
 *   the sample is the greedy maximal independent set in key order (visit rows by ascending key, keep a row that
 *   conflicts with no kept row): no two samples conflict, every row is a sample or conflicts with one.
 *   radius > 0; n <= 2^31 - 1.  out_idx (capacity n, int32): the sampled rows, ascending;  out_count: device int64;
 *   out_rounds (may be NULL): device int32, selection rounds run (one grid barrier each).  DEVICE pointers. */
int pcu_b200_poisson_disk_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double radius, uint32_t seed,
                              int32_t* out_idx, int64_t* out_count, int32_t* out_rounds, void* stream);
int pcu_b200_poisson_disk_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double radius, uint32_t seed,
                              int32_t* out_idx, int64_t* out_count, int32_t* out_rounds, void* stream);

/* ---- Voronoi cells in the unit cube / square and Lloyd relaxation ------------------------------
 * Replace voronoi_centroids_unit_cube, lloyd_3d and lloyd_2d (src/lloyd.cpp:166-300), whose geogram restricted Voronoi
 * diagram, initial sampling and HLBFGS Newton iterations are not available; the results are defined in DESIGN.md §3:
 *   cell V_i = {x in [0,1]^dim : |x - c_i|^2 <= |x - c_j|^2 for every c_j != c_i}; seeds at one position share one cell,
 *   owned by the lowest index.  Centroid row i = centroid of V_i when vol(V_i) > 1e-30, else c_i.  All fp64.
 * pcu_b200_voronoi_centroids: centers (n, dim) and out_centroids (n, dim) are DEVICE pointers; centers must lie in
 *   [0,1]^dim (outside it the rows are unspecified).  dim 2 or 3, 1 <= n <= 2^31 - 2.  out_moments (DEVICE, may be NULL):
 *   (n, 5) per cell: volume, first moment about the seed (x, y, z; z = 0 in 2-D), second moment about the seed.
 * pcu_b200_lloyd: the initial sample of (n, dim, seed), num_lloyd centroid steps, then at most num_newton L-BFGS steps on
 *   the CVT energy; out_points (n, dim) DEVICE.  out_energy (HOST, num_newton + 1 doubles, may be NULL): the energy of
 *   the starting point and of every accepted Newton step; out_newton_steps (HOST, may be NULL): accepted steps.
 * out_passes (HOST, 3 int64, may be NULL): cells handled by the first pass, the longer-list pass and the all-seeds pass,
 *   summed over every cell evaluation of the call.  Both calls synchronise `stream` (the fallback passes are sized on
 *   the host; DESIGN.md §8). */
int pcu_b200_voronoi_centroids(pcu_b200_workspace* ws, const double* centers, int64_t n, int dim, double* out_centroids,
                               double* out_moments, int64_t* out_passes, void* stream);
int pcu_b200_lloyd(pcu_b200_workspace* ws, int64_t n, int dim, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                   double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream);

/* ---- Voronoi cells restricted to a triangle mesh and Lloyd sampling of its surface -----------------------------
 * Replace sample_mesh_lloyd (src/lloyd.cpp:357-401), whose geogram restricted Voronoi diagram and initial sampling are
 * not available; the results are defined in DESIGN.md §3:
 *   cell R_i = {y on the faces : |y - x_i|^2 <= |y - x_j|^2 for every x_j != x_i}; seeds at one position share one
 *   cell, owned by the lowest index; faces of zero area contribute nothing; seeds need not lie on the faces.  All fp64.
 * v (nv, 3), f (nf, 3) of index kind f_kind (pcu_b200_index_kind) and every array below are DEVICE pointers.
 * pcu_b200_restricted_voronoi_moments: seeds (n, 3), 1 <= n <= 2^31 - 2; out_moments (n, 5) per cell: area, first
 *   moment about the seed (x, y, z), second moment about the seed.  A face with a corner out of range fails the call.
 * pcu_b200_sample_mesh_lloyd: the first num_samples samples of pcu_b200_sample_mesh_random_f64 at `seed` (their
 *   positions fl((b0 a + b1 b) + b2 c)), num_lloyd centroid steps, then at most num_newton L-BFGS steps on the energy
 *   sum_i int_{R_i} |y - x_i|^2 dA with no domain test; out_points (num_samples, 3).  out_energy (HOST, num_newton + 1
 *   doubles, may be NULL) and out_newton_steps (HOST, may be NULL) as for pcu_b200_lloyd.  A face with a corner out of
 *   range or a mesh of zero area fails the call (PCU_B200_INVALID_ARGUMENT).
 * out_passes (HOST, 3 int64, may be NULL): (face, seed) pairs handled by the first pass, the longer-list pass and the
 *   all-seeds pass, summed over every cell evaluation of the call.  Both calls synchronise `stream` (the pairs and the
 *   fallback passes are sized on the host); too many pairs for device memory fail with PCU_B200_OUT_OF_MEMORY. */
int pcu_b200_restricted_voronoi_moments(pcu_b200_workspace* ws, const double* seeds, int64_t n, const double* v, int64_t nv,
                                        const void* f, int64_t nf, int f_kind, double* out_moments, int64_t* out_passes, void* stream);
int pcu_b200_sample_mesh_lloyd(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                               int64_t num_samples, uint32_t seed, int num_lloyd, int num_newton, double* out_points,
                               double* out_energy, int32_t* out_newton_steps, int64_t* out_passes, void* stream);

/* ---- mesh sampling and barycentric interpolation ----------------------------------------------
 * Replaces sample_mesh_random / sample_mesh_poisson_disk (src/sample_mesh.cpp) and interpolate_barycentric_coords
 * (point_cloud_utils/__init__.py:203-217).  The reference draws with std::rand and libigl; the samples here are pure
 * functions of (v, f, seed), defined in DESIGN.md §3 and csrc/meshsample.cuh:
 *   face weights  A_f = |(b - a) x (c - a)| in fp64, every operation rounded on its own; 0 when not finite or when a
 *                 corner is outside [0, nv) (such faces are counted in bad_faces);  scale S = 2^(62 - ceil(log2 nf)) / max A
 *                 (0 when max A = 0);  w_f = floor(A_f * S) (uint64);  C = inclusive prefix sum of w;  W = C[nf - 1].
 *   sample s      h(j) = mix64(mix64(3 s + j) ^ seed), mix64 = splitmix64 with its +0x9E3779B97F4A7C15 step;
 *                 face = first f with C_f > mulhi64(h(0), W);  u1, u2 = (h(1) >> 11) 2^-53, (h(2) >> 11) 2^-53;
 *                 a = sqrt(u1);  bc = (1 - a, a (1 - u2), a u2) in fp64, rounded once to the vertices' type.
 * Faces are (nf, 3) integers of the kind f_kind; every pointer is a DEVICE pointer and every call is stream-ordered. */
enum pcu_b200_index_kind { PCU_B200_INDEX_I32 = 0, PCU_B200_INDEX_I64 = 1, PCU_B200_INDEX_U32 = 2, PCU_B200_INDEX_U64 = 3 };
typedef struct pcu_b200_mesh_area {
    uint64_t total_weight;   /* W; 0: the mesh has zero area.  The total area is total_weight / scale / 2. */
    double scale;            /* S */
    uint64_t bad_faces;      /* faces with a corner outside [0, nv): weight 0 (the reference reads out of bounds) */
} pcu_b200_mesh_area;
/* Writes {W, S, bad_faces} to *out_area (device, 24 bytes). */
int pcu_b200_mesh_area_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                           pcu_b200_mesh_area* out_area, void* stream);
int pcu_b200_mesh_area_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                           pcu_b200_mesh_area* out_area, void* stream);
/* Samples 0 .. num_samples - 1: out_fidx (num_samples, f's width: 4 bytes for I32 / U32, 8 for I64 / U64), out_bc
 * (num_samples, 3).  out_area (may be NULL) receives {W, S, bad_faces}; when W == 0 the outputs are not written. */
int pcu_b200_sample_mesh_random_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                    int64_t num_samples, uint32_t seed, void* out_fidx, float* out_bc, pcu_b200_mesh_area* out_area,
                                    void* stream);
int pcu_b200_sample_mesh_random_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                    int64_t num_samples, uint32_t seed, void* out_fidx, double* out_bc, pcu_b200_mesh_area* out_area,
                                    void* stream);
/* Draws the samples 0 .. n_dense - 1, positions p_s = fl((bc0 a + bc1 b) + bc2 c) per axis in fp64 from the unrounded
 * coordinates, selects among them with pcu_b200_poisson_disk_* at (radius, seed), and writes the kept samples' faces
 * and coordinates in ascending sample order: out_fidx / out_bc (capacity n_dense), out_count (device int64).
 * radius > 0, 1 <= n_dense <= 2^31 - 1; the caller derives both from {W, S} (pcu_b200_mesh_area_*). */
int pcu_b200_sample_mesh_poisson_disk_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                          double radius, int64_t n_dense, uint32_t seed, void* out_fidx, float* out_bc,
                                          int64_t* out_count, void* stream);
int pcu_b200_sample_mesh_poisson_disk_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                          double radius, int64_t n_dense, uint32_t seed, void* out_fidx, double* out_bc,
                                          int64_t* out_count, void* stream);
/* out[i, d] = ((x0 b0 + x1 b1) + x2 b2), x_k = attribute[f[fi[i], k], d], products and sums in the output type with
 * no FMA (numpy's (attribute[f[fi]] * bc[:, :, None]).sum(1) bit for bit).  Negative indices of signed kinds wrap as
 * in numpy; a row with an index out of range is never loaded: it is NaN and counted in *out_bad (device uint64).
 * _f32: bc and attribute float32; _f64: each float32 or float64. */
int pcu_b200_interpolate_barycentric_f32(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, const void* fi, int64_t n,
                                         int fi_kind, const float* bc, const float* attribute, int64_t nv, int64_t dim, float* out,
                                         uint64_t* out_bad, void* stream);
int pcu_b200_interpolate_barycentric_f64(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, const void* fi, int64_t n,
                                         int fi_kind, const void* bc, int bc_is_f64, const void* attribute, int attribute_is_f64,
                                         int64_t nv, int64_t dim, double* out, uint64_t* out_bad, void* stream);

/* ---- closest points on a mesh ---------------------------------------------------------------------------------
 * Replaces closest_points_on_mesh (src/closest_point_on_mesh.cpp, libigl's AABB tree).  For each query p_i (np rows,
 * np >= 0): out_d[i] = sqrt(d^2), out_fidx[i] (f's width: 4 bytes for I32 / U32, 8 for I64 / U64) and out_bc[i, 0:3]
 * of the face that minimises (d^2, face index) lexicographically, d^2 and bc from the Voronoi-region closest point on
 * each face in the vertices' precision with every operation rounded on its own (DESIGN.md §3, csrc/meshquery.cuh).
 * Faces with a corner outside [0, nv) are left out and counted in *out_bad (device uint64); when it is not zero the
 * outputs are unspecified.  Every pointer is a DEVICE pointer and the call is stream-ordered. */
int pcu_b200_closest_points_on_mesh_f32(pcu_b200_workspace* ws, const float* p, int64_t np, const float* v, int64_t nv, const void* f,
                                        int64_t nf, int f_kind, float* out_d, void* out_fidx, float* out_bc, uint64_t* out_bad,
                                        void* stream);
int pcu_b200_closest_points_on_mesh_f64(pcu_b200_workspace* ws, const double* p, int64_t np, const double* v, int64_t nv, const void* f,
                                        int64_t nf, int f_kind, double* out_d, void* out_fidx, double* out_bc, uint64_t* out_bad,
                                        void* stream);

/* ---- winding numbers and signed distances to a mesh -------------------------------------------------------------
 * Replace triangle_soup_fast_winding_number (src/fast_winding_numbers.cpp) and signed_distance_to_mesh
 * (src/signed_distance.cpp), libigl's fast winding numbers (Barill et al. 2018).  Both build the tree of the closest-point
 * query over the valid faces, with Barill's order-2 far-field data on every node (DESIGN.md §3, csrc/winding.cuh).
 *   fast_winding_number: out_w[i] (nq rows) is the winding number at q_i, evaluated in fp32 with an fp64 sum; a node
 *     whose centre is more than accuracy_scale times its radius from q_i contributes its expansion.  accuracy_scale
 *     must be positive (the library's functions use 2); +inf evaluates every face exactly.  The result is a function of
 *     (v, f, q_i) alone.
 *   signed_distance_to_mesh: out_fidx (int32) and out_bc are those of closest_points_on_mesh; out_s[i] =
 *     fl(fl(1 - 2|w_i|) d_i), w_i the winding number at accuracy_scale 2.  Queries whose squared distance lies outside
 *     libigl's band of (lower_bound, upper_bound) get out_s = NaN, out_fidx = nf + 1, out_bc = NaN.  The bounds are
 *     float, as the reference binding's are.
 * Faces with a corner outside [0, nv) are left out and counted in *out_bad (device uint64); when it is not zero the
 * outputs are unspecified.  Every pointer is a DEVICE pointer and the call is stream-ordered. */
int pcu_b200_fast_winding_number_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                     const float* q, int64_t nq, double accuracy_scale, float* out_w, uint64_t* out_bad, void* stream);
int pcu_b200_fast_winding_number_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                     const double* q, int64_t nq, double accuracy_scale, double* out_w, uint64_t* out_bad, void* stream);
/* Replaces point_cloud_fast_winding_number (src/fast_winding_numbers.cpp): the winding number of the oriented point
 * cloud (p, n, a) (np points; p and n (np, 3), a np values) at the nq queries q, out_w[i] (nq rows).  Each point
 * contributes the dipole a_i n_i . (p_i - q) / |p_i - q|^3 (n used as given, not normalised); the same tree, far field
 * and fp64 sum as fast_winding_number, over the points (DESIGN.md §3).  accuracy_scale as there: positive, 2 in the
 * library's function, +inf evaluates every point exactly.  np = 0 gives out_w = 0.  np and nq are below 2^31 - 1.
 * Every pointer is a DEVICE pointer and the call is stream-ordered. */
int pcu_b200_point_cloud_fast_winding_number_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* a, int64_t np,
                                                 const float* q, int64_t nq, double accuracy_scale, float* out_w, void* stream);
int pcu_b200_point_cloud_fast_winding_number_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* a, int64_t np,
                                                 const double* q, int64_t nq, double accuracy_scale, double* out_w, void* stream);
/* Replaces estimate_point_cloud_areas (src/point_areas.cpp, libigl's igl::copyleft::cgal::point_areas): out_areas[r]
 * (n rows) is the area of point idx[r, 0] from the neighbour row idx[r, 0:k], defined in DESIGN.md §3 -- the neighbours
 * whose normals have a positive dot product with the centre's, projected onto their PCA plane, and the centre's mixed
 * Voronoi area over its star in the 2-D Delaunay triangulation; fp64 throughout, rounded once to the suffix's type.
 * points and normals (n, 3), idx (n, k) of kind idx_kind (pcu_b200_index_kind), 0 <= k <= 256, 0 <= n < 2^31 - 1.
 * Entries of idx outside [0, n) are left out of their row and counted in *out_bad (device uint64); when it is not zero
 * the outputs are unspecified.  Every pointer is a DEVICE pointer and the call is stream-ordered. */
int pcu_b200_estimate_point_cloud_areas_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* normals, const void* idx,
                                            int k, int idx_kind, float* out_areas, uint64_t* out_bad, void* stream);
int pcu_b200_estimate_point_cloud_areas_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* normals,
                                            const void* idx, int k, int idx_kind, double* out_areas, uint64_t* out_bad, void* stream);
/* pointcloud_apss_curvature and project_points_onto_apss: the algebraic point set surface (Guennebaud & Gross 2007,
 * the spherical fit with beta = 1) of the oriented cloud (p, n) with ball radius r, a true distance, finite and > 0
 * (DESIGN.md §3).  Each query is iterated onto the surface (at most 20 steps, until a step of at most 1e-10 r):
 * out_x (nq, 3) its projection, out_n (nq, 3) the unit normal and out_kh (nq) the signed mean curvature of the last
 * fitted sphere, +1/R on a sphere with outward normals.  Normals are normalised in fp64; a zero normal leaves its
 * point out of every fit.  A query whose ball holds fewer than 4 points with a normal, or whose fit has no step, is
 * undetermined: x = NaN, n = 0, kh = NaN; np = 0 makes every query undetermined.  fp64 throughout, rounded once.
 * q == NULL: the queries are the points themselves (nq = np), run in cell order, each result in its point's row.
 * out_x and out_n may be NULL.  0 <= np < 2^31 - 1.  Every pointer is a DEVICE pointer and the call is stream-ordered:
 * it does not synchronise. */
int pcu_b200_apss_project_f32(pcu_b200_workspace* ws, const float* p, const float* n, int64_t np, const float* q, int64_t nq, double r,
                              float* out_x, float* out_n, float* out_kh, void* stream);
int pcu_b200_apss_project_f64(pcu_b200_workspace* ws, const double* p, const double* n, int64_t np, const double* q, int64_t nq, double r,
                              double* out_x, double* out_n, double* out_kh, void* stream);
int pcu_b200_signed_distance_to_mesh_f32(pcu_b200_workspace* ws, const float* p, int64_t np, const float* v, int64_t nv, const void* f,
                                         int64_t nf, int f_kind, float lower_bound, float upper_bound, float* out_s, int32_t* out_fidx,
                                         float* out_bc, uint64_t* out_bad, void* stream);
int pcu_b200_signed_distance_to_mesh_f64(pcu_b200_workspace* ws, const double* p, int64_t np, const double* v, int64_t nv, const void* f,
                                         int64_t nf, int f_kind, float lower_bound, float upper_bound, double* out_s, int32_t* out_fidx,
                                         double* out_bc, uint64_t* out_bad, void* stream);

/* ---- rays against a mesh -----------------------------------------------------------------------------------------
 * Replace ray_mesh_intersection and RayMeshIntersector (src/ray_mesh_intersection.cpp, one Embree ray at a time).  For
 * each ray i (n rays, n >= 0) with origin o[i * o_stride .. + 3] (o_stride 0: one origin for every ray, 3: one per ray)
 * and direction d[3 i .. 3 i + 3]: out_fidx[i], out_bc[i, 0:3] and out_t[i] of the face that minimises (t, face index)
 * lexicographically over the faces hit with near < t <= far, by the watertight test of Woop, Benthin and Wald (JCGT
 * 2013) in fp32 on the fp32-rounded corners, origin and direction, both sides of a face counting (DESIGN.md §3,
 * csrc/raycast.cuh).  bc = (fl((1 - b1) - b2 in fp64), b1, b2), t in units of |d|.  A ray that hits nothing, and a
 * ray whose origin or direction is zero or not finite, gets out_fidx = -1, out_t = +inf and out_bc = 0.
 *   ray_mesh_intersection: builds the tree of the closest-point query for the call; out_fidx has f's width (4 bytes for
 *     I32 / U32, 8 for I64 / U64).  Faces with a corner outside [0, nv) are left out and counted in *out_bad (device
 *     uint64); when it is not zero the outputs are unspecified.
 *   mesh_prepare: builds that tree once into a private device block (*out_mesh) and counts the bad faces in *out_bad as
 *     above (a handle whose count is not zero should be destroyed).  pcu_b200_mesh_destroy synchronises the device;
 *     pcu_b200_mesh_size is the face count.
 *   ray_mesh_intersection_prepared: rays against a prepared mesh of either precision (the suffix is the rays'); out_fidx
 *     is int32.  Results equal ray_mesh_intersection's on the same mesh.
 * Every array pointer is a DEVICE pointer and the calls are stream-ordered. */
typedef struct pcu_b200_mesh pcu_b200_mesh;
int pcu_b200_ray_mesh_intersection_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                       const float* o, int o_stride, const float* d, int64_t n, float near, float far, void* out_fidx,
                                       float* out_bc, float* out_t, uint64_t* out_bad, void* stream);
int pcu_b200_ray_mesh_intersection_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                       const double* o, int o_stride, const double* d, int64_t n, float near, float far, void* out_fidx,
                                       double* out_bc, double* out_t, uint64_t* out_bad, void* stream);
int pcu_b200_mesh_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                              pcu_b200_mesh** out_mesh, uint64_t* out_bad, void* stream);
int pcu_b200_mesh_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                              pcu_b200_mesh** out_mesh, uint64_t* out_bad, void* stream);
int pcu_b200_mesh_destroy(pcu_b200_mesh* mesh);
int64_t pcu_b200_mesh_size(const pcu_b200_mesh* mesh);
int pcu_b200_ray_mesh_intersection_prepared_f32(pcu_b200_workspace* ws, const pcu_b200_mesh* mesh, const float* o, int o_stride,
                                                const float* d, int64_t n, float near, float far, int32_t* out_fidx, float* out_bc,
                                                float* out_t, void* stream);
int pcu_b200_ray_mesh_intersection_prepared_f64(pcu_b200_workspace* ws, const pcu_b200_mesh* mesh, const double* o, int o_stride,
                                                const double* d, int64_t n, float near, float far, int32_t* out_fidx, double* out_bc,
                                                double* out_t, void* stream);

/* ---- rays against surfels -----------------------------------------------------------------------------------------
 * Replace ray_surfel_intersection, RaySurfelIntersector and pointcloud_surfel_geometry (src/ray_point_cloud_intersection.cpp,
 * "circle" geometry).  Point i (np points, 0 <= np < 2^31 - 1) is a disk of radius r[i] around p[i] facing n[i], drawn
 * as a fan of s = subdivs triangles (4 <= s <= 2^24): rim vertex j at angle theta_j = 2 pi j / s in the reference's
 * basis, computed in fp32 op by op, with fl32(cos theta_j) and fl32(sin theta_j) from the C library (DESIGN.md §3).
 * For each ray (as for rays against a mesh): out_pid[i] (int32) and out_t[i] of the point that minimises (t, point id)
 * over the fan triangles hit with near < t <= far, by the same fp32 watertight test.  Misses, invalid rays, np = 0 and
 * points whose fan has a non-finite coordinate (a zero normal, non-finite p or r) give pid = -1, t = +inf.
 *   ray_surfel_intersection: builds the surfel tree for the call.
 *   surfel_prepare: builds it once into a private device block (*out_surfels, a pcu_b200_mesh handle freed by
 *     pcu_b200_mesh_destroy; pcu_b200_mesh_size is np).
 *   ray_surfel_intersection_prepared: rays of either precision (the suffix is the rays') against prepared surfels of
 *     either precision.  Results equal ray_surfel_intersection's on the same input.
 *   pointcloud_surfel_geometry: the fans as a mesh: out_v ((s + 1) np rows, rim j of point i at i (s + 1) + j, the
 *     centre at i (s + 1) + s) in p's precision, and out_f (s np rows (centre, rim j, rim (j + 1) mod s)) int32;
 *     (s + 1) np must be below 2^31 - 1.
 *   pointcloud_sphere_geometry ("sphere" geometry, make_sphere_geometry): a UV sphere of radius r[i] around p[i] with
 *     num_stacks >= 1 latitudinal and num_slices >= 1 longitudinal divisions.  V = (stacks + 1)(slices + 1) vertices per
 *     point in p's precision, vertex (a, b) at row i V + a (slices + 1) + b, and F = 2 (stacks - 1) slices int32 faces per
 *     point at rows i F .., in the reference's loop order; poles and seam duplicated.  Coordinates are computed in fp64
 *     without contraction from cos and sin of the reference's angles (C library, on the host) and rounded once to p's
 *     type (DESIGN.md §3).  V np must be below 2^31 - 1; np = 0 does nothing.
 * Every array pointer is a DEVICE pointer and the calls are stream-ordered. */
int pcu_b200_ray_surfel_intersection_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                         const float* o, int o_stride, const float* d, int64_t nr, float near, float far, int32_t* out_pid,
                                         float* out_t, void* stream);
int pcu_b200_ray_surfel_intersection_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np, int subdivs,
                                         const double* o, int o_stride, const double* d, int64_t nr, float near, float far, int32_t* out_pid,
                                         double* out_t, void* stream);
int pcu_b200_surfel_prepare_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                pcu_b200_mesh** out_surfels, void* stream);
int pcu_b200_surfel_prepare_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np, int subdivs,
                                pcu_b200_mesh** out_surfels, void* stream);
int pcu_b200_ray_surfel_intersection_prepared_f32(pcu_b200_workspace* ws, const pcu_b200_mesh* surfels, const float* o, int o_stride,
                                                  const float* d, int64_t nr, float near, float far, int32_t* out_pid, float* out_t,
                                                  void* stream);
int pcu_b200_ray_surfel_intersection_prepared_f64(pcu_b200_workspace* ws, const pcu_b200_mesh* surfels, const double* o, int o_stride,
                                                  const double* d, int64_t nr, float near, float far, int32_t* out_pid, double* out_t,
                                                  void* stream);
int pcu_b200_pointcloud_surfel_geometry_f32(pcu_b200_workspace* ws, const float* p, const float* n, const float* r, int64_t np, int subdivs,
                                            float* out_v, int32_t* out_f, void* stream);
int pcu_b200_pointcloud_surfel_geometry_f64(pcu_b200_workspace* ws, const double* p, const double* n, const double* r, int64_t np,
                                            int subdivs, double* out_v, int32_t* out_f, void* stream);
int pcu_b200_pointcloud_sphere_geometry_f32(pcu_b200_workspace* ws, const float* p, const float* r, int64_t np, int num_stacks,
                                            int num_slices, float* out_v, int32_t* out_f, void* stream);
int pcu_b200_pointcloud_sphere_geometry_f64(pcu_b200_workspace* ws, const double* p, const double* r, int64_t np, int num_stacks,
                                            int num_slices, double* out_v, int32_t* out_f, void* stream);

/* ---- marching cubes on a sparse voxel grid and the grid's boundary ---------------------------------------------------
 * Replace marching_cubes_sparse_voxel_grid (src/marching_cubes.cpp:35-85) and sparse_voxel_grid_boundary
 * (src/sparse_voxel_grid.cpp:463-522).  The marching-cubes result is defined in DESIGN.md §3: one vertex per distinct
 * unordered pair of corner indices on a crossing edge, numbered by first appearance (cube by cube, edge by edge), each
 * interpolated in the coordinates' precision T from that first edge; faces cube by cube in the generated case table's
 * order.  The suffix is T; scalars are float or double (scalars_f64), cube_idx is (m, 8) of kind idx_kind, 16-byte
 * aligned; 1 <= n < 2^31 - 1, m >= 1.
 *   marching_cubes_prepare: classifies the cubes, synchronises `stream` to read the crossing-edge and face counts, then
 *     numbers the vertices and synchronises again to read their count.  *out_counts = {#v, #f} (host int64).  A cube
 *     corner outside [0, n), 2^32 or more crossing edges, or more vertices than idx_kind can index fail with
 *     PCU_B200_INVALID_ARGUMENT.  *out_mc (a handle; scalars, coords and cube_idx must stay alive until emit) is freed
 *     by marching_cubes_destroy, stream-ordered on the stream it was prepared on.
 *   marching_cubes_emit: writes out_v (#v, 3) in T and out_f (#f, 3) of idx_kind's width; stream-ordered.
 *   sparse_voxel_grid_boundary: grid (n, 3) int32 (idx_kind I32) or int64 (I64), n >= 1; out_idx (capacity n, int64)
 *     receives the boundary voxels' rows in ascending order, out_counts[0] (device int64) their number and
 *     out_counts[1] the rows with a coordinate outside [INT32_MIN + 1, INT32_MAX - 1] (then the output is unspecified).
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_marching_cubes pcu_b200_marching_cubes;
int pcu_b200_marching_cubes_prepare_f32(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const float* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream);
int pcu_b200_marching_cubes_prepare_f64(pcu_b200_workspace* ws, const void* scalars, int scalars_f64, const double* coords, int64_t n,
                                        const void* cube_idx, int64_t m, int idx_kind, double isovalue, pcu_b200_marching_cubes** out_mc,
                                        int64_t out_counts[2], void* stream);
int pcu_b200_marching_cubes_emit(pcu_b200_workspace* ws, const pcu_b200_marching_cubes* mc, void* out_v, void* out_f, void* stream);
int pcu_b200_marching_cubes_destroy(pcu_b200_marching_cubes* mc);
int pcu_b200_sparse_voxel_grid_boundary(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, int64_t* out_idx,
                                        int64_t* out_counts, void* stream);

/* ---- sparse voxel grids: from points, dilation, erosion, hex mesh; voxel cube meshes --------------------------------
 * Replace sparse_voxel_grid_from_pointcloud, dilate_sparse_voxel_grid, erode_sparse_voxel_grid and
 * sparse_voxel_grid_to_hex_mesh (the reference's src/sparse_voxel_grid.cpp:78-460) and voxel_grid_geometry
 * (src/mesh_for_voxels.cpp).  Results, and the three divergences from the reference's bindings (all 26 neighbours,
 * per-axis half voxel, shape check), are defined in DESIGN.md §3.  Voxels are identified by 64-bit Morton codes of
 * their int32 coordinates; grids are int32 (idx_kind I32) or int64 (I64) rows, n >= 1; a coordinate outside
 * [INT32_MIN + 1, INT32_MAX - 1] (and any unsigned grid) fails with PCU_B200_INVALID_ARGUMENT and the reference's
 * message "Invalid vertex leads to an overflow integer. ...".
 *   sparse_grid_from_points: points (n, 3) in the suffix's type, n < 2^31 - 1, voxel_size and origin host arrays of 3;
 *     voxel index round((p - o) / s) per axis in fp64.  Synchronises `stream` once; *out_counts = {distinct voxels u,
 *     n} (host int64).
 *   sparse_grid_dilate_prepare: one dilation round of an (n, 3) grid, n <= 82 595 524 (26 n flags are ranked in 32
 *     bits).  Synchronises `stream` once; *out_counts = {rows of the result, new rows}.  grid must stay alive until emit.
 *   sparse_grid_hex_prepare: the hex mesh of an (n, 3) grid, n < 2^28; vertices in double (vertices_f64) or float.
 *     Synchronises `stream` once; *out_counts = {#v, 8 n}.
 *   sparse_grid_emit: from points: out_rows (u, 3) int32 grid, out_index (n) int64 point_to_vox; dilation: out_rows
 *     (n + new, 3) of the grid's kind (the input rows, then the new ones), out_index unused; hex mesh: out_rows (#v, 3)
 *     vertices, out_index (n, 8) int64 cubes.  Stream-ordered.
 *   sparse_grid_destroy: frees a prepared handle, stream-ordered on the stream it was prepared on.
 *   sparse_grid_erode: one erosion round of an (n, 3) grid, n < 2^31 - 1: out_grid (capacity n rows, the grid's kind)
 *     receives the kept rows in order, out_counts[0] (device int64) their number and out_counts[1] the rows out of
 *     range (then the output is unspecified).  Stream-ordered, no synchronisation.
 *   voxel_grid_geometry: ijk (n, 3) of any index kind, 1 <= n <= 2^28, voxel_size > 0 (NaN passes, as in the
 *     reference); out_v (8 n, 3) float and out_f (12 n, 3) int32.  Stream-ordered, no synchronisation.
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_sparse_grid pcu_b200_sparse_grid;
int pcu_b200_sparse_grid_from_points_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream);
int pcu_b200_sparse_grid_from_points_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double voxel_size[3],
                                         const double origin[3], pcu_b200_sparse_grid** out_grid, int64_t out_counts[2], void* stream);
int pcu_b200_sparse_grid_dilate_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, pcu_b200_sparse_grid** out_grid,
                                        int64_t out_counts[2], void* stream);
int pcu_b200_sparse_grid_hex_prepare(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, const double voxel_size[3],
                                     const double origin[3], int vertices_f64, pcu_b200_sparse_grid** out_grid, int64_t out_counts[2],
                                     void* stream);
int pcu_b200_sparse_grid_emit(pcu_b200_workspace* ws, const pcu_b200_sparse_grid* sg, void* out_rows, int64_t* out_index, void* stream);
int pcu_b200_sparse_grid_destroy(pcu_b200_sparse_grid* sg);
int pcu_b200_sparse_grid_erode(pcu_b200_workspace* ws, const void* grid, int64_t n, int idx_kind, void* out_grid, int64_t* out_counts,
                               void* stream);
int pcu_b200_voxel_grid_geometry(pcu_b200_workspace* ws, const void* ijk, int64_t n, int idx_kind, const double voxel_size[3],
                                 const double voxel_origin[3], double gap_fraction, float* out_v, int32_t* out_f, void* stream);

/* ---- triangle-mesh voxelization and 3-D flood fill -----------------------------------------------------------------
 * Replace voxelize_triangle_mesh and flood_fill_3d (the reference's point_cloud_utils/_voxels.py,
 * src/voxelize_triangle_mesh.cpp, src/flood_fill_3d.cpp).  Results defined in DESIGN.md §3.
 *   voxelize_prepare: v (nv, 3) in the suffix's type, f (nf, 3) of kind f_kind, voxel_size > 0 and voxel_origin (host
 *     arrays of 3).  Voxel (i, j, k) is the box centred at origin + (i, j, k) * size with half-size size / 2; a face
 *     keeps the voxels of its index bounds [floor((min - o) / s), ceil((max - o) / s)] (x included over the whole
 *     range) that the reference's triBoxOverlap accepts, in fp64 operation for operation.  Synchronises `stream`
 *     twice: once to read the accepted count (which sizes the code buffer), once to read the number of distinct
 *     voxels.  *out_counts = {distinct voxels n, accepted (face, voxel) pairs} (host int64).  A corner outside [0, nv), a non-finite vertex, index bounds outside [INT32_MIN, INT32_MAX - 1], a
 *     candidate total that overflows int64, 2^31 - 1 or more accepted (face, voxel) pairs, or none at all fail with
 *     PCU_B200_INVALID_ARGUMENT.  *out_vx (v and f need not outlive prepare) is freed by voxelize_destroy,
 *     stream-ordered on the stream it was prepared on.
 *   voxelize_emit: writes out_ijk (n, 3) int32: morton_decode of the distinct 64-bit Morton codes of the kept
 *     voxels, in ascending code order (coordinates alias beyond 21 bits as in the reference's morton_encode).
 *   flood_fill_3d: grid (w, h, d) C-ordered of grid_kind, w h d < 2^31, seed inside the grid.  out (same shape and
 *     type) = grid with fill_value (converted as the reference's x86 build converts a double: integers truncate, NaN
 *     or out of range give INT_MIN of the type) written over the seed's component among the voxels equal to the
 *     seed's value, linear index o adjacent to o +- 1, o +- d, o +- h d inside [0, w h d) (so steps past the y and z
 *     faces wrap, as in the reference).  fill == seed value: out is a copy.  Stream-ordered, no synchronisation.
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_voxelize pcu_b200_voxelize;
enum pcu_b200_grid_kind { PCU_B200_GRID_I32 = 0, PCU_B200_GRID_I64 = 1, PCU_B200_GRID_F32 = 2, PCU_B200_GRID_F64 = 3 };
int pcu_b200_voxelize_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream);
int pcu_b200_voxelize_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                  const double voxel_size[3], const double voxel_origin[3], pcu_b200_voxelize** out_vx,
                                  int64_t out_counts[2], void* stream);
int pcu_b200_voxelize_emit(pcu_b200_workspace* ws, const pcu_b200_voxelize* vx, int32_t* out_ijk, void* stream);
int pcu_b200_voxelize_destroy(pcu_b200_voxelize* vx);
int pcu_b200_flood_fill_3d(pcu_b200_workspace* ws, const void* grid, int grid_kind, int64_t w, int64_t h, int64_t d, int64_t seed_x,
                           int64_t seed_y, int64_t seed_z, double fill_value, void* out, void* stream);

/* ---- watertight manifold remeshing ---------------------------------------------------------------------------------
 * Replaces make_mesh_watertight (the reference's src/manifold.cpp).  Result defined in DESIGN.md §3: the outer
 * surface of the mesh's voxel occupancy on a cubic grid of 2^d voxels per side (d in [3, 10], the smallest whose
 * occupied count reaches `resolution`), extracted by marching cubes and projected onto the input in 10 rounds.
 *   make_mesh_watertight_prepare: v (nv, 3) in the suffix's type, f (nf, 3) of kind f_kind, 1 <= nv, nf < 2^31 - 1.
 *     Synchronises `stream` once for v's bounds, once or twice per depth tried, once for the surface's counts and once
 *     per flip pass of each projection round.  *out_counts = {#vw, #fw, d} (host int64).  A non-finite vertex, a
 *     corner outside [0, nv), a mesh whose vertices all coincide, or more output vertices than f_kind can index fail
 *     with PCU_B200_INVALID_ARGUMENT.  Dense scratch of 5 bytes per voxel (5 GiB at d = 10) lives for the call only.
 *     *out_wt (v and f need not outlive prepare) is freed by make_mesh_watertight_destroy, stream-ordered on the
 *     stream it was prepared on.
 *   make_mesh_watertight_emit: writes out_v (#vw, 3) in the suffix's type and out_f (#fw, 3) in f's width.
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_watertight pcu_b200_watertight;
int pcu_b200_make_mesh_watertight_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream);
int pcu_b200_make_mesh_watertight_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                              double resolution, pcu_b200_watertight** out_wt, int64_t out_counts[3], void* stream);
int pcu_b200_make_mesh_watertight_emit(pcu_b200_workspace* ws, const pcu_b200_watertight* wt, void* out_v, void* out_f, void* stream);
int pcu_b200_make_mesh_watertight_destroy(pcu_b200_watertight* wt);

/* ---- shortest-edge decimation -----------------------------------------------------------------------------------------
 * Replaces decimate_triangle_mesh (the reference's src/mesh_decimate.cpp, libigl's decimate).  Result defined in
 * DESIGN.md §3: rounds of independent shortest-edge collapses under the link condition, midpoint placement, until at
 * most max_faces faces remain (max_faces or max_faces - 1 unless the mesh stalls) or no edge can collapse.
 *   decimate_triangle_mesh_prepare: v (nv, 3) in the suffix's type, f (nf, 3) of kind f_kind, 1 <= nv < 2^31 - 1,
 *     1 <= nf <= (2^31 - 2) / 6, 1 <= max_faces <= nf.  Synchronises `stream` once for the input check, once for the
 *     acceptance test, once per round and once for the output counts.  *out_counts = {#v_out, #f_out, rounds} (host
 *     int64).  A corner outside [0, nv), a non-finite vertex, or a mesh the definition rejects (a repeated corner, an
 *     edge in three or more faces, a vertex with other than zero or two boundary edges) fail with
 *     PCU_B200_INVALID_ARGUMENT.  *out_dc (v and f need not outlive prepare) is freed by
 *     decimate_triangle_mesh_destroy, stream-ordered on the stream it was prepared on.
 *   decimate_triangle_mesh_emit: writes out_v (#v_out, 3) in the suffix's type, out_f (#f_out, 3), out_v_corr (#v_out)
 *     and out_f_corr (#f_out) in f's width.
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_decimate pcu_b200_decimate;
int pcu_b200_decimate_triangle_mesh_prepare_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                int64_t max_faces, pcu_b200_decimate** out_dc, int64_t out_counts[3], void* stream);
int pcu_b200_decimate_triangle_mesh_prepare_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                int64_t max_faces, pcu_b200_decimate** out_dc, int64_t out_counts[3], void* stream);
int pcu_b200_decimate_triangle_mesh_emit(pcu_b200_workspace* ws, const pcu_b200_decimate* dc, void* out_v, void* out_f, void* out_v_corr,
                                         void* out_f_corr, void* stream);
int pcu_b200_decimate_triangle_mesh_destroy(pcu_b200_decimate* dc);

/* ---- mesh topology: connected components and vertex removal ----------------------------------------------------------
 * Replace connected_components, remove_mesh_vertices and remove_unreferenced_mesh_vertices (the reference's
 * src/connected_components.cpp, src/remove_mesh_vertices.cpp, src/remove_unreferenced_mesh_vertices.cpp).  Results
 * defined in DESIGN.md §3.  Index arrays are of kind f_kind (pcu_b200_index_kind); outputs of "f's width" are int32
 * for the 32-bit kinds and int64 for the 64-bit ones (unsigned kinds share the bits).
 *   connected_components_prepare: f (nf, f_cols), 1 <= nf < 2^31 - 1, f_cols >= 1.  The graph's vertices are [0, n),
 *     n = max(f) + 1; corner j of every row is joined to corner j + 1.  Component j is the j-th in ascending order of
 *     its smallest vertex.  Synchronises `stream` twice: once to read max(f) (which sizes the buffers), once to read the
 *     component count k.  *out_counts = {n, k} (host int64).  An entry of f that is negative or above 2^31 - 2 fails with
 *     PCU_B200_INVALID_ARGUMENT.  *out_cc (f need not outlive prepare) is freed by connected_components_destroy,
 *     stream-ordered on the stream it was prepared on.
 *   connected_components_emit: writes out_cv (n), out_nv (k), out_cf (nf) and out_nf (k) in f's width: the component of
 *     every vertex, the vertices of every component, the component of every face (that of its first corner) and the
 *     faces of every component.
 *   remove_mesh_vertices: v (nv, 3) in the suffix's type, f (nf, 3) int32 or int64, mask (nv) bytes, nonzero = keep.
 *     out_v (capacity nv rows) receives the kept vertices in input order, out_f (capacity nf rows, f's width) the faces
 *     whose three corners are kept, re-indexed, in input order.  Synchronises `stream` once; *out_counts = {kept
 *     vertices, kept faces} (host int64).
 *   remove_unreferenced_mesh_vertices: v (nv, 3), f (nf, 3) of any index kind.  out_v (capacity nv rows) = v[J];
 *     out_corr_v (capacity nv) = J, the vertices some corner names, ascending; out_corr_f (nv) = I, I[J[j]] = j and -1
 *     (all ones for the unsigned kinds) elsewhere; out_f (nf, 3) = I[f]; all in f's width.  Synchronises `stream`
 *     once; *out_count = #J (host int64).
 *   For both removals 1 <= nv, nf < 2^31 - 1, and a corner outside [0, nv) fails with PCU_B200_INVALID_ARGUMENT.
 *   orient_mesh_faces (the reference's src/orient_mesh_faces.cpp, libigl's bfs_orient): f (nf, 3) of any index kind,
 *     1 <= nf <= 2^30 - 1.  Ids are only compared for equality, so every value is legal.  out_f (nf, 3) receives the
 *     rows, consistently oriented within each patch (faces joined by edges that no third face has), and
 *     out_components (nf) each face's patch, patch j being the j-th in ascending order of its smallest face; both in
 *     f's width.  Never synchronises `stream`.
 *   adjacency_list_prepare (the reference's src/adjacency_list.cpp, libigl's adjacency_list): f (nf, 3) of any index
 *     kind, 1 <= nf <= 357913941 (6 nf directed edges fit int32 ranks).  List i of the n = max(f) + 1 lists holds, in
 *     ascending order and once each, every vertex that shares a face with i, and i itself when some face names i at
 *     two or more corners; an index no face names has an empty list.  Synchronises `stream` twice: once to read max(f),
 *     once to read the entry count nnz.  *out_counts = {n, nnz} (host int64).  An entry of f that is negative or above
 *     2^31 - 2 fails with PCU_B200_INVALID_ARGUMENT.  *out_adj (f need not outlive prepare) is freed by
 *     adjacency_list_destroy, stream-ordered on the stream it was prepared on.
 *   adjacency_list_emit: writes out_offsets (n + 1) and out_neighbors (nnz) in f's width: list i is
 *     out_neighbors[out_offsets[i] .. out_offsets[i + 1]).
 * Every array pointer is a DEVICE pointer. */
typedef struct pcu_b200_components pcu_b200_components;
int pcu_b200_connected_components_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_cols, int f_kind,
                                           pcu_b200_components** out_cc, int64_t out_counts[2], void* stream);
int pcu_b200_connected_components_emit(pcu_b200_workspace* ws, const pcu_b200_components* cc, void* out_cv, void* out_nv, void* out_cf,
                                        void* out_nf, void* stream);
int pcu_b200_connected_components_destroy(pcu_b200_components* cc);
int pcu_b200_remove_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, float* out_v, void* out_f, int64_t out_counts[2], void* stream);
int pcu_b200_remove_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                      const uint8_t* mask, double* out_v, void* out_f, int64_t out_counts[2], void* stream);
int pcu_b200_remove_unreferenced_mesh_vertices_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   float* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream);
int pcu_b200_remove_unreferenced_mesh_vertices_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind,
                                                   double* out_v, void* out_f, void* out_corr_v, void* out_corr_f, int64_t* out_count,
                                                   void* stream);
int pcu_b200_orient_mesh_faces(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, void* out_f, void* out_components,
                               void* stream);
typedef struct pcu_b200_adjacency pcu_b200_adjacency;
int pcu_b200_adjacency_list_prepare(pcu_b200_workspace* ws, const void* f, int64_t nf, int f_kind, pcu_b200_adjacency** out_adj,
                                    int64_t out_counts[2], void* stream);
int pcu_b200_adjacency_list_emit(pcu_b200_workspace* ws, const pcu_b200_adjacency* adj, void* out_offsets, void* out_neighbors, void* stream);
int pcu_b200_adjacency_list_destroy(pcu_b200_adjacency* adj);

/* ---- mesh normals, face areas, curvatures and Laplacian smoothing ------------------------------------------------
 * Replace mesh_face_areas, estimate_mesh_face_normals, estimate_mesh_vertex_normals, mesh_principal_curvatures and
 * laplacian_smooth_mesh (the reference's src/face_areas.cpp, src/mesh_normals.cpp, src/curvature.cpp, src/smooth.cpp).
 * Results defined in DESIGN.md §3.  v (nv, 3) in the suffix's type, f (nf, 3) of kind f_kind (pcu_b200_index_kind); 1 <= nv <= 2^31 - 2, 1 <= nf <= 357913941.
 * A face with a corner outside [0, nv) fails with PCU_B200_INVALID_ARGUMENT (the outputs are written nonetheless).
 *   mesh_face_areas: out_areas (nf), the reference's formula in v's precision.  Synchronises `stream` once.
 *   mesh_face_normals: out_n (nf, 3), unit normals from fp64, 0 for a face of zero area.  Synchronises once.
 *   mesh_vertex_normals: out_n (nv, 3); weighting 0 uniform, 1 area, 2 angle.  Synchronises once.
 *   mesh_principal_curvatures: out_k1, out_k2 (nv) and out_d1, out_d2 (nv, 3), k1 >= k2, NaN curvatures and zero
 *     directions where undetermined.  r <= 0: the one-ring tensor estimate; r > 0: a quadric fit over the ball of
 *     radius r around each vertex.  A non-finite r fails with PCU_B200_INVALID_ARGUMENT.  Synchronises once.
 *   laplacian_smooth_mesh: out_v (nv, 3); num_iters >= 0 (0 copies v and does not synchronise).  out_cg_iters and
 *     out_residual (host, num_iters entries) receive every step's conjugate-gradient iterations and its largest
 *     |r| / |b| at exit (<= 1e-12 when it converged; a step stops after max_cg_iters iterations).  Synchronises once
 *     after assembling the Laplacian, once per 16 CG iterations of every step and, with use_cotan_weights, once at the
 *     end.  Non-finite coordinates and (use_cotan_weights) a total area of 0 fail with PCU_B200_INVALID_ARGUMENT.
 * Every array pointer is a DEVICE pointer unless stated otherwise. */
int pcu_b200_mesh_face_areas_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_areas,
                                 void* stream);
int pcu_b200_mesh_face_areas_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_areas,
                                 void* stream);
int pcu_b200_mesh_face_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, float* out_n,
                                   void* stream);
int pcu_b200_mesh_face_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double* out_n,
                                   void* stream);
int pcu_b200_mesh_vertex_normals_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     float* out_n, void* stream);
int pcu_b200_mesh_vertex_normals_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int weighting,
                                     double* out_n, void* stream);
int pcu_b200_mesh_principal_curvatures_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, double r,
                                           float* out_k1, float* out_k2, float* out_d1, float* out_d2, void* stream);
int pcu_b200_mesh_principal_curvatures_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, double r,
                                           double* out_k1, double* out_k2, double* out_d1, double* out_d2, void* stream);
int pcu_b200_laplacian_smooth_mesh_f32(pcu_b200_workspace* ws, const float* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, float* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream);
int pcu_b200_laplacian_smooth_mesh_f64(pcu_b200_workspace* ws, const double* v, int64_t nv, const void* f, int64_t nf, int f_kind, int num_iters,
                                       double step_size, int use_cotan_weights, int max_cg_iters, double* out_v, int32_t* out_cg_iters,
                                       double* out_residual, void* stream);

/* ---- voxel-grid down-sampling (SURVEY.md 8f, N2) --------------------------------------------
 * Replaces downsample_point_cloud_voxel_grid_internal (src/sample_point_cloud.cpp:336-367, :163-244): every point
 * goes to voxel int(floor((p - min_bound) / voxel_size)) per axis, computed in the cloud's precision exactly like the
 * reference; every voxel with at least min_points_per_voxel points yields one output row, the mean of its points and
 * of its rows of `attrib` ((n, attrib_cols) float or double, attrib_cols may be 0).  Exact: voxel assignment, the set
 * of output voxels, their point counts (out_counts, may be NULL).  Different by construction and documented: the
 * reference's row order is the iteration order of a std::unordered_map -- here rows follow the first point of each
 * voxel in the input; the reference sums in the cloud's precision point by point -- here in fp64, so means agree to
 * the rounding of its float sums.  Capacity of the outputs: n rows; out_rows: device int64.  DEVICE pointers. */
int pcu_b200_voxel_downsample_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, float* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream);
int pcu_b200_voxel_downsample_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const void* attrib, int attrib_cols,
                                  int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                  int min_points_per_voxel, double* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows,
                                  void* stream);

/* ---- dense pairwise distances and Sinkhorn (SURVEY.md 8f, N4) -------------------------------
 * Replace the numpy code of point_cloud_utils/_sinkhorn.py: pairwise_distances (:4-34), sinkhorn (:37-126) and the
 * cost (P * M).sum() of earth_movers_distance (:129-156).  DEVICE pointers, row-major dense arrays:
 *   pairwise: a (nb, n, d), b (nb, m, d) -> out (nb, n, m), out[k, i, j] = || a[k, i] - b[k, j] ||_p;
 *             norm_kind 0: p = 2 (np.linalg.norm default), 1: p = 1, 2: inf, 3: -inf, 4: p = 0 (count of non-zeros),
 *             5: general p (the double argument)
 *   sinkhorn: weights a (nb, n), b (nb, m), costs M (nb, n, m), eps, max_iters, stop_thresh -> plan out_P (nb, n, m);
 *             out_cost (nb) fp64 = sum_ij P * M per batch or NULL; out_iters: device int32 or NULL.  The log-domain
 *             iteration of the reference, its convergence test evaluated on the device (no host synchronisation).
 * Any number of rows and batches.  Floating point: pairwise norm kinds 0-4 equal numpy bit for bit (the same rounded
 * operations, sums in numpy's pairwise order, NaN propagated); kind 5 evaluates pow in fp64, within a few ulp of numpy.
 * Sinkhorn: element-wise expressions in the arrays' precision and the reference's order, the two reductions in fp64
 * -- agreement with numpy to rounding; the iteration count is the reference's, a NaN change never counting as
 * converged (tests/test_dense_metrics.py states the tolerances). */
int pcu_b200_pairwise_distances_f32(pcu_b200_workspace* ws, const float* a, const float* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, float* out, void* stream);
int pcu_b200_pairwise_distances_f64(pcu_b200_workspace* ws, const double* a, const double* b, int64_t nb, int64_t n, int64_t m, int d,
                                    int norm_kind, double p, double* out, void* stream);
int pcu_b200_sinkhorn_f32(pcu_b200_workspace* ws, const float* a, const float* b, const float* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, float* out_P, double* out_cost, int32_t* out_iters, void* stream);
int pcu_b200_sinkhorn_f64(pcu_b200_workspace* ws, const double* a, const double* b, const double* M, int64_t nb, int64_t n, int64_t m,
                          double eps, int max_iters, double stop_thresh, double* out_P, double* out_cost, int32_t* out_iters, void* stream);

/* ---- 64-bit 3-D Morton codes (SURVEY.md 8f, N3) --------------------------------------------
 * Replace MortonCode64 (src/common/morton_code.cpp:43-163) and the bindings morton_encode / morton_decode /
 * morton_add / morton_subtract / morton_knn (src/morton.cpp:185-239, :253-310, :26-103, :106-183, :324-414).
 * Integer work: bit-identical.  pts: (n, 3) int32 (or int64, truncated to int32 as the reference does);
 * coordinates in [-2^20, 2^20).  morton_knn: `codes` ascending; out_idx (m, k) = the k consecutive positions
 * around the lower bound of each query code (k <= n: the binding clamps like morton.cpp:351); sort_dist != 0
 * orders each row by squared distance to the query point -- an order the reference leaves undefined (its
 * comparator reads uninitialised variables, :381-398); the set of positions is the reference's.  DEVICE pointers. */
int pcu_b200_morton_encode_i32(pcu_b200_workspace* ws, const int32_t* pts, int64_t n, uint64_t* out_codes, void* stream);
int pcu_b200_morton_encode_i64(pcu_b200_workspace* ws, const int64_t* pts, int64_t n, uint64_t* out_codes, void* stream);
int pcu_b200_morton_decode(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, int32_t* out_pts, void* stream);
int pcu_b200_morton_add(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream);
int pcu_b200_morton_subtract(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out, void* stream);
int pcu_b200_morton_knn(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, const uint64_t* qcodes, int64_t m, int k,
                        int sort_dist, int64_t* out_idx, void* stream);

/* ---- HOST-pointer conveniences (H2D + kernels + D2H, synchronous) --------------------------
 * The calls the numpy-facing binding makes; these are what `e2e` in bench.py times.              */
int pcu_b200_knn_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset, int64_t m,
                          int k, int squared, float* out_dist, int64_t* out_idx, int64_t* out_n_tied);
int pcu_b200_knn_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset, int64_t m,
                          int k, int squared, double* out_dist, int64_t* out_idx, int64_t* out_n_tied);
int pcu_b200_nn_stats_host_f32(pcu_b200_workspace* ws, const float* query, int64_t n, const float* dataset,
                               int64_t m, pcu_b200_nn_stats* out_stats);
int pcu_b200_nn_stats_host_f64(pcu_b200_workspace* ws, const double* query, int64_t n, const double* dataset,
                               int64_t m, pcu_b200_nn_stats* out_stats);
int pcu_b200_chamfer_host_f32(pcu_b200_workspace* ws, const float* x, int64_t n, const float* y, int64_t m,
                              pcu_b200_nn_stats* out_stats, float* out_value);
int pcu_b200_chamfer_host_f64(pcu_b200_workspace* ws, const double* x, int64_t n, const double* y, int64_t m,
                              pcu_b200_nn_stats* out_stats, double* out_value);
int pcu_b200_batched_chamfer_host_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch,
                                      int64_t n, int64_t m, float* out_per_pair, double* out_sum);
int pcu_b200_morton_encode_host_i32(pcu_b200_workspace* ws, const int32_t* pts, int64_t n, uint64_t* out_codes);
int pcu_b200_morton_encode_host_i64(pcu_b200_workspace* ws, const int64_t* pts, int64_t n, uint64_t* out_codes);
int pcu_b200_morton_decode_host(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, int32_t* out_pts);
int pcu_b200_morton_add_host(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out);
int pcu_b200_morton_subtract_host(pcu_b200_workspace* ws, const uint64_t* a, const uint64_t* b, int64_t n, uint64_t* out);
int pcu_b200_morton_knn_host(pcu_b200_workspace* ws, const uint64_t* codes, int64_t n, const uint64_t* qcodes, int64_t m, int k,
                             int sort_dist, int64_t* out_idx);
int pcu_b200_normals_knn_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs, int k,
                                  double drop_angle_threshold, int64_t* out_idx, float* out_normals, int64_t* out_count);
int pcu_b200_normals_knn_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs, int k,
                                  double drop_angle_threshold, int64_t* out_idx, double* out_normals, int64_t* out_count);
/* voxel-grid down-sampling / duplicate removal on HOST arrays (outputs sized for the worst case as in the device
 * forms; out_rows / out_counts are HOST integers here) */
int pcu_b200_voxel_downsample_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const void* attrib, int attrib_cols,
                                       int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                       int min_points_per_voxel, float* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows);
int pcu_b200_voxel_downsample_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const void* attrib, int attrib_cols,
                                       int attrib_is_f64, const double voxel_size[3], const double min_bound[3], const double max_bound[3],
                                       int min_points_per_voxel, double* out_points, void* out_attrib, int32_t* out_counts, int64_t* out_rows);
int pcu_b200_deduplicate_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                                  int face_cols, int faces_are_i64, float* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                                  int64_t* out_counts);
int pcu_b200_deduplicate_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, double epsilon, const void* faces, int64_t n_faces,
                                  int face_cols, int faces_are_i64, double* out_points, int32_t* out_svi, int32_t* out_svj, void* out_faces,
                                  int64_t* out_counts);
int pcu_b200_normals_ball_host_f32(pcu_b200_workspace* ws, const float* points, int64_t n, const float* view_dirs,
                                   const pcu_b200_ball_options* options, int64_t* out_idx, float* out_normals, int64_t* out_count);
int pcu_b200_normals_ball_host_f64(pcu_b200_workspace* ws, const double* points, int64_t n, const double* view_dirs,
                                   const pcu_b200_ball_options* options, int64_t* out_idx, double* out_normals, int64_t* out_count);

/* Timeline of the last kd-tree build on the workspace's device (globaltimer, ns; synchronises the device):
 * [0] start, [1] set-up done, [2 + l] grid-wide level l done (l < 28), [30] grid-wide phase done, [31] last CTA done,
 * [32] grid-wide levels, [33] subtrees built by single CTAs. */
int pcu_b200_debug_kd_times(pcu_b200_workspace* ws, uint64_t* out40);

/* ---- diagnostics ----------------------------------------------------------------------------
 * Builds the kd-tree replica used by the tie replay for HOST points and copies it out, so tests can
 * compare it node for node with the reference's tree.  order: (m) slot -> point index (nanoflann's
 * vAcc); per node (capacity node_cap, at most 2 m - 1 are used): split dimension (-1 = leaf),
 * divlow, divhigh, slot range [first, last), children.  Returns the node count through out_nodes.  */
int pcu_b200_debug_kd_tree_f32(pcu_b200_workspace* ws, const float* points, int64_t m, int max_points_per_leaf,
                               int32_t* order, int64_t node_cap, int32_t* feat, float* div_lo, float* div_hi,
                               int32_t* first, int32_t* last, int32_t* kid0, int32_t* kid1, int64_t* out_nodes);
int pcu_b200_debug_kd_tree_f64(pcu_b200_workspace* ws, const double* points, int64_t m, int max_points_per_leaf,
                               int32_t* order, int64_t node_cap, int32_t* feat, double* div_lo, double* div_hi,
                               int32_t* first, int32_t* last, int32_t* kid0, int32_t* kid1, int64_t* out_nodes);
/* pcu_b200_batched_chamfer_f32 that also leaves every pair's two statistics records in out_stats (DEVICE, 2 * batch
 * records: [2p] = x_p -> y_p, [2p + 1] = y_p -> x_p), so tests can check each pair's sweeps query by query through
 * their sums.  out_per_pair (DEVICE, batch scalars) as for the batched call; runs the same kernels. */
int pcu_b200_debug_batched_chamfer_stats_f32(pcu_b200_workspace* ws, const float* x, const float* y, int64_t batch, int64_t n,
                                             int64_t m, pcu_b200_nn_stats* out_stats, float* out_per_pair, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PCU_B200_H */
