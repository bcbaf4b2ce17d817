/*
 * plslam_b200 -- C ABI of the H100-native ICP-odometry hot path of pyLiDAR-SLAM.
 *
 * Drop-in boundary (SURVEY.md section 8b): these are the entry points the Python
 * plug-in classes of pylidar_slam_b200 (mirrors of the reference's OdometryAlgorithm /
 * LocalMap / RigidAlignment / Filter interfaces) bind through ctypes.  Every function
 * cites the reference interface it replaces (paths relative to the reference root).
 *
 * Conventions
 *  - Every call returns an int status (PLS_OK == 0).  pls_last_error(ctx) gives text.
 *  - Data pointers may be HOST or DEVICE pointers; the library classifies each pointer
 *    with cudaPointerGetAttributes and stages host memory itself (pinned host memory is
 *    copied asynchronously).  Results are written back to wherever the out-pointer lives.
 *    A call returns after its results are visible to the caller.
 *  - Point clouds are row-major [N,3]; projection maps are planar [C,H,W] (the reference's
 *    layouts); poses are row-major 4x4; pose parameters are (tx,ty,tz,ex,ey,ez), Euler xyz,
 *    R = Rz(ez) Ry(ey) Rx(ex) (slam/common/rotation.py:144-150).
 *  - float means IEEE binary32, the hot path's arithmetic type (icp_odometry.py:353-354).
 *  - Not re-entrant per context: one host thread drives a context (as one Python thread
 *    drives the reference algorithm).
 */
#ifndef PLSLAM_B200_H
#define PLSLAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PLS_API __attribute__((visibility("default")))
#else
#define PLS_API
#endif

typedef struct pls_context pls_context;

/* Status codes.  PLS_E_SINGULAR <-> RuntimeError("Invalid Jacobian in Gauss Newton
 * minimization") (slam/common/optimization.py:334-336); PLS_W_TINY_RESIDUAL <-> the
 * logging.warning + early return at optimization.py:323-327. */
enum {
    PLS_OK = 0,
    PLS_E_INVALID = 1,       /* bad argument / shape  (AssertionError in the reference) */
    PLS_E_CUDA = 2,          /* CUDA runtime failure */
    PLS_E_SINGULAR = 3,
    PLS_W_TINY_RESIDUAL = 4,
    PLS_E_STATE = 5,         /* call order (e.g. search before any map update) */
    PLS_E_COMM = 6           /* NCCL failure */
};

/* Robust weighting schemes, slam/common/optimization.py:211-226 (_LS_SCHEME). */
enum {
    PLS_SCHEME_DEFAULT = 0,
    PLS_SCHEME_LEAST_SQUARE = 1,
    PLS_SCHEME_HUBER = 2,
    PLS_SCHEME_EXP = 3,
    PLS_SCHEME_NEIGHBORHOOD = 4,
    PLS_SCHEME_GEMAN_MCCLURE = 5,
    PLS_SCHEME_SQUARE_GEMAN_MCCLURE = 6,
    PLS_SCHEME_CAUCHY = 7
};

/* LOCAL_MAP registry, slam/odometry/local_map.py:437-445. */
enum { PLS_MAP_KDTREE = 0, PLS_MAP_PROJECTIVE = 1 };

/* The three input layouts of ICPFrameToModel._read_input, icp_odometry.py:319-358. */
enum {
    PLS_INPUT_NDARRAY = 0,    /* np.ndarray [N,3]: queries = the raw points              */
    PLS_INPUT_TENSOR = 1,     /* torch [N,3]: queries = non-null pixels of its vertex map */
    PLS_INPUT_VERTEX_MAP = 2, /* torch [1,3,H,W]: used as the vertex map directly         */
    /* float64 clouds (e.g. the output of the Distortion filter): the reference projects them in float64 and
     * rounds the vertex map / the points to float32 afterwards (icp_odometry.py:331-352); `data` is double [n,3] */
    PLS_INPUT_NDARRAY_F64 = 3,
    PLS_INPUT_TENSOR_F64 = 4
};

/* Optional residency hints, OR-ed into the `layout` argument of pls_process_frame by a caller that knows where `data`
 * lives (no reference counterpart: the reference's tensors carry their device).  Without a hint the pointer is classified. */
enum { PLS_PTR_DEVICE = 0x100, PLS_PTR_HOST = 0x200 };

/* Configuration = SphericalProjector (projection.py:439-450) + ICPFrameToModelConfig
 * (icp_odometry.py:27-64) + local-map configs (local_map.py:83-88,244-251) +
 * GaussNewtonPointToPlaneConfig.gauss_newton_config (alignment.py:69-77). */
typedef struct pls_config {
    int32_t height, width;          /* projector image size */
    float up_fov_deg, down_fov_deg; /* projector vertical field of view */
    int32_t local_map_type;         /* PLS_MAP_* */
    int32_t local_map_size;         /* frames kept (20) */
    int32_t num_neighbors_normals;  /* kd map: k for normals (10), 3 <= k <= 255 */
    int32_t normals_kernel_size;    /* projective map: box size (5) */
    int32_t scheme;                 /* PLS_SCHEME_* */
    float sigma;                    /* scheme parameter */
    int32_t gn_max_iters;           /* Gauss-Newton iterations per alignment (1) */
    float gn_norm_stop;             /* GN stop on |dx| (1e-3) */
    int32_t max_num_alignments;     /* ICP iterations per frame */
    float threshold_delta_pose;     /* ICP stop on |delta| (1e-4) */
    float threshold_trans;          /* key-frame policy, metres (0.1) */
    float threshold_rot;            /* key-frame policy, degrees (0.3) */
    int32_t device;                 /* CUDA device ordinal */
    void* stream;                   /* cudaStream_t to run on, or NULL for a private stream */
} pls_config;

/* ---- lifetime ------------------------------------------------------------------- */
PLS_API int pls_config_default(pls_config* cfg);
/* PLS_E_INVALID (nothing created) for a config out of range, e.g. num_neighbors_normals outside [3, 255]. */
PLS_API int pls_create(const pls_config* cfg, pls_context** out);
PLS_API int pls_destroy(pls_context* ctx);
PLS_API const char* pls_last_error(pls_context* ctx);
PLS_API const char* pls_version(void);
/* cudaStreamSynchronize on the context's stream. */
PLS_API int pls_synchronize(pls_context* ctx);
/* Orders the work already enqueued on `other_stream` (a cudaStream_t, e.g. PyTorch's current stream that produced a
 * CUDA tensor about to be passed in) before everything this context enqueues afterwards; no host synchronisation. */
PLS_API int pls_wait_stream(pls_context* ctx, void* other_stream);

/* ---- a1: voxel-grid subsample ----------------------------------------------------
 * voxelise + voxel_hashing  (slam/common/pointcloud.py:13-23,40-79): int64 voxel
 * coordinates round_half_even(p / voxel) computed in float64 and the signed 64-bit hash
 * 73856093 x + 19349669 y + 83492791 z.  is_f64 selects float64 input points. */
PLS_API int pls_voxel_hash(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel,
                   int64_t* coords_out /* [n,3] or NULL */, int64_t* hashes_out /* [n] */);
/* voxelise with one voxel length per axis (pointcloud.py:55-79: voxel_x, voxel_y, voxel_z). */
PLS_API int pls_voxel_hash_xyz(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel_x, double voxel_y,
                       double voxel_z, int64_t* coords_out /* [n,3] or NULL */, int64_t* hashes_out /* [n] or NULL */);
/* grid_sample / GridSample.filter (pointcloud.py:170-195, preprocessing.py:213-226):
 * one point per distinct hash (its first occurrence), ordered by ascending hash.
 * out_xyz [n,3] (same dtype as the input), out_idx [n] int64; *out_count = S. */
PLS_API int pls_grid_sample(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel,
                    void* out_xyz, int64_t* out_idx, int64_t* out_count);

/* The same subsample for HOST callers without an extra copy (GridSample.filter hands numpy arrays to the next
 * filter): the gather kernel writes samples and indices straight into the context's pinned, device-mapped staging and
 * keeps a device-resident copy.  *out_xyz_host / *out_idx_host point into the staging (S rows, valid until the next
 * grid-sample call on this context); *out_xyz_dev (optional) is the device copy, which pls_process_frame accepts with
 * PLS_PTR_DEVICE -- the samples then never travel host -> device again.  One stream synchronisation per call.
 * Caller-owned staging: when *out_xyz_host and *out_idx_host are non-NULL ON ENTRY they name pinned, device-mapped
 * buffers from pls_pinned_alloc with room for n rows each, and the kernel writes there instead -- the caller (the
 * GridSample filter) then hands those very buffers on as arrays, no host-side copy at all. */
PLS_API int pls_grid_sample_staged(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel,
                           const void** out_xyz_host, const int64_t** out_idx_host, const void** out_xyz_dev,
                           int64_t* out_count);
/* Page-locked, device-mapped host memory for results a kernel writes straight into (see pls_grid_sample_staged). */
PLS_API int pls_pinned_alloc(int64_t num_bytes, void** out_ptr);
PLS_API int pls_pinned_free(void* ptr);
/* 64-bit fingerprint of a host buffer (256 evenly spread 8-byte words + its length): lets a caller check cheaply that
 * an array it handed out earlier still holds what the device-resident copy holds. */
PLS_API int pls_host_fingerprint(const void* host_ptr, int64_t num_bytes, uint64_t* out);

/* ---- a2/a3: spherical projection + closest-wins z-buffer --------------------------
 * SphericalProjector.project_pointcloud (projection.py:11-73,452-484): float pixel
 * coordinates, rows_cols_out [n,2] = (row, col). */
PLS_API int pls_project_pixels(pls_context* ctx, const float* xyz, int64_t n, int height, int width,
                       float up_fov_deg, float down_fov_deg, float* rows_cols_out);
/* Projector.build_projection_map (projection.py:331-418) for B stacked clouds:
 * xyz [B,n,3]; channels [B,n,C] or NULL (then C = 3 and the xyz are scattered);
 * out [B,C,H,W].  Per pixel the closest point (lowest index on exact ties) survives. */
PLS_API int pls_build_projection_map(pls_context* ctx, const float* xyz, const float* channels,
                             int batch, int64_t n, int num_channels, int height, int width,
                             float up_fov_deg, float down_fov_deg, float* out);
/* The same with the reference's `default_value` (projection.py:333,378-391): pixels no point lands on hold it. */
PLS_API int pls_build_projection_map_filled(pls_context* ctx, const float* xyz, const float* channels,
                                    int batch, int64_t n, int num_channels, int height, int width,
                                    float up_fov_deg, float down_fov_deg, float default_value, float* out);

/* ---- a4: box-filter normal map  (slam/common/geometry.py:240-295) ----------------- */
PLS_API int pls_normal_map(pls_context* ctx, const float* vertex_map /* [B,3,H,W] */, int batch,
                   int height, int width, int kernel_size, float* out /* [B,3,H,W] */);

/* ---- a6: projective association  (slam/common/geometry.py:397-439) ----------------
 * tgt [3,H,W]; ref [K,3,H,W]; fields [K,C,H,W] or NULL; out_nb [3,H,W]; out_fields [C,H,W]. */
PLS_API int pls_compute_neighbors(pls_context* ctx, const float* tgt, const float* ref, const float* fields,
                          int num_ref, int num_field_channels, int height, int width,
                          float* out_nb, float* out_fields);

/* ---- a16: pose algebra  (slam/common/pose.py:120-144,188-207) --------------------- */
PLS_API int pls_build_pose_matrix(pls_context* ctx, const float* params /* [B,6] */, int batch, float* out /* [B,4,4] */);
PLS_API int pls_from_pose_matrix(pls_context* ctx, const float* mats /* [B,4,4] */, int batch, float* out /* [B,6] */);

/* ---- a11-a15: point-to-plane Gauss-Newton alignment --------------------------------
 * GaussNewtonPointToPlaneAlignment.align (alignment.py:91-127) -> GaussNewton.compute
 * (optimization.py:296-344) with PointToPlaneCost closures (optimization.py:356-435).
 * ref/tgt/nrm are [n,3] (batch 1); is_f64 selects float64 data and arithmetic.
 * x0 [6] or NULL (zeros).  Outputs (same dtype as the inputs): out_dT [16], out_x [6],
 * out_loss [n] = (w r)^2 or NULL.  Returns PLS_E_SINGULAR / PLS_W_TINY_RESIDUAL like the
 * reference raises / warns. */
PLS_API int pls_align_p2plane(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t n,
                      int is_f64, int scheme, double sigma, int max_iters, double norm_stop,
                      const void* x0, void* out_dT, void* out_x, void* out_loss);

/* ---- a5/a7/a8/a9: local maps (LocalMap ABC, slam/odometry/local_map.py:31-79) -------
 * One local map lives in a context; its type is cfg.local_map_type. */
PLS_API int pls_map_init(pls_context* ctx); /* LocalMap.init */
/* KdTreeLocalMap.update (local_map.py:302-362): rel_pose [16]; new points [n,3] or NULL.
 * The map is moved by inverse(rel_pose), the new frame appended, the oldest frame dropped
 * beyond local_map_size, the search index rebuilt and the normal cache cleared. */
PLS_API int pls_kdmap_update_points(pls_context* ctx, const float* rel_pose, const float* points, int64_t n);
/* Same, inserting the pixels of a vertex map with |p| > 0.01 (local_map.py:320-324). */
PLS_API int pls_kdmap_update_vertex_map(pls_context* ctx, const float* rel_pose, const float* vertex_map,
                                int height, int width);
PLS_API int pls_kdmap_size(pls_context* ctx, int64_t* num_points);
/* Debug counters of the kd search (enabled by the environment variable PLS_KD_STATS=1), 16 u64. */
PLS_API int pls_kdmap_stats(pls_context* ctx, unsigned long long* out16);
PLS_API int pls_kdmap_points(pls_context* ctx, float* out /* [M,3], insertion order */);
/* KdTreeLocalMap.nearest_neighbor_search (local_map.py:372-422): exact 1-NN; normals from
 * the cfg.num_neighbors_normals nearest map neighbours of the matched map point (smallest-eigenvalue
 * direction), cached per map point until the next update.  out_idx [n] (int64, insertion order) or NULL. */
PLS_API int pls_kdmap_nn_search(pls_context* ctx, const float* queries, int64_t n,
                        float* out_neighbors, float* out_normals, int64_t* out_idx);
/* Test / debug aid: the correspondences of the last kd search of this context -- the last executed iteration of
 * pls_register_frame or pls_process_frame, or pls_kdmap_nn_search.  n = number of queries of that search (the valid
 * rows, in input order).  out_idx [n] insertion index of the match or -1; out_neighbors / out_normals [n,3] (normals
 * NaN after a search without normals); out_search_state [n,4] = the position the query stood at in its last full
 * search and the squared lower bound of its distance to every map point other than its match; out_sums [30] = the
 * accumulators of the last executed ICP iteration (21 JtJ upper, 6 Jtr, sum (w r)^2, sum r^2, count; NaN after
 * pls_kdmap_nn_search).  Every output nullable.  A pending map update is not flushed.  PLS_E_STATE if no kd search has
 * run, if the map was rebuilt since, or if the last ICP split its queries over several ranks. */
PLS_API int pls_kdmap_last_correspondences(pls_context* ctx, int64_t n, int64_t* out_idx, float* out_neighbors,
                                           float* out_normals, float* out_search_state, double* out_sums);
/* Test / debug aid: the exact (k+1)-NN lists of the normals search (0 <= k <= 255) for n arbitrary query rows [n,3]
 * on the current index, ordered by (float32 squared distance, sorted position).  out_idx [n,k+1] insertion index or -1
 * past the map's size; out_d2 [n,k+1] the float32 squared distance (NaN where out_idx is -1); out_pos [n,k+1] the
 * position in the Morton-sorted point array or -1 (nullable).  Touches neither the normal cache nor any ICP state. */
PLS_API int pls_kdmap_knn(pls_context* ctx, const float* queries, int64_t n, int k, int64_t* out_idx, float* out_d2,
                          int32_t* out_pos);
/* KdTreeLocalMap.set_map_pointcloud (local_map.py:289-299): the map becomes the cloud xyz [n,3] (float32, or float64
 * if is_f64, rounded to float32; host or device), in order, with a new search index and no cached normal.  The cloud is
 * held as no frame: a later update moves it and appends frames, and once more than local_map_size frames are held the
 * eviction drops as many rows from the FRONT of the map as the oldest frame had -- prior-map rows first, as the
 * reference's `_local_map[size_first_cloud:]` does.  A row with a NaN or infinite coordinate is refused
 * (PLS_E_INVALID, the map unchanged): the reference keeps such rows, but its search cannot handle them.  n == 0 leaves
 * an empty map. */
PLS_API int pls_kdmap_set_points(pls_context* ctx, const void* xyz, int is_f64, int64_t n);
/* The point counts of the frames the kd map holds, oldest first: *out_num frames (at most local_map_size), out_counts
 * [local_map_size] or NULL.  Rows of the map before the first counted frame are a cloud set by pls_kdmap_set_points. */
PLS_API int pls_kdmap_frames(pls_context* ctx, int64_t* out_counts, int* out_num);
/* Correlative pose search on the kd map ctx holds (no reference counterpart: finding a scan's pose on a prior map
 * without an initial estimate, at start-up or after odometry is lost).  Scores every pose of a dense (base, x, y) grid
 * by how many scan points land in occupied map cells, and returns the best local maxima for an ICP to refine.
 * scan [n,3] float32, host or device; rows with a non-finite coordinate are dropped, the valid rows are the multiset P.
 * Occupancy O: the cells (rint(x/c), rint(y/c), rint(z/c)) of the map's current points, c = cell -- pls_voxel_hash's
 * coordinates: float64 true division of the float32 value, round half to even.
 * bases [A,16] row-major float64 (host or device), base a = (R_a, t_a).  The base cell of p is rint(q / c) per axis,
 * with q_x = ((R00*x + R01*y) + R02*z) + t_x (likewise y, z), every product, sum and the division a separately rounded
 * float64 operation (no fused multiply-add).
 * score(a, i, j) = #{p in P : cell_a(p) + (i, j, 0) in O}, i in [-half_x, half_x], j in [-half_y, half_y].
 * out_scores [A, 2*half_y+1, 2*half_x+1] int32 (nullable): every score, at L = (a*(2*half_y+1) + j+half_y)*(2*half_x+1)
 * + i+half_x.  A pose's key is (score descending, L ascending).  A candidate has score > 0 and a key strictly better than
 * every existing neighbour in its 3x3x3 block (a+-1 without wrap-around, i+-1, j+-1, clipped to the volume).
 * *out_num = min(K, candidates); the candidates in key order: out_score [K] their scores, out_index [K] their L, out_T
 * [K,16] float64 bases[a] with t_x += i*c and t_y += j*c.  K == 0 only fills out_scores (half_x = half_y = 0 then
 * scores A arbitrary poses).  Outputs host or device.  A scan without a valid row gives all-zero scores, *out_num = 0.
 * Touches neither the map, its index, its normal cache nor any ICP state.  The map is the whole kd map on every rank of
 * a communicator.  PLS_E_INVALID, the context unchanged, for a projective map, a map that has had no update, a NULL scan
 * or bases, n <= 0, A <= 0, half_x or half_y < 0, K outside [0, PLS_POSE_SEARCH_MAX_K], a cell that is not finite and
 * > 0, a non-finite base, A*(2*half_x+1)*(2*half_y+1) >= 2^31, or an occupancy bit grid -- the range of the base cells
 * widened by half_x and half_y, x rows padded to whole 32-bit words -- of more than PLS_POSE_SEARCH_MAX_BITS bits (256 MiB; the
 * extent is in pls_last_error) or beyond +-2^40 cells. */
#define PLS_POSE_SEARCH_MAX_BITS (1ll << 31)
enum { PLS_POSE_SEARCH_MAX_K = 1024 };
PLS_API int pls_kdmap_pose_search(pls_context* ctx, const float* scan, int64_t n,
                                  const double* bases /* [A,16] row-major float64 */, int A,
                                  double cell, int half_x, int half_y, int K,
                                  int32_t* out_scores /* [A, 2*half_y+1, 2*half_x+1] or NULL */,
                                  double* out_T /* [K,16] */, int32_t* out_score /* [K] */,
                                  int64_t* out_index /* [K] */, int* out_num);
/* The candidates of pls_kdmap_pose_search found by branch and bound instead of scoring every pose: for windows up to
 * the whole map, where scoring every pose would take seconds.  For any call pls_kdmap_pose_search accepts with
 * out_scores == NULL and K >= 1, the same out_T, out_score, out_index and *out_num, bit for bit: the scores, the cell
 * rule, the key, the 3x3x3 candidate rule and T are the ones defined there.  L is int64.
 * Method (exact): B_0 is the occupancy bit grid over the reachable box (the base cells' box widened by the window)
 * clipped to the map's own cell box -- no map cell lies outside it, so a lookup outside reads 0 -- and B_k(X, Y, Z) is
 * the OR of B_(k-1) at (X, Y), (X + 2^(k-1), Y), (X, Y + 2^(k-1)), (X + 2^(k-1), Y + 2^(k-1)).  A node (a, I, J, k)
 * covers the shifts i + half_x in [I 2^k, (I+1) 2^k), j likewise; its bound #{p : B_k(cell_a(p) - (half_x, half_y, 0)
 * + (I 2^k, J 2^k)) set} is >= the score of each pose under it.  A pass with threshold tau expands every node whose
 * bound is >= tau down to level 0 and keeps E_tau, the poses scoring >= tau; a pose of E_tau is a candidate iff no
 * neighbour in E_tau has a better key.  If K candidates score >= tau, or tau == 1, the first K in key order are the
 * answer; otherwise tau drops to max(1, min(tau - 1, floor(3 tau / 4))).  The first tau is the largest root bound,
 * which no score exceeds.  Roots are at the least level kmax with at most 16 x 16 roots per base.
 * Inputs and outputs host or device, as pls_kdmap_pose_search.  A scan without a valid row, or no map cell in the
 * reachable box, gives *out_num = 0.  Touches neither the map, its index, its normal cache nor any ICP state.
 * PLS_E_INVALID, the context unchanged, for every refusal of pls_kdmap_pose_search except its volume and bit limits,
 * and K < 1, out_T, out_score or out_index NULL, half_x or half_y >= 2^30, or A*(2*half_x+1)*(2*half_y+1) >= 2^62;
 * or when the kmax + 1 levels of the clipped grid (x rows padded to whole 32-bit words) exceed
 * PLS_POSE_SEARCH_PYRAMID_MAX_BITS bits (8 GiB, a tenth of an 80 GB H100; the extent is in pls_last_error), or
 * when the cell of every (base, scan row), 24 bytes each and computed once for all levels, would take more than
 * PLS_POSE_SEARCH_PYRAMID_MAX_CELL_BYTES (8 GiB: n * A < 2^33 / 24, e.g. 2 730 bases of a 131 072-row scan).  Also
 * PLS_E_INVALID, after work was enqueued but with the context unchanged, when more than
 * PLS_POSE_SEARCH_PYRAMID_MAX_NODES nodes survive at one level of one pass (the level and count are in
 * pls_last_error): a map where most poses of the window score alike, or fewer than K candidates in a large volume. */
#define PLS_POSE_SEARCH_PYRAMID_MAX_BITS (1ll << 36)
#define PLS_POSE_SEARCH_PYRAMID_MAX_CELL_BYTES (1ll << 33)
#define PLS_POSE_SEARCH_PYRAMID_MAX_NODES (1ll << 26)
PLS_API int pls_kdmap_pose_search_pyramid(pls_context* ctx, const float* scan, int64_t n,
                                          const double* bases /* [A,16] row-major float64 */, int A, double cell,
                                          int half_x, int half_y, int K /* >= 1 */,
                                          double* out_T /* [K,16] */, int32_t* out_score /* [K] */,
                                          int64_t* out_index /* [K] */, int* out_num);
/* pls_kdmap_pose_search for S scans in one call (a localisation server re-localising many vehicles' scans on one map,
 * offline map matching a recorded drive's scans from their GNSS fixes).  scans[s] [n[s],3] float32, host or device;
 * bases [sum A_s,16] row-major float64 (host or device), scan s's A_s = num_bases[s] bases after the earlier scans';
 * one cell and one K, per-scan windows half_x[s], half_y[s].  For each scan s the outputs are, bit for bit, what
 * pls_kdmap_pose_search(ctx, scans[s], n[s], bases of s, A_s, cell, half_x[s], half_y[s], K, ...) writes: its scores at
 * offset sum_{r<s} V_r of out_scores [sum V_s] (nullable), V_s = A_s*(2*half_x[s]+1)*(2*half_y[s]+1); out_T [S,K,16],
 * out_score [S,K], out_index [S,K] (L local to scan s's own volume) at row s, and out_num[s].  Entries past out_num[s]
 * are not written.  Outputs host or device.  One occupancy grid serves every scan: the bounding box of the union of the
 * scans' reachable boxes (each scan's base-cell box widened by its own window).  Touches neither the map, its index, its
 * normal cache nor any ICP state.  PLS_E_INVALID, the context unchanged, for any refusal pls_kdmap_pose_search would
 * give for some scan s (pls_last_error names s), S <= 0, a NULL array, sum V_s >= 2^31, or a shared grid of more than
 * PLS_POSE_SEARCH_MAX_BITS bits (x rows padded to whole 32-bit words; the extent is in pls_last_error). */
PLS_API int pls_kdmap_pose_search_scans(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                        const double* bases /* [sum A_s,16] */, const int* num_bases /* [S] */,
                                        double cell, const int* half_x /* [S] */, const int* half_y /* [S] */, int K,
                                        int32_t* out_scores /* [sum V_s] or NULL */, double* out_T /* [S,K,16] */,
                                        int32_t* out_score /* [S,K] */, int64_t* out_index /* [S,K] */,
                                        int* out_num /* [S] */);
/* ProjectiveLocalMap.update (local_map.py:126-202): rel_pose [16]; vertex_map [3,H,W] or NULL. */
PLS_API int pls_projmap_update(pls_context* ctx, const float* rel_pose, const float* vertex_map);
PLS_API int pls_projmap_num_frames(pls_context* ctx, int* num_frames);
/* The re-projected model maps _model_vmap/_model_nmap, each [K,3,H,W]. */
PLS_API int pls_projmap_model(pls_context* ctx, float* out_vmap, float* out_nmap);
/* The newest frame's vertex map [3,H,W] as it was inserted (ProjectiveLocalMap.get_last_frame, local_map.py:238-240).
 * PLS_E_STATE if the map holds no frame. */
PLS_API int pls_projmap_last_frame(pls_context* ctx, float* out_vmap);
/* ProjectiveLocalMap.nearest_neighbor_search (local_map.py:205-235): queries [n,3];
 * outputs [Nc,3] each (capacity H*W rows), row-major pixel order; *out_count = Nc. */
PLS_API int pls_projmap_nn_search(pls_context* ctx, const float* queries, int64_t n,
                          float* out_neighbors, float* out_normals, float* out_targets,
                          int64_t* out_count);

/* ---- a17/a18: the odometry ----------------------------------------------------------
 * ICPFrameToModel.init (icp_odometry.py:128-145). */
PLS_API int pls_odometry_init(pls_context* ctx);
/* ICPFrameToModel.register_new_frame (icp_odometry.py:248-299): points [n,3], T0 [16].
 * out_T [16], out_params [6], out_losses [max_num_alignments] (unused entries NaN),
 * *out_iters = iterations executed (= len(losses)). */
PLS_API int pls_register_frame(pls_context* ctx, const float* points, int64_t n, const float* T0,
                       float* out_T, float* out_params, float* out_losses, int* out_iters);
/* B hypotheses of one scan on the local map (kd-tree or projective), in one call (no reference counterpart:
 * relocalisation registers a scan from many initial guesses).  points [n,3] as pls_register_frame; T0s [B,16].
 * out_T [B,16], out_params [B,6], out_losses [B,max_num_alignments], out_iters [B]: hypothesis b's are the bits
 * pls_register_frame gives with T0s[b] on the same map.
 * out_status [B] (nullable): PLS_OK, PLS_W_TINY_RESIDUAL or PLS_E_SINGULAR per hypothesis; without it the call returns
 * PLS_E_SINGULAR if a hypothesis was singular (every output still written).  The map is not updated; afterwards the
 * last hypothesis is the context's last search (pls_kdmap_last_correspondences, pls_last_icp_sums).  Every kernel of an
 * ICP iteration is one launch for up to PLS_MAX_SEQUENCES hypotheses, larger B runs in chunks of that many (on a
 * projective map off the TMA path each hypothesis's correspondence kernel is its own launch).  Needs a map that has had
 * an update, gn_max_iters == 1, no communicator, B > 0 and n > 0. */
PLS_API int pls_register_hypotheses(pls_context* ctx, const float* points, int64_t n, const float* T0s, int B,
                                    float* out_T, float* out_params, float* out_losses, int* out_iters, int* out_status);
/* S scans registered from B initial estimates against the kd map ctx holds, in one call (no reference counterpart: a
 * localisation server registers many vehicles' scans on one map, offline map matching a recorded drive's scans).
 * scans[s]: [n[s],3] float32, host or device, n[s] > 0.  scan_of [B]: the scan registration b uses (NULL: b -> b,
 * which needs B == S).  T0s [B,16].  Outputs as pls_register_hypotheses: out_T [B,16], out_params [B,6],
 * out_losses [B,max_num_alignments], out_iters [B], out_status [B] (nullable, same rule for raising).
 * Registration b gives the bits pls_register_frame(scans[scan_of[b]], T0s[b]) gives on the same context.  The map is
 * not updated, its index not rebuilt; afterwards the last registration is the context's last search
 * (pls_kdmap_last_correspondences, pls_last_icp_sums), as if pls_register_frame had run it last.  One launch packs
 * every scan; every kernel of an ICP iteration is one launch for up to PLS_MAX_SEQUENCES registrations, larger B runs
 * in chunks of that many.  PLS_E_INVALID before any work, the context unchanged: a projective map, gn_max_iters != 1,
 * a communicator, a map that has had no update, S or B <= 0, an n[s] <= 0 or a scan_of entry outside [0, S). */
PLS_API int pls_register_scans(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                               const int* scan_of, const float* T0s, int B, float* out_T, float* out_params,
                               float* out_losses, int* out_iters, int* out_status);
/* pls_register_scans with a correspondence gate (no reference counterpart: the reference registers against its own
 * fresh local map; a prior map is stale -- moved cars, construction, partial overlap -- and a match beyond a distance
 * biases the pose).  Arguments, outputs and rules as pls_register_scans, plus max_distance and out_inliers.
 * For registration b, ICP iteration i, and a valid row p of its scan:
 *   p'      transform_point(T_b,i, p); q p's exact 1-NN in the map -- the point, with the tie rule, the ungated search
 *           returns;
 *   d^2     match_d2_f64 as pls_kdmap_evaluate_poses computes it: float64, every operation rounded on its own;
 *   inlier  d^2 <= max_distance * max_distance in float64.  Only inliers enter the 30 accumulators, the loss and the
 *           count; the search may report no match for an outlier (pls_kdmap_last_correspondences), never another
 *           point than q for an inlier.
 * out_inliers [B] (nullable, host or device): registration b's inlier count in its last executed iteration (its count
 * accumulator, pls_last_icp_sums[29] for the last registration).  A registration with too few inliers to solve stops
 * with PLS_E_SINGULAR in out_status, and so does one whose last iteration had no inlier at all (its pose is the last
 * one solved); the others go on.  max_distance = +inf gives pls_register_scans's bits for every
 * output.  Iteration 0 of a registration accumulates, bit for bit, entries 0..29 of pls_kdmap_evaluate_poses's row for
 * its initial pose and the same max_distance.  The map, its index and the odometry state are unchanged (the normal
 * cache may fill, with the bits it would get anyway); afterwards the last registration is the context's last search.
 * PLS_E_INVALID before any work, the context unchanged: everything pls_register_scans refuses, and a max_distance that
 * is NaN or negative. */
PLS_API int pls_register_scans_gated(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                     const int* scan_of, const float* T0s, int B, double max_distance, float* out_T,
                                     float* out_params, float* out_losses, int* out_iters, int* out_status,
                                     int* out_inliers);
/* pls_register_scans_gated with a solve that acts only in the directions the map constrains (no reference counterpart:
 * a tunnel, a corridor, an underpass or an open field leaves some directions of the pose unconstrained, and an ICP
 * step along them is driven by noise, or makes the registration singular).  This is the solution remapping of Zhang,
 * Kaess and Singh ("On degeneracy of optimization-based state estimation problems", ICRA 2016), which for a
 * Gauss-Newton step taken from the current pose is a truncated eigen-solve.  Arguments, staging, pointer rules,
 * chunking, outputs and the context's state afterwards are those of pls_register_scans_gated (max_distance = +inf: no
 * gate), plus min_eigenvalue, out_degenerate and out_eigenvalues.
 * Unchanged: the matches, normals and the 30 accumulators of every iteration are exactly those the gated call (at
 * +inf, pls_register_scans) forms at that iteration's pose; iteration 0's entries 0..29 are, bit for bit,
 * pls_kdmap_evaluate_poses's row at the initial pose and the same max_distance.  Only the solve differs.  For the sums
 * s of iteration i:
 *   H        the symmetric 6x6 matrix of the 21 upper-triangle entries s[0..20]; g = s[21..26]; N = s[29], the inlier
 *            (or match) count;
 *   (l_k, v_k)  the eigen-decomposition of H, in float64 on the device (cyclic Jacobi);
 *   kept     direction k when N > 0 and l_k >= min_eigenvalue * N in float64; otherwise it is degenerate;
 *   step     dx = -sum over the kept k of v_k (v_k^T g) / l_k, then the float32 cast, the threshold_delta_pose stop test
 *            and the pose update of pls_register_scans.  Along a degenerate direction the pose keeps its estimate.
 * Status: N = 0 is PLS_E_SINGULAR; then the tiny-residual rule (sqrt(s[28]) < 1e-7: PLS_W_TINY_RESIDUAL) as before;
 * then PLS_E_SINGULAR when no direction is kept -- this replaces the |det| >= 1e-7 test.  A finite gate with no inlier
 * in the last iteration is PLS_E_SINGULAR, as in pls_register_scans_gated.
 * out_degenerate [B] (nullable, host or device): the number of degenerate directions in registration b's last executed
 * iteration.  out_eigenvalues [B,6] (nullable, host or device): the ascending eigenvalues of H / N in that iteration
 * (zeros when N = 0).
 * Units: the threshold mixes them, as Zhang's does.  Per point, H's translation block is dimensionless -- at most 1
 * under the unweighted scheme, as it sums n n^T over unit normals -- and its rotation block is in m^2 (it grows with the
 * square of the points' range).  Calibrate min_eigenvalue on your own map from pls_kdmap_evaluate_poses's
 * (evaluate_registrations') eigenvalues / inliers, which is the same quantity as out_eigenvalues.
 * PLS_E_INVALID before any work, the context unchanged: everything pls_register_scans_gated refuses, and a
 * min_eigenvalue that is NaN, <= 0 or infinite. */
PLS_API int pls_register_scans_degeneracy(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                          const int* scan_of, const float* T0s, int B, double max_distance,
                                          double min_eigenvalue, float* out_T, float* out_params, float* out_losses,
                                          int* out_iters, int* out_status, int* out_inliers, int* out_degenerate,
                                          double* out_eigenvalues);
/* The quality of B registrations on the kd map ctx holds, in one call (no reference counterpart: a localiser that feeds
 * a filter or a pose graph needs each registration's inlier fraction, inlier RMSE and information matrix, and a
 * re-ranking of pose candidates needs more than an occupancy score).  Arguments, staging and pointer rules are those
 * of pls_register_scans: scans[s] [n[s],3] float32, host or device; scan_of [B] (NULL: b -> b, which needs B == S);
 * T [B,16] the poses, host or device.  For pose b and scan s = scan_of[b]:
 *   P         the valid rows of scan s (those pack_valid_rows keeps: no NaN coordinate);
 *   p'        transform_point(T_b, p) for p in P; q its exact 1-NN in the map and n_q q's cached normal -- the match and
 *             normal of the first ICP iteration of pls_register_frame(scan s, T_b);
 *   r, J, w   the residual, Jacobian [n, p' x n] and weight of that iteration (the context's scheme and sigma);
 *   d^2       ((dx dx + dy dy) + dz dz) in float64, dx = (double)p'_x - (double)q_x (likewise y, z), every operation
 *             rounded on its own: numpy's element-wise float64 expressions give the same bits;
 *   inlier    a matched query with d^2 <= max_distance * max_distance (float64); max_distance = +inf admits every match.
 * out_stats [B,PLS_EVAL_STATS] (host or device), row b: [0..29] the accumulators of pls_kdmap_last_correspondences's
 * layout (21 JtJ upper, 6 Jtr, sum (w r)^2, sum r^2, count) over the inliers only; [30] sum d^2 over the inliers;
 * [31] |P|.  With max_distance = +inf, [0..29] are bit for bit the out_sums pls_kdmap_last_correspondences reports
 * after pls_register_frame(scan s, T_b) with max_num_alignments = 1 on the same map.  Row b does not depend on B, on
 * b's place in the batch or on the other scans: a batch equals B single-pose calls bit for bit.
 * Nothing is solved.  The map, its index, its frame counts and the odometry state are unchanged (the normal cache may
 * fill, with the bits it would get anyway); afterwards the last pose is the context's last search, as
 * pls_register_scans leaves it, with its row's [0..29] as the last sums (pls_kdmap_last_correspondences,
 * pls_last_icp_sums).  One launch packs every scan; each kernel is one launch for up to PLS_MAX_SEQUENCES poses, larger B
 * runs in chunks of that many.  PLS_E_INVALID before any work, the context unchanged: a projective map, a communicator,
 * a map that has had no update, S or B <= 0, an n[s] <= 0, a scan_of entry outside [0, S), a NULL scans, n, scan, T or
 * out_stats, or a max_distance that is NaN or negative. */
#define PLS_EVAL_STATS 32
PLS_API int pls_kdmap_evaluate_poses(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                     const int* scan_of, const float* T, int B, double max_distance,
                                     double* out_stats);
/* ICPFrameToModel.do_process_next_frame (icp_odometry.py:157-246): `data` is [n,3] points
 * (PLS_INPUT_NDARRAY / PLS_INPUT_TENSOR: float; the _F64 variants: double) or a float [3,H,W] vertex map
 * (PLS_INPUT_VERTEX_MAP, n ignored).  init_pose [16] or NULL (identity).  On frame 0 the map is initialised and
 * *out_has_pose = 0 (the reference writes no "odometry_pose" then).  out_info (optional,
 * 12 doubles): iterations, final loss, queries used, map points, grid samples, NaN rows dropped,
 * status, key-frame inserted, first non-null pixel x/y/z (vertex-map layout), 1 if the correspondences were
 * sharded over the ranks of a multi-GPU communicator (0: every rank ran the whole frame). */
PLS_API int pls_process_frame(pls_context* ctx, const void* data, int layout, int64_t n,
                      const float* init_pose, float* out_pose, float* out_params,
                      int* out_has_pose, double* out_info);
/* Fused preprocessing + odometry for the shipped pipeline (grid_sample.yaml): GridSample
 * (voxel) -> ToTensor -> process_frame(PLS_INPUT_TENSOR or _NDARRAY) with no host hop. */
PLS_API int pls_process_frame_grid_sample(pls_context* ctx, const float* raw_points, int64_t n, double voxel,
                                  int layout, const float* init_pose, float* out_pose,
                                  float* out_params, int* out_has_pose, double* out_info);

/* Several independent sequences, one frame each, in one call (no reference counterpart: the reference's runner
 * processes sequences one after another, odometry_runner.py:145-175).  ctxs [num] distinct contexts on one device,
 * all with kd-tree local maps or all with projective ones (a mixed call is refused); their other settings (frame size,
 * local_map_size, scheme, ...) may differ.  data / layouts / n / init_poses [num] as pls_process_frame (data[i] == NULL:
 * sequence i skipped);
 * voxel > 0 grid-samples every sequence first, as pls_process_frame_grid_sample; outputs [num,16] / [num,6] / [num] /
 * [num,12] / [num], each nullable.  num <= PLS_MAX_SEQUENCES.
 * Every context ends in the state its own pls_process_frame (pls_process_frame_grid_sample) call would have left, with
 * the same outputs, bit for bit; a sequence may be on its first frame.  Each kernel of an ICP iteration is one launch for
 * every sequence.  Contexts must have gn_max_iters == 1 and no communicator; otherwise PLS_E_INVALID before any work.
 * Errors are per sequence: out_status[i] (PLS_E_SINGULAR, or an input pls_process_frame refuses, leaves sequence i as
 * pls_process_frame leaves it after that error, the others complete), pls_last_error(ctxs[i]) its text; the call
 * returns the first non-OK status in sequence order.  A failure of no one sequence (a CUDA error) ends the call: every
 * sequence whose frame had not completed reports it, those that completed keep PLS_OK.  The profiling slots
 * (pls_profile_*) are not credited by this call; PLS_BATCH_TRACE=<file> appends its per-phase times to <file>. */
enum { PLS_MAX_SEQUENCES = 64 };
PLS_API int pls_process_frames(pls_context* const* ctxs, int num, const void* const* data, const int* layouts,
                               const int64_t* n, double voxel, const float* const* init_poses, float* out_poses,
                               float* out_params, int* out_has_pose, double* out_info, int* out_status);
/* Test / debug aid: out_sums [30] = the accumulators of the last executed ICP iteration of the last frame of
 * pls_register_frame, pls_process_frame(_grid_sample) or pls_process_frames on this context, for either map type (the
 * order of pls_kdmap_last_correspondences: 21 JtJ upper, 6 Jtr, sum (w r)^2, sum r^2, count); *out_iters (nullable) =
 * that frame's executed iterations.  Reads the host copy of the frame's result: no kernel, no synchronisation, a
 * pending map update is not flushed.  PLS_E_STATE before the context's first ICP frame. */
PLS_API int pls_last_icp_sums(pls_context* ctx, double* out_sums, int* out_iters);

/* ---- the rows either side of the path (SURVEY.md section 8f, ranks 1-2) -----------------------------------
 * Distortion.filter (slam/preprocessing.py:148-191): de-skew of a frame with the estimated relative motion.
 * xyz [n,3] float32|float64; timestamps [n] float32|float64 (alpha is formed in their dtype, like numpy does);
 * rel_pose [16] float32|float64 (the data_dict's init_rpose); out [n,3] FLOAT64 = Slerp(I -> R)(alpha_i) p_i +
 * alpha_i t.  Constant timestamps give alpha = 0; a NaN timestamp makes every output NaN (np.max/np.min). */
PLS_API int pls_distort(pls_context* ctx, const void* xyz, int xyz_is_f64, const void* timestamps, int ts_is_f64,
                int64_t n, const void* rel_pose, int pose_is_f64, double* out);
/* Voxelization.filter (slam/preprocessing.py:71-97) = voxelise + voxel_hashing + voxel_normal_distribution
 * (slam/common/pointcloud.py:54-79,40-51,83-167).  coords_out [n,3] / hashes_out [n] as pls_voxel_hash (nullable);
 * per distinct hash, in ascending hash order: sizes_out [V] int64, means_out [V,3], covs_out [V,3,3] = the scatter
 * matrix sum (x - mean)(x - mean)^T (not divided by the count), both in the dtype of the input; ids_out [n] int64 =
 * voxel rank of every point.  Per-voxel outputs need capacity n rows; *out_count = V. */
PLS_API int pls_voxel_statistics(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel,
                         int64_t* coords_out, int64_t* hashes_out, int64_t* sizes_out, void* means_out,
                         void* covs_out, int64_t* ids_out, int64_t* out_count);
/* GaussNewtonPointToPointAlignment.align (slam/odometry/alignment.py:144-189) -> GaussNewton.compute
 * (optimization.py:296-344) with PointToPointCost closures (optimization.py:458-541): r = |R p + t - q| and the
 * reference's Jacobian as written, J[k] = (dT/dx_k p~) . (R p + t - q).  Arguments as pls_align_p2plane. */
PLS_API int pls_align_p2point(pls_context* ctx, const void* ref, const void* tgt, int64_t n, int is_f64, int scheme,
                      double sigma, int max_iters, double norm_stop, const void* x0, void* out_dT, void* out_x,
                      void* out_loss);
/* The two alignments on a batch of `batch` correspondence sets of n points each, in one call: ref/tgt/nrm
 * [batch,n,3], x0 [batch,6] or NULL, out_dT [batch,16], out_x [batch,6], out_loss [batch,n] or NULL, out_iters
 * (host int, nullable) the iterations executed.  GaussNewton.compute's batch semantics (optimization.py:318-341):
 * every iteration works on all elements; the tiny-residual guard takes the norm of all batch*n residuals
 * (PLS_W_TINY_RESIDUAL, every x unchanged), one element with |det H| < 1e-7 fails the call (PLS_E_SINGULAR), and
 * all elements stop together once |dx| over all batch*6 increments is below norm_stop.  pls_align_p2plane /
 * pls_align_p2point are this call at batch 1. */
PLS_API int pls_align_p2plane_batch(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t batch,
                                    int64_t n, int is_f64, int scheme, double sigma, int max_iters, double norm_stop,
                                    const void* x0, void* out_dT, void* out_x, void* out_loss, int* out_iters);
PLS_API int pls_align_p2point_batch(pls_context* ctx, const void* ref, const void* tgt, int64_t batch, int64_t n,
                                    int is_f64, int scheme, double sigma, int max_iters, double norm_stop,
                                    const void* x0, void* out_dT, void* out_x, void* out_loss, int* out_iters);
/* weighted_procrustes, numpy path (slam/common/registration.py:15-76): rigid T (float64 [16]) with
 * T * tgt ~ ref.  tgt / ref [n,3] and weights [n] (nullable) share one dtype; the weights only enter the centroids. */
PLS_API int pls_weighted_procrustes(pls_context* ctx, const void* tgt, const void* ref, const void* weights, int64_t n,
                            int is_f64, double* out_T);

/* _PointToPlaneLossModule.point_to_plane_loss (slam/training/loss_modules.py:51-104), forward AND backward: the
 * unsupervised point-to-plane training loss of a batch of (target, reference) vertex-map pairs and its gradient with
 * respect to the predicted poses, as the reference's autograd computes it (values flow through the z-buffer scatter to
 * every point written to a pixel; rounded pixel coordinates carry no gradient).  vm_target / vm_reference /
 * nm_reference [B,3,H,W]; pose_mats [B,16] or NULL (then built from pose_params [B,6], Euler xyz); up/down fov of the
 * projector; scheme / sigma = least_square_scheme.  out_loss [1] = mean_b(sum C(|r|)^2 / sum mask); optional
 * out_loss_per_batch [B], out_grad_mats [B,16] (d loss / d pose matrix, last row 0), out_grad_params [B,6]. */
PLS_API int pls_p2plane_loss(pls_context* ctx, const float* vm_target, const float* vm_reference,
                     const float* nm_reference, const float* pose_mats, const float* pose_params, int batch,
                     int height, int width, float up_fov_deg, float down_fov_deg, int scheme, float sigma,
                     float* out_loss, float* out_loss_per_batch, float* out_grad_mats, float* out_grad_params);

/* ---- the rows either side of the path, rank 4: dataset -> vertex-map ingestion and pose chains --------------------------
 * KITTIOdometrySequence.correct_scan (slam/dataset/kitti_dataset.py:200-231): the HDL-64 intrinsic correction, every point
 * rotated by 0.205 degrees about normalise(p x e_z).  scan [n, stride] float32 rows (x, y, z[, reflectance]), stride 3 or 4;
 * out_xyz [n,3] FLOAT64 (the reference's result dtype).  Points on the vertical axis come out NaN, as in the reference. */
PLS_API int pls_kitti_correct_scan(pls_context* ctx, const float* scan, int64_t n, int stride, double* out_xyz);
/* KITTIOdometrySequence.__getitem__ (kitti_dataset.py:233-249): optional rectification, then the spherical projection +
 * closest-wins z-buffer in float64 (Projector.build_projection_map on the float64 cloud).  out_xyz [n,3] float64 (the
 * `numpy_pc` entry; may be NULL), out_vertex_map [3,H,W] float64 (the `vertex_map` entry). */
PLS_API int pls_ingest_scan(pls_context* ctx, const float* scan, int64_t n, int stride, int correct, int height, int width,
                    float up_fov_deg, float down_fov_deg, double* out_xyz, double* out_vertex_map);
/* compute_relative_poses (slam/eval/eval_odometry.py:80-83): out[i] = inv(poses[i-1]) @ poses[i], out[0] = poses[0];
 * poses / out [n,4,4] float32 or float64 (is_f64), computed in that precision. */
PLS_API int pls_relative_poses(pls_context* ctx, const void* poses, int64_t n, int is_f64, void* out);
/* compute_absolute_poses (eval_odometry.py:86-96): out[0] = rel[0], out[i+1] = out[i] @ rel[i+1] (sequential product). */
PLS_API int pls_absolute_poses(pls_context* ctx, const void* relative_poses, int64_t n, int is_f64, void* out);

/* ---- multi-GPU: per-iteration allreduce of the normal-equation accumulators ---------
 * (no reference counterpart: SURVEY.md section 8e).  Every rank holds the whole local map
 * (kd) or its band of image rows (projective) and a shard of the queries; after
 * pls_comm_init the 30 accumulators are summed across ranks once per ICP iteration.
 * nccl_unique_id: the 128-byte ncclUniqueId created on rank 0 and broadcast by the host
 * program (torch.distributed); nccl_library: path of libnccl.so.2 to dlopen. */
PLS_API int pls_comm_init(pls_context* ctx, int num_ranks, int rank, const void* nccl_unique_id,
                  const char* nccl_library);
PLS_API int pls_comm_unique_id(const char* nccl_library, void* out_id_128_bytes);
/* One-shot peer-to-peer mode (NVLink / NVSwitch peer memory, no NCCL on the data path): the all-reduce is
 * fused into the solve kernel -- every rank stores its 30 partial sums and a sequence flag directly into each
 * peer's exchange slots and sums the slots in rank order.  Step 1: each rank exports the 64-byte CUDA IPC
 * handle of its exchange buffer; the host program all-gathers the handles; step 2 maps them. */
PLS_API int pls_comm_p2p_handle(pls_context* ctx, int num_ranks, void* out_handle_64_bytes);
PLS_API int pls_comm_p2p_init(pls_context* ctx, int num_ranks, int rank, const void* all_handles /* [num_ranks][64] */);
PLS_API int pls_comm_destroy(pls_context* ctx);
/* Sharding threshold: a frame's correspondences are split over the ranks only if every rank gets at least this many work
 * items (queries of the kd map / pixels of the projective map); below it every rank runs the whole frame itself and no
 * exchange takes place (identical inputs + deterministic kernels = identical poses).  Default 24576, a third of it for
 * kd maps of 2 M points and more, where a query costs several times as much (environment
 * variable PLS_SHARD_MIN); a negative value restores the default.  Process-wide; every rank must set the same value. */
PLS_API int pls_set_shard_min(int64_t work_items_per_rank);
/* 1 if the last ICP of this context split its correspondences over the ranks, else 0. */
PLS_API int pls_last_sharded(pls_context* ctx, int* out);

/* ---- measurement ---------------------------------------------------------------------
 * CUDA-event timing of one kernel family inside the library's own launches.
 * which: 0 = kd correspondence+reduction kernel, 1 = projective correspondence+reduction
 * kernel, 2 = model rebuild, 3 = index build, 4 = grid sample, 5 = Gauss-Newton solve.
 * pls_profile_read returns the accumulated device milliseconds, launch count and the
 * algorithmic bytes the launches moved (DESIGN.md states the per-unit figures). */
/* Number of CUDA kernels this library has launched in this process (all contexts). */
PLS_API int pls_launch_count(int64_t* out);
PLS_API int pls_profile_enable(pls_context* ctx, int which, int enable);
PLS_API int pls_profile_read(pls_context* ctx, int which, double* ms_total, int64_t* launches,
                     double* algorithmic_bytes, int reset);

#ifdef __cplusplus
}
#endif
#endif /* PLSLAM_B200_H */
