// Internal declarations shared by the translation units of libplslam_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <deque>
#include <string>
#include <vector>

#include "../../include/plslam_b200.h"

namespace pls {

constexpr int kNumSMs = 132;  // H100 SXM
constexpr int NACC = 30;      // 21 JtJ upper + 6 Jtr + sum (w r)^2 + sum r^2 + count
constexpr int kMaxAlign = 128;
constexpr int kProfileSlots = 16;  // 0-5: kernel families of the bench line; 6-15: single kernels (development)
constexpr size_t kScalarOffset = 2048;  // FrameResult first, then u32 scalar slots

struct Error {
    int code;
    std::string msg;
};

extern long long g_kernel_launches;

#define PLS_CUDA(expr)                                                                            \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            throw pls::Error{PLS_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) +     \
                                             " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"}; \
        }                                                                                         \
    } while (0)

// every kernel launch of the library is followed by this check, which also counts it
#define PLS_CHECK_LAUNCH()            \
    do {                              \
        ++pls::g_kernel_launches;     \
        PLS_CUDA(cudaGetLastError()); \
    } while (0)

// A launch of a kernel on a dependent chain, with programmatic stream serialisation: the kernel may be launched while
// its predecessor in the stream is still finishing, which hides the launch latency between the two.  Every kernel
// launched this way calls pls_grid_dependency_wait() before its first global memory access; the wait returns once the
// predecessor grid has completed and its writes are visible, and is a no-op in a plain launch.
#ifdef __CUDACC__
__device__ __forceinline__ void pls_grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif
template <typename... KArgs, typename... Args>
void launch_dependent(void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    PLS_CUDA(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
    PLS_CHECK_LAUNCH();
}

#define PLS_REQUIRE(cond, text)                                   \
    do {                                                          \
        if (!(cond)) throw pls::Error{PLS_E_INVALID, (text)};     \
    } while (0)

// Growable device buffer.  Growth synchronises the stream (only before steady state).
struct DBuf {
    void* p = nullptr;
    size_t cap = 0;
    template <typename T>
    T* as() const { return reinterpret_cast<T*>(p); }
    void reserve(size_t bytes, cudaStream_t s, bool keep = false);
    void reserve_exact(size_t bytes, cudaStream_t s, bool keep = false);  // no head-room: the caller planned the size
    void release();
};

// Pinned host buffer.
struct HBuf {
    void* p = nullptr;
    size_t cap = 0;
    template <typename T>
    T* as() const { return reinterpret_cast<T*>(p); }
    void reserve(size_t bytes);
    void release();
    void* device_ptr() const;  // the device-side alias of the mapped allocation
};

struct ProfileSlot {
    bool enabled = false;
    std::vector<cudaEvent_t> pool;  // pairs
    size_t used = 0;
    double ms = 0.0;
    int64_t launches = 0;
    double bytes = 0.0;
};

// ---- radix sort / scan scratch ---------------------------------------------------------
struct SortScratch {
    DBuf keys_alt, vals_alt;  // ping-pong partners of the caller's arrays
    DBuf hist;                // [8][256] u32 histograms, then exclusive bases
    DBuf status;              // [passes][tiles][256] look-back words + tile counters
    DBuf plan;                // device-side SortPlan
};

struct ScanScratch {
    DBuf status;  // look-back words + tile counter + total
};

// select_device.cuh: epoch-tagged look-back words of the single-pass selection (one scratch per stream)
struct SelectScratch {
    DBuf status;
    uint32_t epoch = 0;
};

// ---- the kd local map: point storage + the cell-pyramid search index (kdmap_device.cuh) ---------------------
struct KdMap {
    // insertion-ordered storage, float4 (x,y,z,unused); ping-pong for the per-frame move
    DBuf store[2];
    int cur = 0;
    int64_t count = 0;                // points in store[cur]
    std::deque<int64_t> frame_counts; // per inserted frame
    // search index
    DBuf morton, order;     // u64 cell keys, u32 original index (sorted)
    DBuf sorted;            // float4 (x,y,z, bitcast original index), level-0 cell order
    DBuf sorted_prev;       // a device-decided update builds into the other buffer: the sorted points of generation
    uint32_t prev_gen = 0;  // prev_gen (0: none), which the last frame's search ran on, stay exportable
    DBuf normals;           // float4 (nx,ny,nz, state word) in sorted order; states carry the build generation
    DBuf bbox;              // 6 ordered-int words
    bool bbox_clean = false; // the header kernel of the last build left the box empty
    DBuf grid_hdr;          // KdGridHeader (quantisation + cell levels)
    DBuf cells;             // cell hash tables of all levels (generation-stamped entries, never cleared)
    DBuf stats;             // optional debug counters (PLS_KD_STATS=1)
    size_t table_offset[16] = {};
    uint32_t table_mask[16] = {};
    uint32_t gen = 0;       // generation of the current index build (0 = never built)
    int64_t indexed = 0;    // points covered by the index
    bool valid = false;
    int64_t cap_points = 0; // every per-point array holds this many points (kd_reserve_capacity)
    int64_t max_frame = 0;  // largest frame inserted so far (sizes the steady state: local_map_size frames)
    // the last search (an ICP iteration or pls_kdmap_nn_search), whose matches and states nn_prev / kd_nn_state hold
    // (read back by pls_kdmap_last_correspondences)
    bool searched = false;
    bool searched_icp = false;      // an ICP iteration: the query count is the FrameResult's, the sums its last_sums
    bool searched_sharded = false;  // the queries were split over ranks: this rank holds only its share
    bool searched_normals = false;  // the normals of the matched points were computed
    uint32_t searched_gen = 0;      // index generation the matches refer to
    int64_t searched_n = 0;         // query count (pls_kdmap_nn_search)
};

struct ProjMap {
    int K = 0;              // frames held
    int head = 0;           // ring slot of the oldest frame
    DBuf vmaps, nmaps;      // [Kmax+1][3][H][W] ring; logical frame k lives in slot (head + k) % (Kmax+1)
    DBuf poses;             // device copy of [Kmax][16] poses (frame -> newest frame)
    std::vector<float> host_poses;  // [K][16]
    DBuf model_v, model_n;  // [Kmax][3][H][W] re-projected model
    DBuf zbuf;              // [Kmax][H][W] u64
    bool valid = false;
    bool zbuf_clean = false; // the query z-buffer (tmp[3]) is known to be all-empty
    int64_t built_lo = 0, built_hi = 0;  // pixel range the model currently covers (a rank of a sharded job builds its share)
};

struct FrameResult {        // mirrored to pinned host memory at the end of a frame
    float T[16];
    float params[6];
    float losses[kMaxAlign];
    int iters;
    int status;
    int done;
    int pad;
    double last_sums[NACC];
    long long counts[8];    // [0]=samples S, [1]=queries, [2]=valid rows of the frame's points
    float first_pt[4];      // first non-null pixel (vertex-map input quirk)
};

struct Comm;  // NCCL glue (comm.cu)

static_assert(sizeof(FrameResult) <= kScalarOffset, "FrameResult must fit before the scalar slots");

// The kd map update of a frame as its device-side decision (kd_update_decision_kernel, odometry.cu) leaves it for the
// update's launches, in the scalar block behind the FrameResult, so that the frame's one result copy brings it back.
struct KdUpdateWords {
    float X[12];          // the move inverse(T): R row-major, then t
    float delta[16];      // _delta_since_map_update after the frame
    uint32_t gate;        // 1: the update runs -- the frame's ICP is complete and succeeded on a valid grid sample
    uint32_t insert;      // the frame is a key frame
    uint32_t skip;        // points of the evicted frame, at the front of the store
    uint32_t kept;        // points moved
    uint32_t num_new;     // points appended
    uint32_t total;       // map points after the update (kept + num_new; 0 while the gate is closed)
    uint32_t pad[2];
};
constexpr size_t kUpdateOffset = kScalarOffset - 256;
static_assert(sizeof(FrameResult) <= kUpdateOffset && sizeof(KdUpdateWords) <= 256, "KdUpdateWords after FrameResult");

}  // namespace pls

struct pls_context {
    pls_config cfg;
    cudaStream_t stream = nullptr;      // the stream kernels are currently enqueued on
    cudaStream_t stream_main = nullptr; // caller-visible stream (== stream outside a map-update scope)
    cudaStream_t stream_map = nullptr;  // local-map update stream (overlaps the next frame's preprocessing)
    cudaEvent_t ev_map_done = nullptr;  // recorded on stream_map after every asynchronous map update
    cudaEvent_t ev_inputs = nullptr;    // pls_wait_stream: orders the caller's stream before this context's work
    bool map_pending = false;
    bool own_stream = false;
    std::string err;

    // staging for host<->device argument traffic
    pls::DBuf stage_in[4], stage_out[6];
    pls::HBuf pinned;       // FrameResult + small scalars
    pls::DBuf scalars;      // device scalars (counts, flags, FrameResult)

    pls::SortScratch sort;
    pls::SortScratch sort_map;          // radix-sort scratch of the map-update stream
    pls::ScanScratch scan;
    pls::SelectScratch sel[2];          // [0] main stream, [1] map-update stream
    pls::DBuf input_zbuf;               // z-buffer of the frame-input stage (kept all-empty between frames by its consumers)
    bool input_zbuf_clean = false;

    // generic scratch
    pls::DBuf tmp[8];
    // scratch of the stateless filters / alignments either side of the path (filters.cu, registration.cu, voxel
    // statistics): kept apart from tmp[] so that they never alias buffers of an in-flight frame
    pls::DBuf next_buf[8];

    // odometry state (icp_odometry.py:100-121)
    pls::KdMap kd;
    pls::ProjMap pm;
    int frame_index = 0;
    int last_icp_iters = 0;             // iterations the previous frame's ICP executed (sizes the up-front enqueue)
    bool icp_result = false;            // the host FrameResult holds an ICP frame's result (pls_last_icp_sums)
    bool last_sharded = false;          // the last ICP actually split its correspondences over the ranks
    int sample_pointcloud = 0;          // _sample_pointcloud
    float delta_since_update[16];       // _delta_since_map_update
    pls::DBuf frame_vmap_buf[2];        // [3][H][W] of the current frame (double-buffered: the previous one may
    pls::DBuf frame_pts_buf[2];         // still be read by the map-update stream); float4 packed valid points
    int frame_slot = 0;
    // the local-map update of the last frame, decided by the host but not yet enqueued: the next call enqueues it first
    // (flush_map_update).  A kd map's update on one GPU is decided on the device and enqueued with its frame instead
    // (odometry.cu: enqueue_device_map_update), and none is left pending
    bool upd_pending = false, upd_insert = false;
    float upd_T[16];
    int upd_slot = 0;
    long long upd_count = 0;
    pls::DBuf queries;                  // float4 queries P0 (owned storage)
    const float4* query_ptr = nullptr;  // the queries of the current frame (may alias frame_pts)
    pls::DBuf nn_prev;                  // previous-iteration match per query
    pls::DBuf kd_worklist;              // map points whose normal the current iteration has to compute; queued queries
    pls::DBuf kd_nn_state;              // per query: position at its last full search + runner-up bound (float4)
    pls::DBuf partials;                 // [blocks][NACC] doubles
    pls::DBuf batch_buf;                // pls_process_frames led by this context: sequence descriptors, then done flags
    pls::DBuf hyp_buf;                  // pls_register_hypotheses: FrameResults and per-query state of the hypotheses
    pls::DBuf degen_buf;                // pls_register_scans_degeneracy: a chunk's eigenvalues and degenerate counts
    cudaEvent_t ev_batch = nullptr;     // pls_process_frames: this context's input stage, before the batched ICP
    cudaEvent_t ev_icp_done = nullptr;  // a frame's ICP launches and its map-update decision, before the map stream's update
    pls::DBuf gs_keys, gs_vals, gs_out_xyz, gs_out_idx;
    pls::DBuf gs_bins;                  // bucket grid sample: 2^16 bin counts + control words, zero between calls
    pls::DBuf gs_buckets;               // bucket grid sample: bucket starts + look-back words
    uint32_t gs_seq = 0;                // stamp of the last compact-key grid sample (overflow detection)
    pls::HBuf gs_host_xyz, gs_host_idx; // pinned + mapped staging the grid sample's gather writes directly (host callers)
    int64_t last_query_count = 0;

    pls::Comm* comm = nullptr;
    void* p2p_pending_xchg = nullptr;   // exchange buffer exported by pls_comm_p2p_handle, adopted by pls_comm_p2p_init
    pls::ProfileSlot prof[pls::kProfileSlots];
};

namespace pls {
void flush_map_update(pls_context* ctx);  // odometry.cu: enqueues the deferred local-map update of the last frame, if any
}

#define PLS_API_BEGIN(ctx)                               \
    if (!(ctx)) return PLS_E_INVALID;                    \
    try {                                                \
        cudaSetDevice((ctx)->cfg.device);                \
        pls::flush_map_update(ctx);

/* entry points of the per-frame path: they enqueue the pending map update themselves, behind their own first kernels */
#define PLS_API_BEGIN_FRAME(ctx)                         \
    if (!(ctx)) return PLS_E_INVALID;                    \
    try {                                                \
        cudaSetDevice((ctx)->cfg.device);

#define PLS_API_END(ctx)                                 \
    }                                                    \
    catch (const pls::Error& e) {                        \
        (ctx)->err = e.msg;                              \
        return e.code;                                   \
    }                                                    \
    catch (const std::exception& e) {                    \
        (ctx)->err = e.what();                           \
        return PLS_E_INVALID;                            \
    }                                                    \
    return PLS_OK;

namespace pls {

// device scalar slots (u32) living behind the FrameResult in ctx->scalars
enum { SC_GS_COUNT = 0, SC_QUERY_COUNT = 1, SC_NAN_COUNT = 2, SC_INSERT_COUNT = 3, SC_PROJ_NC = 4,
       SC_SPARE0 = 5, SC_SPARE1 = 6,
       SC_GS_OVERFLOW = 7,
       SC_KD_COUNTERS = 8,      // four u64 counters of the kd search kernels (slots 8..15)
       SC_KD_LISTS = 16,        // per-iteration work-list counters of the kd search (kdmap.cu: KDL_*), 8 words
       SC_NUM = 32 };

// ---- pointer classification + staging ---------------------------------------------------
bool is_device_ptr(const void* p);           // cached per address
bool is_device_ptr_uncached(const void* p);
// Returns a device pointer holding `bytes` of `p` (copying through `stage` if p is host).
const void* to_device(pls_context* ctx, const void* p, size_t bytes, DBuf& stage);
// Returns a device pointer results may be written to; if `p` is host, it is `stage` and
// finish_out() copies back.
struct OutArg {
    void* host = nullptr;
    void* dev = nullptr;
    size_t bytes = 0;
};
OutArg out_arg(pls_context* ctx, void* p, size_t bytes, DBuf& stage);
void finish_out(pls_context* ctx, const OutArg& o, size_t bytes_used = (size_t)-1);
// Copies `bytes` of host memory to an output that may be host or device memory; nothing for a NULL dst or zero bytes.
// Synchronous: the caller's host buffer may go once it returns.
void put_out(void* dst, const void* src, size_t bytes);

inline uint32_t* scalar_u32(pls_context* ctx, int i) {
    return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(ctx->scalars.p) + kScalarOffset) + i;
}
inline FrameResult* frame_result_dev(pls_context* ctx) { return reinterpret_cast<FrameResult*>(ctx->scalars.p); }
inline FrameResult* frame_result_host(pls_context* ctx) { return reinterpret_cast<FrameResult*>(ctx->pinned.p); }
inline KdUpdateWords* kd_update_words_dev(pls_context* ctx) {
    return reinterpret_cast<KdUpdateWords*>(reinterpret_cast<char*>(ctx->scalars.p) + kUpdateOffset);
}
inline const KdUpdateWords* kd_update_words_host(pls_context* ctx) {
    return reinterpret_cast<const KdUpdateWords*>(reinterpret_cast<const char*>(ctx->pinned.p) + kUpdateOffset);
}

// The asynchronous map-update scope: kernels enqueued inside run on stream_map with its own sort scratch.
void map_stream_begin(pls_context* ctx);
void map_stream_end(pls_context* ctx);
// Makes the main stream wait for the last asynchronous map update (no-op if none is pending).
void map_stream_wait(pls_context* ctx);
// Host-blocking: both streams idle.
void sync_all(pls_context* ctx);

// ---- profiling ------------------------------------------------------------------------------
struct ProfileScope {
    pls_context* ctx;
    int which;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    // count = false: the launch may be a device-side no-op (ICP already converged); the caller
    // credits launches/bytes afterwards with profile_credit() once the executed count is known
    ProfileScope(pls_context* c, int w, double bytes, bool count = true);
    ~ProfileScope();
};
void profile_collect(pls_context* ctx, int which);
inline void profile_credit(pls_context* ctx, int which, int64_t launches, double bytes) {
    if (!ctx->prof[which].enabled) return;
    ctx->prof[which].launches += launches;
    ctx->prof[which].bytes += bytes;
}

// ---- primitives (sort.cu / scan.cu) ------------------------------------------------------------
// Stable LSD radix sort of (u64 key, u32 value) pairs on bits [0, 8*num_passes).
// keys/vals are sorted in place from the caller's view: on return *keys_out/*vals_out point at
// the arrays holding the result (either the inputs or the scratch partners) -- they are device
// pointers stored in DEVICE memory (the plan), and also returned on the host when the number of
// executed passes is statically known (no skipping), which is how it is used here.
// cap_n >= n: the scratch is sized for cap_n elements (callers whose n grows towards a known bound pass the bound).
// n_dev (nullable): the element count on the device, read by the kernels; n is then a bound of it that sizes the launches.
void radix_sort_pairs(pls_context* ctx, uint64_t* keys, uint32_t* vals, int64_t n, int num_passes,
                      uint64_t** keys_out, uint32_t** vals_out, int64_t cap_n = 0, const uint32_t* n_dev = nullptr);

// Exclusive scan / stream compaction with a single-pass decoupled look-back.
// flags[i] in {0,1}; pos_out[i] = number of set flags before i; *total_dev = number set.
void exclusive_scan_flags(pls_context* ctx, const uint8_t* flags, int64_t n, uint32_t* pos_out,
                          uint32_t* total_dev);

// ---- device-side math shared by kernels ---------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// float <-> order-preserving int (for atomicMin/Max on floats)
__device__ __forceinline__ int float_to_ordered(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int i) {
    return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff);
}
// voxelise's coordinate rule (slam/common/pointcloud.py:13-23): int64(round_half_even(v / voxel)), true float64
// division.  The voxel hash and the pose search's occupancy both use it, so a cell means the same in both.
__device__ __forceinline__ long long voxel_coord(double v, double voxel) { return __double2ll_rn(v / voxel); }
#endif

// ---- module entry points used across translation units -----------------------------------------
// projection.cu
void launch_projection(pls_context* ctx, const float* xyz, const float* channels, int batch, int64_t n,
                       int C, int H, int W, float up, float down, float* out, unsigned long long* zbuf, float fill = 0.f);
// float64 cloud [n,3] -> float32 vertex map [3,H,W]: pixel math, range comparison and validity in float64, values
// rounded to float32 at the end (what the reference does with a float64 input, icp_odometry.py:331-352)
void launch_projection_f64(pls_context* ctx, const double* xyz, int64_t n, int H, int W, float up, float down, float* out,
                           unsigned long long* zbuf);
// z-buffer pass only (no resolve): one 64-bit atomicMin of (range bits << 32 | point index) per point; n_dev (nullable)
// is a device-side point count overriding n.  The buffer must hold ~0 in every pixel beforehand.
void launch_zbuf_points(pls_context* ctx, const float* xyz, int64_t n, const uint32_t* n_dev, int H, int W, float up, float down,
                        unsigned long long* zbuf);
// normal_map.cu
void launch_normal_map(pls_context* ctx, const float* vmap, int batch, int H, int W, int ksize, float* out);
// gn.cu
struct GnParams {
    int scheme;
    double sigma;
};
// kdmap.cu
void kdmap_reset(pls_context* ctx);
// raw rows [n,3] or a vertex map [3,H,W] are packed (NaN rows / near-null pixels dropped) and
// inserted; known_count >= 0 skips the host sync that otherwise reads the packed count.
void kdmap_update(pls_context* ctx, const float* rel_pose_host, const float* pts_dev, int64_t n,
                  const float* vmap_dev, int H, int W, int64_t known_count);
// insertion of already packed float4 points (nullable) whose count the host knows
// The update as the device decided it (*upd, written on the map stream's side of an event before the launches run).
// kdmap_device_update_bound: the point count the launches are sized for -- the map's count + new_bound new points,
// clamped to the capacity already planned -- or 0 when the update has to stay on the host's path (a first insertion, a
// generation restart).  The device closes the update's gate when the new count exceeds the bound, and the host then
// decides and enqueues that update itself, re-planning the capacity as it always did: capacity and index geometry come
// out as a host-decided update plans them.  kdmap_settle_device_update: the host mirror (counts, the per-frame counts,
// the index size) once *upd is back on the host with the gate open.
int64_t kdmap_device_update_bound(const pls_context* ctx, int64_t new_bound);
void kdmap_update_on_device(pls_context* ctx, const float4* fresh_dev, int64_t bound, const KdUpdateWords* upd);
void kdmap_settle_device_update(pls_context* ctx, const KdUpdateWords& w, int local_map_size);
void kdmap_update_packed(pls_context* ctx, const float* rel_pose_host, const float4* fresh_dev, int64_t num_new,
                         bool has_new);
// pls_process_frames: the ICP of `num` sequences (distinct kd-map contexts, no communicator) in batched launches on st.
// begin uploads their descriptors into lead->batch_buf and returns the launch widths in grid[KD_BATCH_GRID]; iterations enqueues
// ICP iterations [first, last) of all of them; done reads every sequence's done flag with one copy and one sync.
constexpr int KD_BATCH_GRID = 6;
void kdmap_batch_begin(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                       int* grid);
// max_distance (pls_register_scans_gated, registrations only): finite, the iterations run the gated kernels with that
// gate (KdGate); +inf, the ungated ones.  min_eigenvalue > 0 (pls_register_scans_degeneracy, registrations only): the
// gated kernels' twins with the eigenvalue-thresholded solve, at any max_distance; registration j of the batch writes
// its eigenvalues and degenerate count to degen + ICP_DEGEN_STRIDE j (icp_device.cuh).
void kdmap_batch_iterations(pls_context* lead, int num, cudaStream_t st, const int* grid, int first, int last,
                            double max_distance = HUGE_VAL, double min_eigenvalue = 0.0, double* degen = nullptr);
void kdmap_batch_done(pls_context* lead, int num, cudaStream_t st, int* out);
// The scan one registration of pls_register_hypotheses / pls_register_scans reads: its packed float4 queries, their
// count on the device (u32) and the query bound of its single pls_register_frame call (the scan's row count).
struct KdScan {
    const float4* queries;
    const uint32_t* nq_dev;
    int64_t bound;
};
// pls_register_hypotheses / pls_register_scans: `num` <= PLS_MAX_SEQUENCES registrations on ctx's map, registration h of
// scans[h], driven by kdmap_batch_iterations / kdmap_batch_done with lead = ctx.  begin returns their FrameResults and
// 16 counter and work-list words each (for the caller to initialise, as frame_begin does); adopt makes registration h,
// of scan `scan`, ctx's last search: its matches, search states, FrameResult, query count and queries.
void kdmap_hypotheses_begin(pls_context* ctx, const KdScan* scans, int num, cudaStream_t st, int* grid, FrameResult** frs,
                            uint32_t** words);
void kdmap_hypothesis_adopt(pls_context* ctx, const KdScan& scan, int h, cudaStream_t st);
// pls_kdmap_evaluate_poses: after kdmap_hypotheses_begin and the registrations' start at their poses, iteration 0's
// 1-NN and normals, then the residual pass gated by max_d2 and no solve; registration h's row of PLS_EVAL_STATS
// doubles into out[PLS_EVAL_STATS h] (device), its entries 0..29 also into its FrameResult's last_sums.  Enqueued on st.
void kdmap_evaluate_batch(pls_context* ctx, int num, cudaStream_t st, const int* grid, double max_d2, double* out);
// pls_register_scans: one scan to pack, its device rows [n,3] (n > 0) and where its valid rows and their count go.
struct KdScanRows {
    const float* rows;
    int64_t n;
    float4* out;
    uint32_t* count;
};
// One launch packs every scan, each as pack_valid_rows packs it alone.
void pack_valid_scans(pls_context* ctx, const std::vector<KdScanRows>& scans);
// ICP iteration `it` of the frame over ctx->query_ptr; returns the number of partial rows written
// it == 0: no previous matches; fuse_threshold >= 0: finish the iteration (sum + solve + pose update) in the last
// block of the reduction kernel (*solved tells).  bound_dev (nullable, unsharded frames only): a device-side count that
// tightens query_bound; the kernels then use the block count of min(query_bound, *bound_dev) queries, and the returned
// count is the launched one, that of query_bound.
int kdmap_icp_iteration(pls_context* ctx, int64_t query_bound, const uint32_t* bound_dev, int rank, int num_ranks, int it,
                        float fuse_threshold, bool* solved);
// pack [n,3] rows without NaN into float4 (stable); count -> *count_dev (u32)
void pack_valid_rows(pls_context* ctx, const float* pts_dev, int64_t n, float4* out, uint32_t* count_dev);
void pack_valid_rows_f64(pls_context* ctx, const double* pts_dev, int64_t n, float4* out, uint32_t* count_dev);
// pack the pixels of a [3,H,W] map with |p| > min_norm (NaN dropped) into float4, row-major order
void pack_valid_pixels(pls_context* ctx, const float* vmap_dev, int64_t hw, float min_norm, float4* out,
                       uint32_t* count_dev);
// grid_sample.cu
// A grid sample whose sample count the host reads back: xyz [n,3] (float64 if f64, else float32) -> out_xyz [<=n,3] and
// out_idx [<=n] (nullable) on the device; with host_xyz and host_idx (device aliases of mapped pinned memory) the
// gather also writes a host copy.
struct GridSample {
    const void* xyz;
    bool f64;
    int64_t n;
    double voxel;
    void* out_xyz;
    long long* out_idx;
    void* host_xyz;
    long long* host_idx;
};
// The sample runs in two halves on ctx->stream, so that a caller can synchronise once for several contexts.  enqueue
// sorts on 40-bit keys (5 radix passes instead of 8), exact whenever every hash lies in [-2^39, 2^39), i.e. voxel
// coordinates up to ~3 000 000 in magnitude, and copies the count and the overflow stamp to the host.  finish, once
// ctx->stream has been synchronised, returns the count; if a hash overflowed the compact keys it first samples once more
// on the raw 64-bit keys and reads that count (one more copy and stream synchronisation).
// count_to_host = false leaves the count and the stamp in the device scalars (SC_GS_COUNT, SC_GS_OVERFLOW) for a caller
// that copies them back later with its own result (the FrameResult copy covers both); grid_sample_host_count then reads
// them from that copy.
void grid_sample_enqueue(pls_context* ctx, const GridSample& g, bool count_to_host = true);
uint32_t grid_sample_finish(pls_context* ctx, const GridSample& g);
uint32_t grid_sample_host_count(pls_context* ctx, bool* overflowed);
// projmap.cu
void projmap_reset(pls_context* ctx);
// pls_process_frames on projective maps, the counterparts of kdmap_batch_*: begin uploads the descriptors into
// lead->batch_buf and returns the launch widths and the TMA kernel's dynamic shared memory in grid[4]; iterations
// enqueues ICP iterations [first, last) of all of them, solve included; done reads every sequence's done flag.
void projmap_batch_begin(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                         int* grid);
void projmap_batch_iterations(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                              const int* grid, int first, int last);
void projmap_batch_done(pls_context* lead, int num, cudaStream_t st, int* out);
// pls_register_hypotheses on a projective map: `num` <= PLS_MAX_SEQUENCES hypotheses of the scan in ctx->query_ptr on
// ctx's model, driven by projmap_hypotheses_iterations and projmap_batch_done with lead = ctx.  begin returns their
// FrameResults and 16 words each (for hypotheses_begin_kernel); adopt makes hypothesis h ctx's last ICP result.
void projmap_hypotheses_begin(pls_context* ctx, int num, cudaStream_t st, FrameResult** frs, uint32_t** words);
void projmap_hypotheses_iterations(pls_context* ctx, int64_t query_bound, int num, cudaStream_t st, int first, int last);
void projmap_hypothesis_adopt(pls_context* ctx, int h, cudaStream_t st);
// odometry.cu: would an ICP iteration over `work` items be split across the ranks (the rule of enqueue_icp_iterations)?
bool icp_shards(pls_context* ctx, int64_t work);
// comm.cu
int comm_rank(pls_context* ctx);
int comm_size(pls_context* ctx);
void projmap_update(pls_context* ctx, const float* rel_pose_host, const float* vmap_dev);
// odometry.cu
void odometry_reset(pls_context* ctx);
// comm.cu
void comm_allreduce_sums(pls_context* ctx, double* sums_dev);
void comm_free(pls_context* ctx);

}  // namespace pls
