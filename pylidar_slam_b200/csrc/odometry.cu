// The frame-to-model ICP odometry state machine (replaces ICPFrameToModel,
// slam/odometry/icp_odometry.py:72-380) driven from the host with NO per-iteration host sync:
// every ICP iteration is {correspondence+reduction kernel, [allreduce], icp_step_kernel}; the
// convergence test (icp_odometry.py:292), the Gauss-Newton guards (optimization.py:323-336) and
// the pose composition with its Euler round trip (icp_odometry.py:296-297) run on the device
// and latch a `done` flag that turns the remaining launches of the frame into no-ops.
// One device->host copy of the FrameResult ends the frame.
#include <stdlib.h>

#include <chrono>
#include <functional>
#include <optional>
#include <utility>
#include <vector>

#include "internal.cuh"
#include "icp_device.cuh"
#include "pose_device.cuh"
#include "projection_device.cuh"
#include "select_device.cuh"

namespace pls {

// projmap.cu
int projmap_icp_iteration(pls_context* ctx, int64_t query_bound, int rank, int num_ranks);
// comm.cu
int comm_rank(pls_context* ctx);
int comm_size(pls_context* ctx);
bool comm_is_p2p(pls_context* ctx);
void* comm_p2p_peers(pls_context* ctx);
unsigned long long* comm_p2p_seq(pls_context* ctx);
double* comm_allreduce_buffer(pls_context* ctx);

namespace {

int64_t g_shard_min_override = -1;  // pls_set_shard_min
int64_t shard_min_default() {
    static const int64_t v = getenv("PLS_SHARD_MIN") ? atoll(getenv("PLS_SHARD_MIN")) : 24576;
    return v;
}

struct Pose16 {
    float m[16];
};

// The start of a frame's ICP.  The initial pose is T0_dev if given, else T0 (a kernel argument: no copy in front of the
// kernel).  The frame's counts: the input stage wrote the low words of counts[1] (queries; copied from counts[2] here
// when the queries are the valid rows themselves) and counts[2] (valid rows); every other word is cleared.
__device__ __forceinline__ void frame_begin_body(FrameResult* fr, const float* T0_dev /*16, or null*/, const Pose16& T0,
                                                 uint32_t* worklist_counts /*16*/, int queries_are_rows) {
    int t = threadIdx.x;
    if (t < 16) worklist_counts[t] = 0;  // SC_KD_COUNTERS + SC_KD_LISTS: the kd search's counters and work lists
    if (t < 16) fr->T[t] = T0_dev ? T0_dev[t] : T0.m[t];
    uint32_t* cw = reinterpret_cast<uint32_t*>(fr->counts);  // word 2i: the low half of counts[i]
    static_assert(sizeof(fr->counts) == 16 * sizeof(uint32_t), "counts: 8 words of 64 bits");
    if (t < 16 && t != 2 && t != 4) cw[t] = 0u;
    if (t == 2 && queries_are_rows) cw[2] = cw[4];
    if (t < 6) fr->params[t] = 0.f;
    if (t < kMaxAlign) fr->losses[t] = __int_as_float(0x7fc00000);
    if (t == 0) {
        fr->iters = 0;
        fr->status = 0;
        fr->done = 0;
        fr->pad = 0;  // last-block ticket of the fused correspondence+solve kernels
    }
    if (t < NACC) fr->last_sums[t] = 0.0;
}

__global__ void frame_begin_kernel(FrameResult* fr, const float* T0_dev /*16, or null*/, Pose16 T0, int max_iters,
                                   uint32_t* worklist_counts /*16*/, int queries_are_rows) {
    frame_begin_body(fr, T0_dev, T0, worklist_counts, queries_are_rows);
}

// pls_register_hypotheses: block h starts hypothesis h at T0s[16 h], as frame_begin_kernel starts a frame.
__global__ void hypotheses_begin_kernel(FrameResult* frs, const float* __restrict__ T0s, uint32_t* words) {
    frame_begin_body(frs + blockIdx.x, T0s + 16 * blockIdx.x, Pose16{}, words + 16 * blockIdx.x, 0);
}


// NCCL mode, before the all-reduce: this rank's sums go to the exchange buffer `out` (not into the FrameResult: the
// all-reduce runs in place, and launches enqueued after convergence must leave the frame's result alone).
__global__ void __launch_bounds__(256) reduce_partials_kernel(const FrameResult* fr, const double* __restrict__ partials,
                                                              int num_blocks, double* __restrict__ out) {
    if (fr->done) return;
    __shared__ double sums[NACC];
    sum_partials_256(partials, num_blocks, sums);
    __syncthreads();
    if (threadIdx.x < NACC) out[threadIdx.x] = sums[threadIdx.x];
}

// K7: normal-equation solve + ICP bookkeeping (256 threads).  num_blocks == 0: `reduced` holds the (all-reduced) sums.
__global__ void __launch_bounds__(256) icp_step_kernel(FrameResult* fr, const double* __restrict__ partials,
                                                       int num_blocks, const double* __restrict__ reduced, float threshold_delta) {
    icp_step_body(fr, partials, num_blocks, reduced, threshold_delta);
}

// K9 fused: block-partial sum + ONE-SHOT all-reduce over NVLink peer memory + solve, in one kernel.
// Every rank owns an exchange buffer mapped into all peers (CUDA IPC): slot[parity][r] is written by rank r.
// A rank stores its 30 sums into slot[parity][me] of EVERY peer (plain stores to peer-mapped addresses), fences
// system-wide, then stores the launch's sequence number; it then spins on its LOCAL slots until all peers'
// sequence numbers arrived and adds the slots in rank order -- the same order on every rank, so all ranks
// obtain bit-identical sums and hence bit-identical poses without any broadcast.  Two parities make the
// overwrite of a slot wait for a full further round.  The spin is bounded: a peer that never shows up turns
// into PLS_E_COMM instead of a hang.
struct P2PSlot {
    double sums[NACC];
    unsigned long long seq;
    unsigned long long pad;
};
static_assert(sizeof(P2PSlot) == 256, "P2PSlot must match comm.cu's kP2PSlotBytes");
__global__ void __launch_bounds__(256)
icp_step_p2p_kernel(FrameResult* fr, const double* __restrict__ partials, int num_blocks, float threshold_delta,
                    P2PSlot* const* __restrict__ peers, int world, int rank, unsigned long long* seq_counter) {
    if (fr->done) return;
    __shared__ double sums[NACC];
    __shared__ int timed_out;
    __shared__ unsigned long long s_seq;
    if (threadIdx.x == 0) {
        timed_out = 0;
        s_seq = ++(*seq_counter);  // this exchange's round
    }
    sum_partials_256(partials, num_blocks, sums);
    __syncthreads();
    const unsigned long long seq = s_seq;
    const int parity = (int)(seq & 1ull);
    if (threadIdx.x < NACC)
        for (int r = 0; r < world; ++r) peers[r][parity * world + rank].sums[threadIdx.x] = sums[threadIdx.x];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) {
        volatile unsigned long long* flag = &peers[threadIdx.x][parity * world + rank].seq;
        *flag = seq;
    }
    if (threadIdx.x < world) {
        volatile unsigned long long* mine = &peers[rank][parity * world + threadIdx.x].seq;
        const long long t0 = clock64();
        while (*mine < seq) {
            if (clock64() - t0 > 6000000000ll) {  // ~3 s: a peer is gone
                timed_out = 1;
                break;
            }
        }
    }
    __threadfence_system();
    __syncthreads();
    if (timed_out) {
        if (threadIdx.x == 0) {
            fr->status = PLS_E_COMM;
            fr->done = 1;
        }
        return;
    }
    if (threadIdx.x < NACC) {
        double s = 0.0;
        for (int r = 0; r < world; ++r) s += __ldcv(&peers[rank][parity * world + r].sums[threadIdx.x]);
        sums[threadIdx.x] = s;
        fr->last_sums[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    icp_solve_and_update(fr, sums, threshold_delta);
}

__global__ void scrub_vertex_map_kernel(const float* __restrict__ in, int64_t hw, float* __restrict__ out) {
    // modify_nan_pmap (utils.py:187-196): a pixel with any NaN channel becomes 0
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x) {
        float x = in[i], y = in[hw + i], z = in[2 * hw + i];
        bool bad = !(x == x) || !(y == y) || !(z == z);
        out[i] = bad ? 0.f : x;
        out[hw + i] = bad ? 0.f : y;
        out[2 * hw + i] = bad ? 0.f : z;
    }
}

__global__ void first_point_kernel(const float4* __restrict__ packed, const uint32_t* __restrict__ count,
                                   float4* __restrict__ out, uint32_t* __restrict__ out_count, FrameResult* fr) {
    // reference quirk (icp_odometry.py:342-344,356-358): with a vertex-map input `_tgt_pc` keeps
    // only the first non-null pixel
    if (threadIdx.x == 0) {
        uint32_t c = *count;
        if (c > 0) {
            out[0] = packed[0];
            fr->first_pt[0] = packed[0].x; fr->first_pt[1] = packed[0].y; fr->first_pt[2] = packed[0].z;
        }
        *out_count = c > 0 ? 1u : 0u;
    }
}

// _read_input + sample_points of a float32 point layout on the kd map after frame 0, in one selection pass over the
// input rows (select_device.cuh): the NaN-free rows (utils.py:169-184) are packed as float4 -- the points the map
// update inserts -- and, when the queries are the non-null pixels of the cloud's vertex map (icp_odometry.py:303-305),
// the rows that won their pixel of the z-buffer (closest point, lowest index on ties: projection.py:393-415) are packed
// as the queries.  The vertex map itself is never materialised: its non-null pixels ARE the winners.  (The queries come
// out in input order rather than pixel order; the reduction over them is order-independent up to fp64 rounding.)
// Each winner also resets its pixel, which leaves the z-buffer empty for the next frame.
struct FrameInputSelect {
    const float* pts;
    ProjConst pc;
    unsigned long long* zbuf;   // null: no query selection (queries = the valid rows)
    float4* frame_pts;
    float4* queries;
    struct State {
        float x, y, z;
        int pix;
    };
    __device__ __forceinline__ uint32_t flags(int64_t i, State& s) const {
        s.x = pts[3 * i];
        s.y = pts[3 * i + 1];
        s.z = pts[3 * i + 2];
        s.pix = -1;
        const bool valid = s.x == s.x && s.y == s.y && s.z == s.z;
        if (!valid) return 0u;
        uint32_t f = 1u;
        if (zbuf) {
            int pix;
            float r;
            // zbuf_points_kernel's order: a range one ulp off would drop this query
            if (project_to_pixel(s.x, s.y, s.z, pc, pix, r, RangeOrder::kYFirst) &&
                zbuf[pix] == (((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)i)) {
                s.pix = pix;
                f |= 2u;
            }
        }
        return f;
    }
    __device__ __forceinline__ void emit(int64_t, int which, uint32_t pos, const State& s) const {
        if (which == 0) {
            frame_pts[pos] = make_float4(s.x, s.y, s.z, 0.f);
        } else {
            queries[pos] = make_float4(s.x, s.y, s.z, 0.f);
            zbuf[s.pix] = ~0ull;
        }
    }
};

}  // namespace

bool icp_shards(pls_context* ctx, int64_t work) {
    const int size = comm_size(ctx);
    int64_t shard_min = g_shard_min_override >= 0 ? g_shard_min_override : shard_min_default();
    // a query against a multi-million-point kd map walks cold cell tables and misses L2: a third of the usual share
    // already outweighs the exchange (BASELINE config 4: 131 k queries, 5 M points, still split at 8 ranks)
    if (g_shard_min_override < 0 && ctx->cfg.local_map_type == PLS_MAP_KDTREE && ctx->kd.indexed >= 2000000) shard_min /= 3;
    return size > 1 && work / size >= shard_min;
}

namespace {

inline int grid_for(int64_t n, int threads = 256) {
    int64_t b = (n + threads - 1) / threads;
    int64_t cap = 8 * kNumSMs;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

uint32_t* count_slot(pls_context* ctx, int i) { return reinterpret_cast<uint32_t*>(&frame_result_dev(ctx)->counts[i]); }

// Enqueues ICP iterations [first, last) (icp_odometry.py:274-297).  bound_dev: see kdmap_icp_iteration.
int enqueue_icp_iterations(pls_context* ctx, int64_t query_bound, const uint32_t* bound_dev, int first, int last) {
    cudaStream_t st = ctx->stream;
    FrameResult* fr = frame_result_dev(ctx);
    int rank = comm_rank(ctx), size = comm_size(ctx);
    // Sharding pays only when a rank's share of the correspondences outweighs the exchange it buys: below
    // PLS_SHARD_MIN work items (queries / pixels) per rank every rank runs the whole iteration itself -- same inputs,
    // same deterministic kernels, hence the same bits on every rank, and no exchange at all.  (The bound is a host
    // value every rank computes alike, so the ranks always take the same branch.)
    if (size > 1) {
        PLS_REQUIRE(!bound_dev, "ICP: a device-side query bound cannot decide the sharding");
        const int64_t work = ctx->cfg.local_map_type == PLS_MAP_KDTREE ? query_bound : (int64_t)ctx->cfg.height * ctx->cfg.width;
        if (!icp_shards(ctx, work)) {
            rank = 0;
            size = 1;
        }
    }
    ctx->last_sharded = size > 1;
    int last_blocks = 0;
    for (int it = first; it < last; ++it) {
        int blocks;
        bool solved = false;  // the kd kernels finish the iteration themselves on a single GPU
        if (ctx->cfg.local_map_type == PLS_MAP_KDTREE)
            blocks = kdmap_icp_iteration(ctx, query_bound, bound_dev, rank, size, it,
                                         size == 1 ? ctx->cfg.threshold_delta_pose : -1.f, &solved);
        else
            blocks = projmap_icp_iteration(ctx, query_bound, rank, size);
        last_blocks = blocks;
        if (solved) continue;
        if (size > 1 && comm_is_p2p(ctx)) {
            icp_step_p2p_kernel<<<1, 256, 0, st>>>(fr, ctx->partials.as<double>(), blocks, ctx->cfg.threshold_delta_pose,
                                                   (P2PSlot* const*)comm_p2p_peers(ctx), size, rank, comm_p2p_seq(ctx));
            PLS_CHECK_LAUNCH();
            continue;
        }
        const double* reduced = nullptr;
        if (size > 1) {
            double* buf = comm_allreduce_buffer(ctx);
            reduce_partials_kernel<<<1, 256, 0, st>>>(fr, ctx->partials.as<double>(), blocks, buf);
            PLS_CHECK_LAUNCH();
            comm_allreduce_sums(ctx, buf);
            reduced = buf;
            blocks = 0;
        }
        icp_step_kernel<<<1, 256, 0, st>>>(fr, ctx->partials.as<double>(), blocks, reduced, ctx->cfg.threshold_delta_pose);
        PLS_CHECK_LAUNCH();
    }
    return last_blocks;
}

// __update_map's key-frame decision (keyframe_decision) and the move of the map (kdmap_update_packed) on the device,
// one thread, behind a frame's ICP launches: the map update can then be enqueued before the host has seen the pose.
// The float and double arithmetic is that of the host code, rounded operation by operation (__fmul_rn & co.: no
// contraction into FMAs, which the host build does not do either), so that the move X and the new delta are the host's
// bits.  The decision also goes through atan2f, whose device result may differ from glibc's by a few ulp (CUDA documents
// a 3-ulp bound): a decision can only differ from the host's when the rotation angle lies within a few ulp of
// threshold_rot.
// The gate opens when the frame needs no further ICP launches (done, or max_num_alignments iterations), its ICP did not
// fail, its grid sample's compact keys did not overflow (gs_overflow: the stamp word, or null), and the new map count
// fits total_limit, the count the update's launches are sized for; while it is closed every count is 0 and the update's
// launches do nothing.
__device__ __forceinline__ void mat4_mul_rn(const float* A, const float* B, float* C) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float s = 0.f;
            for (int k = 0; k < 4; ++k) s = __fadd_rn(s, __fmul_rn(A[i * 4 + k], B[k * 4 + j]));
            C[i * 4 + j] = s;
        }
}

__device__ __forceinline__ float norm3_rn(float a, float b, float c) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c)));
}

__global__ void kd_update_decision_kernel(const FrameResult* __restrict__ fr, KdUpdateWords* __restrict__ w, Pose16 delta,
                                          float threshold_trans, float threshold_rot, int max_num_alignments,
                                          uint32_t map_count, uint32_t evict_count, uint32_t total_limit,
                                          const uint32_t* __restrict__ gs_overflow, uint32_t gs_seq) {
    const bool failed = fr->status == PLS_E_SINGULAR || fr->status == PLS_E_COMM;
    const bool ready = (fr->done || fr->iters >= max_num_alignments) && !failed && !(gs_overflow && *gs_overflow == gs_seq);
    float T[16];
    for (int i = 0; i < 16; ++i) T[i] = fr->T[i];
    // keyframe_decision: the accumulated motion nd = delta T, its translation and Euler-angle norms
    float nd[16];
    mat4_mul_rn(delta.m, T, nd);
    float sy = __fsqrt_rn(__fadd_rn(__fmul_rn(nd[0], nd[0]), __fmul_rn(nd[4], nd[4])));
    float e[3];  // mat_to_euler
    if (!(sy < 1e-6f)) {
        e[0] = atan2f(nd[9], nd[10]);
        e[1] = atan2f(-nd[8], sy);
        e[2] = atan2f(nd[4], nd[0]);
    } else {
        e[0] = atan2f(-nd[6], nd[5]);
        e[1] = atan2f(-nd[8], sy);
        e[2] = 0.f;
    }
    const float tn = norm3_rn(nd[3], nd[7], nd[11]);
    const float rn = norm3_rn(e[0], e[1], e[2]);
    bool insert = ready && (tn > threshold_trans ||
                            __fdiv_rn(__fmul_rn(rn, 180.0f), 3.14159265358979323846f) > threshold_rot);
    // the new count: kdmap_update_packed's kept + num_new (a larger one is left to the host, which re-plans the capacity)
    const bool gate = ready && map_count - (insert ? evict_count : 0u) + (insert ? (uint32_t)fr->counts[2] : 0u) <= total_limit;
    insert = insert && gate;
    // rigid_inverse(T): (R^T, -R^T t) in double
    const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    const double t[3] = {T[3], T[7], T[11]};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) w->X[3 * i + j] = (float)R[j * 3 + i];
        w->X[9 + i] = __double2float_rn(
            -__dadd_rn(__dadd_rn(__dmul_rn(R[i], t[0]), __dmul_rn(R[3 + i], t[1])), __dmul_rn(R[6 + i], t[2])));
    }
    for (int i = 0; i < 16; ++i) w->delta[i] = !gate ? delta.m[i] : (insert ? ((i % 5 == 0) ? 1.f : 0.f) : nd[i]);
    const uint32_t num_new = insert ? (uint32_t)fr->counts[2] : 0u;
    const uint32_t skip = insert ? evict_count : 0u;
    w->gate = gate ? 1u : 0u;
    w->insert = insert ? 1u : 0u;
    w->skip = gate ? skip : 0u;
    w->kept = gate ? map_count - skip : 0u;
    w->num_new = num_new;
    w->total = gate ? map_count - skip + num_new : 0u;
}

// PLS_HOST_TRACE=1: host-side time of the phases of a frame (the grid-sampled call's prologue: a deferred map-update
// enqueue, then the grid-sample enqueue; the enqueue of the input stage and the ICP, the wait for the pose, the map
// update: its enqueue behind the ICP when the device decides it, else the host's decision), averaged and printed every
// 64 frames -- a development aid for the end-to-end path.
struct HostTrace {
    bool on = getenv("PLS_HOST_TRACE") != nullptr;
    bool in_call = false;  // begin_call() ran: process_frame_device closes the prologue lap instead of starting afresh
    double acc[6] = {0, 0, 0, 0, 0, 0};
    int frames = 0, extra_rounds = 0;
    std::chrono::steady_clock::time_point t;
    void start() { if (on) t = std::chrono::steady_clock::now(); }
    void begin_call() {
        start();
        in_call = on;
    }
    void frame_start() {  // the start of process_frame_device
        if (in_call) lap(5);
        else start();
        in_call = false;
    }
    void lap(int k) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        acc[k] += std::chrono::duration<double, std::micro>(now - t).count();
        t = now;
    }
    void end_frame() {
        if (!on || ++frames < 64) return;
        fprintf(stderr, "[plslam_b200 host trace] per frame: call prologue: map-update flush %.1f us, grid-sample "
                        "enqueue %.1f us; enqueue input+ICP %.1f us, wait for the pose %.1f us, map update %.1f us, "
                        "rest %.1f us; %d of %d frames needed a second round of ICP launches\n",
                acc[4] / frames, acc[5] / frames, acc[0] / frames, acc[1] / frames, acc[2] / frames, acc[3] / frames,
                extra_rounds, frames);
        frames = 0;
        extra_rounds = 0;
        for (double& a : acc) a = 0;
    }
};
HostTrace g_trace;

// PLS_BATCH_TRACE=<file>: one JSON line per pls_process_frames call, appended to <file> -- CUDA-event times on the lead
// stream of the input stage (call start until every sequence's input stage is done) and of the batched ICP (until the
// FrameResults are copied back), the host time of the epilogue and of the whole call, and the extra ICP rounds.
// A development aid for the per-phase split of a batched step (tools/multi_sequence_bench.py --phases).
struct BatchTrace {
    const char* path = nullptr;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    std::chrono::steady_clock::time_point t_call, t_epi;
    int sequences = 0, icp_sequences = 0, extra_rounds = 0;
    void begin(cudaStream_t st) {
        path = getenv("PLS_BATCH_TRACE");
        if (!path) return;
        t_call = std::chrono::steady_clock::now();
        for (auto& e : ev) PLS_CUDA(cudaEventCreate(&e));
        PLS_CUDA(cudaEventRecord(ev[0], st));
    }
    void inputs_done(cudaStream_t st, int num, int icp) {
        sequences = num;
        icp_sequences = icp;
        if (path) PLS_CUDA(cudaEventRecord(ev[1], st));
    }
    void icp_done(cudaStream_t st) {
        if (path) PLS_CUDA(cudaEventRecord(ev[2], st));
    }
    void epilogue_begin() {
        if (path) t_epi = std::chrono::steady_clock::now();
    }
    void end() {
        if (!path) return;
        const auto now = std::chrono::steady_clock::now();
        float input_ms = 0.f, icp_ms = 0.f;
        PLS_CUDA(cudaEventSynchronize(ev[1]));
        PLS_CUDA(cudaEventElapsedTime(&input_ms, ev[0], ev[1]));
        if (icp_sequences > 0) PLS_CUDA(cudaEventElapsedTime(&icp_ms, ev[1], ev[2]));
        FILE* f = fopen(path, "a");
        if (!f) return;
        fprintf(f, "{\"sequences\": %d, \"icp_sequences\": %d, \"input_ms\": %.6f, \"icp_ms\": %.6f, \"epilogue_ms\": %.6f, "
                   "\"call_ms\": %.6f, \"extra_rounds\": %d}\n",
                sequences, icp_sequences, input_ms, icp_ms,
                std::chrono::duration<double, std::milli>(now - t_epi).count(),
                std::chrono::duration<double, std::milli>(now - t_call).count(), extra_rounds);
        fclose(f);
    }
    ~BatchTrace() {
        for (auto e : ev)
            if (e) cudaEventDestroy(e);
    }
};

// The start of a frame's ICP: the FrameResult at T0 (T0_dev on the device, else T0_host, else the identity), the search
// counters cleared.
void frame_begin(pls_context* ctx, const float* T0_host, const float* T0_dev, bool queries_are_rows) {
    Pose16 T0;
    for (int i = 0; i < 16; ++i) T0.m[i] = T0_host ? T0_host[i] : ((i % 5 == 0) ? 1.f : 0.f);
    frame_begin_kernel<<<1, kMaxAlign, 0, ctx->stream>>>(frame_result_dev(ctx), T0_dev, T0, ctx->cfg.max_num_alignments,
                                                         scalar_u32(ctx, SC_KD_COUNTERS), queries_are_rows ? 1 : 0);
    PLS_CHECK_LAUNCH();
}

// The ICP rounds (icp_odometry.py:248-299) of the frames of ctxs[0, num), after their frame_begin.  Iterations are
// enqueued without host syncs and turn into no-ops once a frame's device-side `done` flag latches.  To avoid paying for
// max_num_alignments launches when ICP converges in 2-3, only the previous frame's count + 1 are enqueued up front (the
// most any of the frames asks for); while a frame has not latched `done` and may iterate further, up to 4 more follow
// each host look at the flags (rare: one extra sync per round).
// enqueue(first, last) enqueues iterations [first, last) of every frame; read_done(done) waits for the enqueued work and
// stores each frame's done flag.  Returns the number of extra rounds.
template <typename Enqueue, typename ReadDone>
int icp_rounds(pls_context* const* ctxs, int num, Enqueue enqueue, ReadDone read_done) {
    int upfront = 0, max_it = 0;
    for (int j = 0; j < num; ++j) {
        const int last = ctxs[j]->last_icp_iters, m = ctxs[j]->cfg.max_num_alignments;
        const int u = last > 0 && last + 1 < m ? last + 1 : m;
        upfront = u > upfront ? u : upfront;
        max_it = m > max_it ? m : max_it;
    }
    enqueue(0, upfront);
    int enq = upfront, extra = 0;
    int done[PLS_MAX_SEQUENCES];
    while (enq < max_it) {
        read_done(done);
        bool more = false;
        for (int j = 0; j < num; ++j) more = more || (!done[j] && enq < ctxs[j]->cfg.max_num_alignments);
        if (!more) break;
        const int k = (max_it - enq) < 4 ? (max_it - enq) : 4;
        enqueue(enq, enq + k);
        enq += k;
        extra += 1;
    }
    return extra;
}

// The FrameResult and the u32 / u64 scalar slots behind it in one copy to the pinned host mirror, on st.
void enqueue_result_copy(pls_context* ctx, cudaStream_t st) {
    PLS_CUDA(cudaMemcpyAsync(ctx->pinned.p, ctx->scalars.p, kScalarOffset + SC_NUM * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                             st));
}

void fetch_result(pls_context* ctx) {
    enqueue_result_copy(ctx, ctx->stream);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
}

// The ICP loop of one frame over ctx->query_ptr / counts[1], on ctx->stream, up to the host copy of its result.
// after_upfront (may be empty) is enqueued behind the up-front launches, before the host first waits.  Each look at the
// done flag copies the whole result, so a frame that needs no second round of launches costs the host one wait.
// Returns the launched block count of the correspondence kernel; *extra_rounds: the rounds of launches after the first.
int run_icp(pls_context* ctx, int64_t query_bound, const uint32_t* bound_dev, const std::function<void()>& after_upfront,
            int* extra_rounds) {
    if (query_bound < 1) query_bound = 1;
    ctx->pm.zbuf_clean = false;  // tmp[3] may have been used by the frame's own projection
    int blocks = 0;
    bool fresh = false;  // the host copy holds the result of every launch enqueued so far
    auto enqueue = [&](int first, int last) {
        blocks = enqueue_icp_iterations(ctx, query_bound, bound_dev, first, last);
        fresh = false;
        if (first == 0) {
            g_trace.lap(0);
            if (after_upfront) {
                after_upfront();
                g_trace.lap(2);
            }
        }
    };
    auto read_done = [&](int* done) {
        fetch_result(ctx);
        fresh = true;
        done[0] = frame_result_host(ctx)->done;
    };
    *extra_rounds = icp_rounds(&ctx, 1, enqueue, read_done);
    g_trace.extra_rounds += *extra_rounds;
    if (*extra_rounds > 0 && after_upfront) {  // behind the last round: the update's gate opens this time
        after_upfront();
        fresh = false;
    }
    if (!fresh) fetch_result(ctx);
    return blocks;
}

// Algorithmic bytes of the frame's executed ICP iterations, by SURVEY.md 8d's formulas.
// kd map:  K5a exact 1-NN    per query 12 B (query) + 27 * 8 B (cell-range lookups) + 4 B (match), plus 16 B per
//                            candidate actually tested (counted by the kernel);
//          K5b/c normals     per computed normal 16 B (point) + 16 B (normal written), plus 16 B per candidate tested;
//          K6 reduction      per correspondence 36 B, plus one 30-double partial row per block.
// (bench.py also reports the lower bound SURVEY names: 44 B per query + 16 B per touched map point.)
void credit_icp_profile(pls_context* ctx, const FrameResult* h, int blocks) {
    if (ctx->cfg.local_map_type == PLS_MAP_KDTREE) {
        const unsigned long long* kc = reinterpret_cast<const unsigned long long*>(
            reinterpret_cast<const char*>(h) + kScalarOffset + SC_KD_COUNTERS * sizeof(uint32_t));
        // a rank of a sharded frame handles its share of the queries (the counters already are per rank)
        const double iters = (double)h->iters, nq = (double)h->counts[1] / (ctx->last_sharded ? (double)comm_size(ctx) : 1.0);
        const double bytes = iters * nq * (12.0 + 27.0 * 8.0 + 4.0) + 16.0 * (double)kc[0]      // K5a
                             + 32.0 * (double)kc[2] + 16.0 * (double)kc[1]                      // K5b/c
                             + iters * (nq * 36.0 + (double)blocks * NACC * 8.0);               // K6
        profile_credit(ctx, 0, h->iters, bytes);
    } else {
        // projective map (SURVEY 8d): HW*12*(K+1) (target + K candidate vertex maps, each read once)
        // + N_c*12 (winner normals) + one partial row per block
        // a rank of a sharded frame streams its share of the tiles
        const double share = ctx->last_sharded ? 1.0 / (double)comm_size(ctx) : 1.0;
        const double hw = (double)ctx->cfg.height * ctx->cfg.width * share;
        profile_credit(ctx, 1, h->iters, (double)h->iters * (hw * 12.0 * (ctx->pm.K + 1) + h->last_sums[29] * share * 12.0 +
                                                              (double)blocks * NACC * 8.0));
    }
}

void raise_status(pls_context* ctx, int status) {
    if (status == PLS_E_COMM) throw pls::Error{PLS_E_COMM, "peer-to-peer all-reduce timed out waiting for a peer rank"};
    if (status == PLS_E_SINGULAR) throw pls::Error{PLS_E_SINGULAR, "Invalid Jacobian in Gauss Newton minimization"};
}

// __update_map (icp_odometry.py:360-380), host side: key-frame policy on the accumulated motion.
bool keyframe_decision(pls_context* ctx, const float* T) {
    float nd[16], prm[6];
    mat4_mul(ctx->delta_since_update, T, nd);
    from_pose(nd, prm);
    const float tn = sqrtf(prm[0] * prm[0] + prm[1] * prm[1] + prm[2] * prm[2]);
    const float rn = sqrtf(prm[3] * prm[3] + prm[4] * prm[4] + prm[5] * prm[5]);
    const bool insert = tn > ctx->cfg.threshold_trans || rn * 180.0f / 3.14159265358979323846f > ctx->cfg.threshold_rot;
    if (insert) {
        for (int i = 0; i < 16; ++i) ctx->delta_since_update[i] = (i % 5 == 0) ? 1.f : 0.f;
    } else {
        memcpy(ctx->delta_since_update, nd, sizeof(nd));
    }
    return insert;
}

}  // namespace

// The deferred local-map update (ICPFrameToModel.__update_map, icp_odometry.py:360-380) of the last frame: move / append /
// evict + index rebuild, or the projective model rebuild, on the map stream.
void flush_map_update(pls_context* ctx) {
    if (!ctx->upd_pending) return;
    ctx->upd_pending = false;
    const bool kd = ctx->cfg.local_map_type == PLS_MAP_KDTREE;
    DBuf& frame_vmap = ctx->frame_vmap_buf[ctx->upd_slot];
    DBuf& frame_pts = ctx->frame_pts_buf[ctx->upd_slot];
    map_stream_begin(ctx);
    try {
        if (kd) {
            if (ctx->upd_insert) kdmap_update_packed(ctx, ctx->upd_T, frame_pts.as<float4>(), (int64_t)ctx->upd_count, true);
            else kdmap_update_packed(ctx, ctx->upd_T, nullptr, 0, false);
        } else {
            projmap_update(ctx, ctx->upd_T, ctx->upd_insert ? frame_vmap.as<float>() : nullptr);
        }
    } catch (...) {
        map_stream_end(ctx);
        throw;
    }
    map_stream_end(ctx);
}

namespace {

// What a frame's input stage hands to its ICP and its epilogue.
struct FrameIn {
    int64_t pts_bound = 0;    // rows of the frame's own points, NaN rows included (a bound of them, with n_dev)
    int64_t query_bound = 0;  // bound of the query count
    const uint32_t* n_dev = nullptr;  // the row count on the device, when the host knows only the bound pts_bound
    int64_t map_points = 0;   // points of the kd map the frame registers against (info[3])
};

// The caller's outputs of one frame, each nullable.
struct FrameOut {
    float* pose;
    float* params;
    int* has_pose;
    double* info;
    int64_t samples;  // >= 0: the frame's rows are a grid sample of this many points, reported as info[4]
    void put_samples() const {
        if (info && samples >= 0) info[4] = (double)samples;
    }
};

// Why ctx cannot run a frame of `layout` (without its residency hint) and n rows, grid-sampled at `voxel` if voxel > 0;
// null if it can.  layout < 0: no frame this call (a skipped sequence of a batch), only the context is checked.
const char* frame_refusal(const pls_context* ctx, int layout, int64_t n, double voxel) {
    if (ctx->cfg.gn_max_iters != 1) return "fused ICP path supports gauss_newton_config.max_iters == 1";
    if (layout < 0) return nullptr;
    if (layout < PLS_INPUT_NDARRAY || layout > PLS_INPUT_TENSOR_F64) return "process_frame: unknown layout";
    if (voxel > 0.0 && layout != PLS_INPUT_NDARRAY && layout != PLS_INPUT_TENSOR) return "grid-sampled input is a point layout";
    if (layout != PLS_INPUT_VERTEX_MAP && n <= 0) return "process_frame: empty point cloud";
    return nullptr;
}

// A frame's input on the device.  *layout may carry a residency hint in its high bits: the caller knows where `data`
// lives (a device-resident grid-sample result handed over by pls_grid_sample_staged, a CUDA tensor, a numpy array) and
// saves the classification; host data is copied through ctx->stage_in[0].  Leaves the bare layout in *layout.
const void* stage_frame_input(pls_context* ctx, const void* data, int* layout, int64_t n) {
    const int hint = *layout & (PLS_PTR_DEVICE | PLS_PTR_HOST);
    *layout &= ~(PLS_PTR_DEVICE | PLS_PTR_HOST);
    const bool is64 = *layout == PLS_INPUT_NDARRAY_F64 || *layout == PLS_INPUT_TENSOR_F64;
    const size_t bytes = *layout == PLS_INPUT_VERTEX_MAP ? (size_t)3 * ctx->cfg.height * ctx->cfg.width * sizeof(float)
                                                         : (size_t)n * 3 * (is64 ? sizeof(double) : sizeof(float));
    if (hint == PLS_PTR_DEVICE) return data;
    if (hint != PLS_PTR_HOST) return to_device(ctx, data, bytes, ctx->stage_in[0]);
    ctx->stage_in[0].reserve(bytes, ctx->stream);
    PLS_CUDA(cudaMemcpyAsync(ctx->stage_in[0].p, data, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return ctx->stage_in[0].p;
}

// The grid sample of a frame's raw float32 rows into ctx->gs_out_xyz, which then holds the frame's input.
GridSample frame_grid_sample(pls_context* ctx, const void* raw, int64_t n, double voxel) {
    ctx->gs_out_xyz.reserve((size_t)n * 3 * sizeof(float), ctx->stream);
    return GridSample{raw, false, n, voxel, ctx->gs_out_xyz.p, nullptr, nullptr, nullptr};
}

// The input stage of a frame (icp_odometry.py:319-358, 301-308): input selection, the map-update flush and
// frame_begin_kernel, on ctx->stream.  A sequence's first frame only initialises the map (icp_odometry.py:171-181): that
// is done here, outputs included, and false returned.
// n_dev (nullable): the frame has *n_dev rows, a count still being computed on the device, and n is a bound of it; only
// the fused selection of a float32 frame on the kd map after the first frame reads its rows from a device count.
bool frame_input(pls_context* ctx, const void* data_void, int layout, int64_t n, const uint32_t* n_dev,
                 const float* init_pose, FrameIn& in, const FrameOut& out) {
    cudaStream_t st = ctx->stream;
    // float64 point layouts: same flow, the cloud is rounded to float32 for the queries / map insertion while the frame's
    // own vertex map is projected in float64 (icp_odometry.py:331-352)
    const bool is64 = layout == PLS_INPUT_NDARRAY_F64 || layout == PLS_INPUT_TENSOR_F64;
    if (layout == PLS_INPUT_NDARRAY_F64) layout = PLS_INPUT_NDARRAY;
    if (layout == PLS_INPUT_TENSOR_F64) layout = PLS_INPUT_TENSOR;
    const float* data_dev = is64 ? nullptr : (const float*)data_void;
    const double* data64 = is64 ? (const double*)data_void : nullptr;
    const int H = ctx->cfg.height, W = ctx->cfg.width;
    const int64_t hw = (int64_t)H * W;
    const bool kd = ctx->cfg.local_map_type == PLS_MAP_KDTREE;
    FrameResult* fr = frame_result_dev(ctx);
    if (layout == PLS_INPUT_NDARRAY) ctx->sample_pointcloud = 1;  // icp_odometry.py:330
    const bool first = ctx->frame_index == 0;
    // the previous frame's buffers may still feed the asynchronous map update: use the other pair
    ctx->frame_slot ^= 1;
    DBuf& frame_vmap = ctx->frame_vmap_buf[ctx->frame_slot];
    DBuf& frame_pts = ctx->frame_pts_buf[ctx->frame_slot];

    // ---- _read_input (icp_odometry.py:319-358)
    frame_vmap.reserve((size_t)3 * hw * sizeof(float), st);
    int64_t pts_bound = 0;
    bool fused_input = false;
    if (layout == PLS_INPUT_VERTEX_MAP) {
        scrub_vertex_map_kernel<<<grid_for(hw), 256, 0, st>>>(data_dev, hw, frame_vmap.as<float>());
        PLS_CHECK_LAUNCH();
        ctx->tmp[5].reserve((size_t)hw * sizeof(float4), st);
        // points[points.norm(dim=-1) > 0]  (icp_odometry.py:303-305)
        pack_valid_pixels(ctx, frame_vmap.as<float>(), hw, 0.f, ctx->tmp[5].as<float4>(), count_slot(ctx, 1));
        frame_pts.reserve(sizeof(float4) * 4, st);
        first_point_kernel<<<1, 32, 0, st>>>(ctx->tmp[5].as<float4>(), count_slot(ctx, 1), frame_pts.as<float4>(),
                                              count_slot(ctx, 2), fr);
        PLS_CHECK_LAUNCH();
        pts_bound = 1;
    } else {
        PLS_REQUIRE(n > 0, "process_frame: empty point cloud");
        frame_pts.reserve((size_t)n * sizeof(float4), st);
        pts_bound = n;
        // the shipped pipelines (float32 points, kd map, any frame but the first): one z-buffer pass and one selection
        fused_input = !is64 && kd && !first && n <= SEL_MAX_N && n < (1ll << 32);
        PLS_REQUIRE(fused_input || !n_dev, "process_frame: a device-side row count needs the fused kd input stage");
        if (fused_input) {
            const bool pixel_queries = !ctx->sample_pointcloud;
            FrameInputSelect op;
            op.pts = data_dev;
            op.pc = make_proj_const(H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
            op.zbuf = nullptr;
            op.frame_pts = frame_pts.as<float4>();
            op.queries = nullptr;
            if (pixel_queries) {
                if (ctx->input_zbuf.cap < (size_t)hw * sizeof(unsigned long long)) ctx->input_zbuf_clean = false;
                ctx->input_zbuf.reserve((size_t)hw * sizeof(unsigned long long), st);
                if (!ctx->input_zbuf_clean)
                    PLS_CUDA(cudaMemsetAsync(ctx->input_zbuf.p, 0xff, (size_t)hw * sizeof(unsigned long long), st));
                ctx->input_zbuf_clean = false;  // dirty until the selection below (whose winners reset their pixels) is enqueued
                ctx->queries.reserve((size_t)(n < hw ? n : hw) * sizeof(float4), st);
                launch_zbuf_points(ctx, data_dev, n, n_dev, H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg,
                                   ctx->input_zbuf.as<unsigned long long>());
                op.zbuf = ctx->input_zbuf.as<unsigned long long>();
                op.queries = ctx->queries.as<float4>();
            }
            select_launch(ctx, op, n, n_dev, count_slot(ctx, 2), pixel_queries ? count_slot(ctx, 1) : nullptr);
            if (pixel_queries) ctx->input_zbuf_clean = true;
        } else if (is64) {
            pack_valid_rows_f64(ctx, data64, n, frame_pts.as<float4>(), count_slot(ctx, 2));
        } else {
            pack_valid_rows(ctx, data_dev, n, frame_pts.as<float4>(), count_slot(ctx, 2));
        }
        // the vertex map of the points is needed on frame 0 (map initialisation), as the query
        // source when _sample_pointcloud is False, and by the projective map's update
        if (!fused_input && (first || !ctx->sample_pointcloud || !kd)) {
            ctx->tmp[3].reserve((size_t)hw * sizeof(unsigned long long), st);
            if (is64)
                launch_projection_f64(ctx, data64, n, H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg, frame_vmap.as<float>(),
                                      ctx->tmp[3].as<unsigned long long>());
            else
                launch_projection(ctx, data_dev, nullptr, 1, n, 3, H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg,
                                  frame_vmap.as<float>(), ctx->tmp[3].as<unsigned long long>());
        }
    }
    in.pts_bound = pts_bound;
    in.n_dev = n_dev;

    float eye[16];
    for (int i = 0; i < 16; ++i) eye[i] = (i % 5 == 0) ? 1.f : 0.f;

    if (first) {
        // icp_odometry.py:171-181: the first frame only initialises the map, via its vertex map
        flush_map_update(ctx);
        map_stream_wait(ctx);
        if (kd) kdmap_update(ctx, eye, nullptr, 0, frame_vmap.as<float>(), H, W, -1);
        else projmap_update(ctx, eye, frame_vmap.as<float>());
        ctx->frame_index = 1;
        if (out.has_pose) *out.has_pose = 0;
        if (out.pose) memcpy(out.pose, eye, sizeof(eye));
        if (out.params) memset(out.params, 0, 6 * sizeof(float));
        fetch_result(ctx);
        if (out.info) {
            FrameResult* h = frame_result_host(ctx);
            for (int i = 0; i < 12; ++i) out.info[i] = 0.0;
            out.info[3] = (double)ctx->kd.count;
            out.info[5] = (double)(pts_bound - (int64_t)h->counts[2]);
        }
        out.put_samples();
        return false;
    }

    // ---- sample_points (icp_odometry.py:301-308)
    int64_t query_bound;
    const bool queries_are_rows = ctx->sample_pointcloud && layout != PLS_INPUT_VERTEX_MAP;
    if (queries_are_rows) {
        // queries = the (NaN-free) input points themselves (frame_begin_kernel copies their count)
        ctx->query_ptr = frame_pts.as<float4>();
        query_bound = n;
    } else if (layout == PLS_INPUT_VERTEX_MAP) {
        ctx->query_ptr = ctx->tmp[5].as<float4>();
        query_bound = hw;
    } else if (fused_input) {
        ctx->query_ptr = ctx->queries.as<float4>();  // selected together with the valid rows above
        query_bound = n < hw ? n : hw;
    } else {
        ctx->queries.reserve((size_t)hw * sizeof(float4), st);
        pack_valid_pixels(ctx, frame_vmap.as<float>(), hw, 0.f, ctx->queries.as<float4>(), count_slot(ctx, 1));
        ctx->query_ptr = ctx->queries.as<float4>();
        query_bound = n < hw ? n : hw;
    }
    in.query_bound = query_bound;

    // ---- register_new_frame
    flush_map_update(ctx);  // (already enqueued by the grid-sample call of this frame, if there was one)
    map_stream_wait(ctx);   // the ICP below reads the local map the previous frame's update is still building
    in.map_points = ctx->kd.count;
    frame_begin(ctx, init_pose, nullptr, queries_are_rows);
    return true;
}

// The epilogue of a frame whose ICP result is in the host FrameResult: status, key-frame decision, the deferred map
// update, outputs.  Throws on a failed ICP, leaving the frame unadvanced and no map update pending.
// upd (nullable): the device decided and enqueued the kd map update (with its gate open); the host mirror follows it.
void frame_epilogue(pls_context* ctx, const FrameIn& in, const FrameOut& out, bool trace, const KdUpdateWords* upd) {
    FrameResult* h = frame_result_host(ctx);
    ctx->last_icp_iters = h->iters;
    raise_status(ctx, h->status);

    // ---- __update_map
    bool insert;
    if (upd) {
        insert = upd->insert != 0;
        memcpy(ctx->delta_since_update, upd->delta, sizeof(ctx->delta_since_update));
        kdmap_settle_device_update(ctx, *upd, ctx->cfg.local_map_size);
    } else {  // decided now, enqueued (on the map stream, beside the NEXT frame's preprocessing) by the next call
        insert = keyframe_decision(ctx, h->T);
        ctx->upd_pending = true;
        ctx->upd_insert = insert;
        memcpy(ctx->upd_T, h->T, sizeof(ctx->upd_T));
        ctx->upd_slot = ctx->frame_slot;
        ctx->upd_count = (long long)h->counts[2];
    }
    if (trace) g_trace.lap(2);
    ctx->frame_index += 1;
    if (out.pose) memcpy(out.pose, h->T, 16 * sizeof(float));
    if (out.params) memcpy(out.params, h->params, 6 * sizeof(float));
    if (out.has_pose) *out.has_pose = 1;
    if (out.info) {
        out.info[0] = (double)h->iters;
        out.info[1] = h->iters > 0 ? (double)h->losses[h->iters - 1] : 0.0;
        out.info[2] = (double)h->counts[1];
        out.info[3] = (double)in.map_points;
        out.info[4] = (double)h->counts[0];
        out.info[5] = (double)(in.pts_bound - (int64_t)h->counts[2]);
        out.info[6] = (double)h->status;
        out.info[7] = insert ? 1.0 : 0.0;
        out.info[8] = h->first_pt[0]; out.info[9] = h->first_pt[1]; out.info[10] = h->first_pt[2];
        out.info[11] = ctx->last_sharded ? 1.0 : 0.0;  // the correspondences were split over the ranks
    }
    out.put_samples();
}

// What enqueueing a device-decided kd map update changes in the host mirror of the map.  The mirror goes back to the
// state before it at once -- ICP launches of a second round still search the frame's map -- and takes the state after
// it once the result shows the update's gate open (with it closed, the device left the map as it was).
struct KdMirror {
    int cur;
    int64_t count, indexed;
    bool valid, bbox_clean;
    uint32_t gen, prev_gen;
    const void* sorted;
    explicit KdMirror(const pls_context* ctx)
        : cur(ctx->kd.cur), count(ctx->kd.count), indexed(ctx->kd.indexed), valid(ctx->kd.valid),
          bbox_clean(ctx->kd.bbox_clean), gen(ctx->kd.gen), prev_gen(ctx->kd.prev_gen), sorted(ctx->kd.sorted.p) {}
    void restore(pls_context* ctx) const {
        KdMap& kd = ctx->kd;
        kd.cur = cur;
        kd.count = count;
        kd.indexed = indexed;
        kd.valid = valid;
        kd.bbox_clean = bbox_clean;
        kd.gen = gen;
        kd.prev_gen = prev_gen;
        if (kd.sorted.p != sorted) std::swap(kd.sorted, kd.sorted_prev);
    }
};

// The frame's kd map update, decided on the device behind the ICP launches enqueued so far and enqueued on the map
// stream right away, so that its launches leave the host's path between this frame's ICP and the next frame.  Leaves
// the host mirror of the map as the update's launches advanced it (see KdMirror); the counts are settled from the
// result copy (kdmap_settle_device_update).
void enqueue_device_map_update(pls_context* ctx, const FrameIn& in) {
    KdMap& kd = ctx->kd;
    const int64_t bound = kdmap_device_update_bound(ctx, in.pts_bound);
    // the evicted frame's points if this frame is inserted (kdmap_update_packed's deque, one frame ahead)
    const int64_t evict =
        (int64_t)kd.frame_counts.size() + 1 > ctx->cfg.local_map_size ? kd.frame_counts.front() : 0;
    Pose16 delta;
    memcpy(delta.m, ctx->delta_since_update, sizeof(delta.m));
    map_stream_wait(ctx);  // an earlier update of this frame (closed gate) still reads the words rewritten here
    kd_update_decision_kernel<<<1, 1, 0, ctx->stream>>>(frame_result_dev(ctx), kd_update_words_dev(ctx), delta,
                                                         ctx->cfg.threshold_trans, ctx->cfg.threshold_rot,
                                                         ctx->cfg.max_num_alignments, (uint32_t)kd.count, (uint32_t)evict,
                                                         (uint32_t)bound, in.n_dev ? scalar_u32(ctx, SC_GS_OVERFLOW) : nullptr, ctx->gs_seq);
    PLS_CHECK_LAUNCH();
    if (!ctx->ev_icp_done) PLS_CUDA(cudaEventCreateWithFlags(&ctx->ev_icp_done, cudaEventDisableTiming));
    PLS_CUDA(cudaEventRecord(ctx->ev_icp_done, ctx->stream_main));
    PLS_CUDA(cudaStreamWaitEvent(ctx->stream_map, ctx->ev_icp_done, 0));
    map_stream_begin(ctx);
    try {
        kdmap_update_on_device(ctx, ctx->frame_pts_buf[ctx->frame_slot].as<float4>(), bound, kd_update_words_dev(ctx));
    } catch (...) {
        map_stream_end(ctx);
        throw;
    }
    map_stream_end(ctx);
}

// One frame, enqueued in one go; the host waits once, for its result.  n_dev: see frame_input -- here it is the count of a
// grid sample enqueued on compact keys, whose overflow stamp comes back with the result: if the keys overflowed, the
// frame ran on a wrong sample, nothing is reported or advanced past the input stage, and false is returned for the
// caller to roll back and replay.
// On a kd map after its first insertion, on one GPU, the frame's map update is decided on the device and enqueued before
// the host waits (enqueue_device_map_update); a frame that needs a second round of ICP launches enqueues it again behind
// them.  Otherwise -- and when the new map count would exceed the capacity planned so far -- the update is decided by
// the host after the wait and enqueued by the next call (flush_map_update).
bool process_frame_device(pls_context* ctx, const void* data_void, int layout, int64_t n, const uint32_t* n_dev,
                          const float* init_pose, FrameOut out) {
    g_trace.frame_start();
    FrameIn in;
    if (!frame_input(ctx, data_void, layout, n, n_dev, init_pose, in, out)) return true;
    const bool device_update = ctx->cfg.local_map_type == PLS_MAP_KDTREE && comm_size(ctx) == 1 &&
                               kdmap_device_update_bound(ctx, in.pts_bound) > 0;
    const KdMirror before(ctx);
    std::optional<KdMirror> after;
    std::function<void()> update;
    if (device_update)
        update = [&] {
            enqueue_device_map_update(ctx, in);
            after.emplace(ctx);
            before.restore(ctx);
        };
    int extra_rounds = 0;
    int icp_blocks = run_icp(ctx, in.query_bound, in.n_dev, update, &extra_rounds);
    g_trace.lap(1);
    // a closed gate: the device left the map as it was.  An overflowed sample is replayed and a failed ICP reported
    // below; a map grown beyond the planned capacity is updated by the host's path (frame_epilogue, flush_map_update)
    const KdUpdateWords* upd = device_update && kd_update_words_host(ctx)->gate ? kd_update_words_host(ctx) : nullptr;
    if (upd) after->restore(ctx);
    if (in.n_dev) {
        bool overflowed = false;
        const int64_t rows = grid_sample_host_count(ctx, &overflowed);
        if (overflowed) return false;
        in.pts_bound = rows;
        out.samples = rows;
        // the block count the correspondence kernels ran with (kd_logical_blocks)
        const int64_t q = rows < in.query_bound ? rows : in.query_bound;
        icp_blocks = grid_for(q < 1 ? 1 : q);
    }
    ctx->icp_result = true;
    credit_icp_profile(ctx, frame_result_host(ctx), icp_blocks);
    frame_epilogue(ctx, in, out, true, upd);
    g_trace.lap(3);
    g_trace.end_frame();
    return true;
}

// What a frame changes in its context before its result is known: the state a replayed frame starts again from.
struct FrameEntryState {
    int frame_slot, frame_index, last_icp_iters;
    bool input_zbuf_clean;
    explicit FrameEntryState(const pls_context* ctx)
        : frame_slot(ctx->frame_slot), frame_index(ctx->frame_index), last_icp_iters(ctx->last_icp_iters),
          input_zbuf_clean(ctx->input_zbuf_clean) {}
    void restore(pls_context* ctx) const {
        ctx->frame_slot = frame_slot;
        ctx->frame_index = frame_index;
        ctx->last_icp_iters = last_icp_iters;
        ctx->input_zbuf_clean = input_zbuf_clean;
    }
};

}  // namespace

void odometry_reset(pls_context* ctx) {
    kdmap_reset(ctx);
    projmap_reset(ctx);
    ctx->frame_index = 0;
    ctx->last_icp_iters = 0;
    // _sample_pointcloud is set in the reference's constructor only: ICPFrameToModel.init() keeps it
    // (icp_odometry.py:105,128-137), so a re-initialised sequence samples like the last frame of the previous one
    for (int i = 0; i < 16; ++i) ctx->delta_since_update[i] = (i % 5 == 0) ? 1.f : 0.f;
}

// The B registrations of pls_register_hypotheses / pls_register_scans from T0_dev [B,16] on ctx's map, whose queries are
// packed, in chunks of PLS_MAX_SEQUENCES.  kd map: registration b reads scans[b].  Projective map: every registration
// reads the scan in ctx->query_ptr, bound n.  Outputs and status as pls_register_hypotheses; afterwards the last
// registration is ctx's last search and last ICP result, as if pls_register_frame had run it last.
// max_distance (kd map): the gate of pls_register_scans_gated, +inf for none; out_inliers [B] (nullable): each
// registration's count accumulator of its last executed iteration, its inliers there.  A gated registration whose last
// iteration had no inlier reports PLS_E_SINGULAR: its sums are all zero, which the solve's zero-residual test would
// otherwise report as PLS_W_TINY_RESIDUAL, the flag of a near-perfect fit.
// min_eigenvalue > 0 (kd map): the eigenvalue-thresholded solve of pls_register_scans_degeneracy; out_degenerate [B] and
// out_eigenvalues [B,6] (nullable): each registration's degenerate count and eigenvalues of H / N in its last executed
// iteration.
static void register_batch(pls_context* ctx, const KdScan* scans, int64_t n, const float* T0_dev, int B, float* out_T,
                           float* out_params, float* out_losses, int* out_iters, int* out_status,
                           double max_distance = HUGE_VAL, int* out_inliers = nullptr, double min_eigenvalue = 0.0,
                           int* out_degenerate = nullptr, double* out_eigenvalues = nullptr) {
    const bool kd = ctx->cfg.local_map_type == PLS_MAP_KDTREE;
    cudaStream_t st = ctx->stream;
    const int M = ctx->cfg.max_num_alignments;
    std::vector<FrameResult> h((size_t)PLS_MAX_SEQUENCES);
    std::vector<float> T((size_t)B * 16), params((size_t)B * 6), losses((size_t)B * M);
    std::vector<int> iters((size_t)B), status((size_t)B), inliers((size_t)B), degenerate((size_t)B);
    std::vector<double> eigenvalues((size_t)B * 6), degen_rows;
    const bool thresholded = min_eigenvalue > 0.0;
    double* degen = nullptr;
    if (thresholded) {
        ctx->degen_buf.reserve((size_t)PLS_MAX_SEQUENCES * ICP_DEGEN_STRIDE * sizeof(double), st);
        degen = ctx->degen_buf.as<double>();
        degen_rows.resize((size_t)PLS_MAX_SEQUENCES * ICP_DEGEN_STRIDE);
    }
    int first_error = PLS_OK, last = 0;
    for (int c0 = 0; c0 < B; c0 += PLS_MAX_SEQUENCES) {  // chunks of at most PLS_MAX_SEQUENCES registrations
        const int num = B - c0 < PLS_MAX_SEQUENCES ? B - c0 : PLS_MAX_SEQUENCES;
        int grid[KD_BATCH_GRID];
        FrameResult* frs = nullptr;
        uint32_t* words = nullptr;
        if (kd) kdmap_hypotheses_begin(ctx, scans + c0, num, st, grid, &frs, &words);
        else projmap_hypotheses_begin(ctx, num, st, &frs, &words);
        hypotheses_begin_kernel<<<num, kMaxAlign, 0, st>>>(frs, T0_dev + 16 * (size_t)c0, words);
        PLS_CHECK_LAUNCH();
        // every registration has ctx's settings: icp_rounds sees num copies of ctx
        std::vector<pls_context*> same((size_t)num, ctx);
        if (kd)
            icp_rounds(same.data(), num,
                       [&](int a, int b) {
                           kdmap_batch_iterations(ctx, num, st, grid, a, b, max_distance, min_eigenvalue, degen);
                       },
                       [&](int* done) { kdmap_batch_done(ctx, num, st, done); });
        else
            icp_rounds(same.data(), num, [&](int a, int b) { projmap_hypotheses_iterations(ctx, n, num, st, a, b); },
                       [&](int* done) { projmap_batch_done(ctx, num, st, done); });
        PLS_CUDA(cudaMemcpyAsync(h.data(), frs, (size_t)num * sizeof(FrameResult), cudaMemcpyDeviceToHost, st));
        if (thresholded)
            PLS_CUDA(cudaMemcpyAsync(degen_rows.data(), degen, (size_t)num * ICP_DEGEN_STRIDE * sizeof(double),
                                     cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        for (int j = 0; j < num; ++j) {
            const FrameResult& r = h[(size_t)j];
            const size_t b = (size_t)(c0 + j);
            memcpy(&T[16 * b], r.T, 16 * sizeof(float));
            memcpy(&params[6 * b], r.params, 6 * sizeof(float));
            memcpy(&losses[(size_t)M * b], r.losses, (size_t)M * sizeof(float));
            iters[b] = r.iters;
            status[b] = r.status;
            inliers[b] = (int)r.last_sums[29];
            if (!isinf(max_distance) && inliers[b] == 0) status[b] = PLS_E_SINGULAR;
            if (thresholded) {
                const double* row = &degen_rows[(size_t)ICP_DEGEN_STRIDE * j];
                memcpy(&eigenvalues[6 * b], row, 6 * sizeof(double));
                degenerate[b] = (int)row[6];
            }
            if (first_error == PLS_OK && (status[b] == PLS_E_SINGULAR || r.status == PLS_E_COMM)) first_error = status[b];
        }
        last = num - 1;
    }
    if (kd) kdmap_hypothesis_adopt(ctx, scans[B - 1], last, st);
    else projmap_hypothesis_adopt(ctx, last, st);
    fetch_result(ctx);
    ctx->icp_result = true;
    put_out(out_T, T.data(), T.size() * sizeof(float));
    put_out(out_params, params.data(), params.size() * sizeof(float));
    put_out(out_losses, losses.data(), losses.size() * sizeof(float));
    put_out(out_iters, iters.data(), iters.size() * sizeof(int));
    put_out(out_status, status.data(), status.size() * sizeof(int));
    put_out(out_inliers, inliers.data(), inliers.size() * sizeof(int));
    put_out(out_degenerate, degenerate.data(), degenerate.size() * sizeof(int));
    put_out(out_eigenvalues, eigenvalues.data(), eigenvalues.size() * sizeof(double));
    if (!out_status) raise_status(ctx, first_error);
}

// pls_register_scans / pls_kdmap_evaluate_poses: the S scans staged (host scans back to back, as to_device stages one)
// and packed into ctx->queries by one launch; returns the scan each of the B registrations reads.
static std::vector<KdScan> stage_scans(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                       const int* scan_of, int B) {
    cudaStream_t st = ctx->stream;
    size_t host_rows = 0;
    for (int s = 0; s < S; ++s)
        if (!is_device_ptr(scans[s])) host_rows += (size_t)n[s];
    if (host_rows) ctx->stage_in[0].reserve(host_rows * 3 * sizeof(float), st);
    // scan s's packed rows go to ctx->queries at the sum of the earlier scans' row counts, the S counts behind them
    size_t rows = 0;
    for (int s = 0; s < S; ++s) rows += (size_t)n[s];
    ctx->queries.reserve(rows * sizeof(float4) + (size_t)S * sizeof(uint32_t), st);
    float4* q = ctx->queries.as<float4>();
    uint32_t* counts = reinterpret_cast<uint32_t*>(q + rows);
    std::vector<KdScanRows> pack((size_t)S);
    std::vector<KdScan> packed((size_t)S);
    float* staged = ctx->stage_in[0].as<float>();
    for (int s = 0; s < S; ++s) {
        const float* d = scans[s];
        if (!is_device_ptr(d)) {
            PLS_CUDA(cudaMemcpyAsync(staged, d, (size_t)n[s] * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
            d = staged;
            staged += (size_t)n[s] * 3;
        }
        pack[(size_t)s] = KdScanRows{d, n[s], q, counts + s};
        packed[(size_t)s] = KdScan{q, counts + s, n[s]};
        q += n[s];
    }
    FrameResult* fr = frame_result_dev(ctx);
    PLS_CUDA(cudaMemsetAsync(fr->counts, 0, sizeof(fr->counts), st));
    pack_valid_scans(ctx, pack);
    std::vector<KdScan> regs((size_t)B);
    for (int b = 0; b < B; ++b) regs[(size_t)b] = packed[(size_t)(scan_of ? scan_of[b] : b)];
    return regs;
}

}  // namespace pls

using namespace pls;

extern "C" {

int pls_map_init(pls_context* ctx) {
    PLS_API_BEGIN(ctx)
    sync_all(ctx);
    kdmap_reset(ctx);
    projmap_reset(ctx);
    PLS_API_END(ctx)
}

int pls_set_shard_min(int64_t work_items_per_rank) {
    g_shard_min_override = work_items_per_rank;
    return PLS_OK;
}

int pls_last_sharded(pls_context* ctx, int* out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(out, "pls_last_sharded: null output");
    *out = ctx->last_sharded ? 1 : 0;
    PLS_API_END(ctx)
}

int pls_odometry_init(pls_context* ctx) {
    PLS_API_BEGIN(ctx)
    sync_all(ctx);
    odometry_reset(ctx);
    PLS_API_END(ctx)
}

int pls_register_frame(pls_context* ctx, const float* points, int64_t n, const float* T0, float* out_T,
                       float* out_params, float* out_losses, int* out_iters) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(points && n > 0, "pls_register_frame: points must be [n,3] with n > 0");
    PLS_REQUIRE(ctx->cfg.gn_max_iters == 1, "fused ICP path supports gauss_newton_config.max_iters == 1");
    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    const float* d = (const float*)to_device(ctx, points, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    FrameResult* fr = frame_result_dev(ctx);
    PLS_CUDA(cudaMemsetAsync(fr->counts, 0, sizeof(fr->counts), st));
    ctx->queries.reserve((size_t)n * sizeof(float4), st);
    pack_valid_rows(ctx, d, n, ctx->queries.as<float4>(), count_slot(ctx, 1));
    ctx->query_ptr = ctx->queries.as<float4>();
    const float* T0_dev = nullptr;
    if (T0) {
        ctx->tmp[6].reserve(16 * sizeof(float), st);
        PLS_CUDA(cudaMemcpyAsync(ctx->tmp[6].p, T0, 16 * sizeof(float),
                                 is_device_ptr(T0) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        T0_dev = ctx->tmp[6].as<float>();
    }
    frame_begin(ctx, nullptr, T0_dev, false);
    int extra_rounds = 0;
    const int icp_blocks = run_icp(ctx, n, nullptr, nullptr, &extra_rounds);
    ctx->icp_result = true;
    FrameResult* h = frame_result_host(ctx);
    credit_icp_profile(ctx, h, icp_blocks);
    put_out(out_T, h->T, 16 * sizeof(float));
    put_out(out_params, h->params, 6 * sizeof(float));
    put_out(out_losses, h->losses, (size_t)ctx->cfg.max_num_alignments * sizeof(float));
    if (out_iters) *out_iters = h->iters;
    raise_status(ctx, h->status);
    PLS_API_END(ctx)
}

int pls_register_hypotheses(pls_context* ctx, const float* points, int64_t n, const float* T0s, int B, float* out_T,
                            float* out_params, float* out_losses, int* out_iters, int* out_status) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(points && n > 0, "pls_register_hypotheses: points must be [n,3] with n > 0");
    PLS_REQUIRE(T0s && B > 0, "pls_register_hypotheses: T0s must be [B,16] with B > 0");
    PLS_REQUIRE(ctx->cfg.gn_max_iters == 1, "fused ICP path supports gauss_newton_config.max_iters == 1");
    const bool kd = ctx->cfg.local_map_type == PLS_MAP_KDTREE;
    PLS_REQUIRE(!ctx->comm, "pls_register_hypotheses: a context with a multi-GPU communicator is not supported");
    if (kd) PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    else PLS_REQUIRE(ctx->pm.valid, "projective map: search before any update");
    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    // the scan is packed once, as pls_register_frame packs it; every hypothesis reads it
    const float* d = (const float*)to_device(ctx, points, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    const float* T0_dev = (const float*)to_device(ctx, T0s, (size_t)B * 16 * sizeof(float), ctx->stage_in[1]);
    FrameResult* fr = frame_result_dev(ctx);
    PLS_CUDA(cudaMemsetAsync(fr->counts, 0, sizeof(fr->counts), st));
    ctx->queries.reserve((size_t)n * sizeof(float4), st);
    pack_valid_rows(ctx, d, n, ctx->queries.as<float4>(), count_slot(ctx, 1));
    ctx->query_ptr = ctx->queries.as<float4>();
    // on a kd map: pls_register_scans's registrations, S = 1, every hypothesis on the one scan
    const std::vector<KdScan> scans(kd ? (size_t)B : 0, KdScan{ctx->query_ptr, count_slot(ctx, 1), n});
    register_batch(ctx, scans.data(), n, T0_dev, B, out_T, out_params, out_losses, out_iters, out_status);
    PLS_API_END(ctx)
}

// pls_register_scans, pls_register_scans_gated and pls_register_scans_degeneracy (fn names the entry point in
// refusals; min_eigenvalue 0: the solve of the first two).
static void register_scans(pls_context* ctx, const char* fn, const float* const* scans, const int64_t* n, int S,
                           const int* scan_of, const float* T0s, int B, double max_distance, float* out_T,
                           float* out_params, float* out_losses, int* out_iters, int* out_status, int* out_inliers,
                           double min_eigenvalue = 0.0, int* out_degenerate = nullptr,
                           double* out_eigenvalues = nullptr) {
    const std::string f(fn);
    // every argument is checked before anything is enqueued: a refused call changes nothing
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, f + ": needs a kd-tree local map");
    PLS_REQUIRE(ctx->cfg.gn_max_iters == 1, "fused ICP path supports gauss_newton_config.max_iters == 1");
    PLS_REQUIRE(!ctx->comm, f + ": a context with a multi-GPU communicator is not supported");
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    PLS_REQUIRE(scans && n && S > 0, f + ": scans and n must hold S > 0 scans");
    PLS_REQUIRE(T0s && B > 0, f + ": T0s must be [B,16] with B > 0");
    PLS_REQUIRE(scan_of || B == S, f + ": without scan_of, B must equal S");
    PLS_REQUIRE(max_distance >= 0.0, f + ": max_distance must be >= 0 (not NaN)");
    for (int s = 0; s < S; ++s) PLS_REQUIRE(scans[s] && n[s] > 0, f + ": every scan must be [n,3] with n > 0");
    for (int b = 0; scan_of && b < B; ++b)
        PLS_REQUIRE(scan_of[b] >= 0 && scan_of[b] < S, f + ": scan_of entries must lie in [0, S)");
    map_stream_wait(ctx);
    const std::vector<KdScan> regs = stage_scans(ctx, scans, n, S, scan_of, B);
    const float* T0_dev = (const float*)to_device(ctx, T0s, (size_t)B * 16 * sizeof(float), ctx->stage_in[1]);
    register_batch(ctx, regs.data(), 0, T0_dev, B, out_T, out_params, out_losses, out_iters, out_status, max_distance,
                   out_inliers, min_eigenvalue, out_degenerate, out_eigenvalues);
}

int pls_register_scans(pls_context* ctx, const float* const* scans, const int64_t* n, int S, const int* scan_of,
                       const float* T0s, int B, float* out_T, float* out_params, float* out_losses, int* out_iters,
                       int* out_status) {
    PLS_API_BEGIN(ctx)
    register_scans(ctx, "pls_register_scans", scans, n, S, scan_of, T0s, B, HUGE_VAL, out_T, out_params, out_losses,
                   out_iters, out_status, nullptr);
    PLS_API_END(ctx)
}

int pls_register_scans_gated(pls_context* ctx, const float* const* scans, const int64_t* n, int S, const int* scan_of,
                             const float* T0s, int B, double max_distance, float* out_T, float* out_params,
                             float* out_losses, int* out_iters, int* out_status, int* out_inliers) {
    PLS_API_BEGIN(ctx)
    register_scans(ctx, "pls_register_scans_gated", scans, n, S, scan_of, T0s, B, max_distance, out_T, out_params,
                   out_losses, out_iters, out_status, out_inliers);
    PLS_API_END(ctx)
}

int pls_register_scans_degeneracy(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                  const int* scan_of, const float* T0s, int B, double max_distance,
                                  double min_eigenvalue, float* out_T, float* out_params, float* out_losses,
                                  int* out_iters, int* out_status, int* out_inliers, int* out_degenerate,
                                  double* out_eigenvalues) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(min_eigenvalue > 0.0 && !isinf(min_eigenvalue),
                "pls_register_scans_degeneracy: min_eigenvalue must be finite and > 0 (not NaN)");
    register_scans(ctx, "pls_register_scans_degeneracy", scans, n, S, scan_of, T0s, B, max_distance, out_T, out_params,
                   out_losses, out_iters, out_status, out_inliers, min_eigenvalue, out_degenerate, out_eigenvalues);
    PLS_API_END(ctx)
}

int pls_kdmap_evaluate_poses(pls_context* ctx, const float* const* scans, const int64_t* n, int S, const int* scan_of,
                             const float* T, int B, double max_distance, double* out_stats) {
    PLS_API_BEGIN(ctx)
    // every argument is checked before anything is enqueued: a refused call changes nothing
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, "pls_kdmap_evaluate_poses: needs a kd-tree local map");
    PLS_REQUIRE(!ctx->comm, "pls_kdmap_evaluate_poses: a context with a multi-GPU communicator is not supported");
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    PLS_REQUIRE(scans && n && S > 0, "pls_kdmap_evaluate_poses: scans and n must hold S > 0 scans");
    PLS_REQUIRE(T && B > 0, "pls_kdmap_evaluate_poses: T must be [B,16] with B > 0");
    PLS_REQUIRE(out_stats, "pls_kdmap_evaluate_poses: null out_stats");
    PLS_REQUIRE(scan_of || B == S, "pls_kdmap_evaluate_poses: without scan_of, B must equal S");
    PLS_REQUIRE(max_distance >= 0.0, "pls_kdmap_evaluate_poses: max_distance must be >= 0 (not NaN)");
    for (int s = 0; s < S; ++s)
        PLS_REQUIRE(scans[s] && n[s] > 0, "pls_kdmap_evaluate_poses: every scan must be [n,3] with n > 0");
    for (int b = 0; scan_of && b < B; ++b)
        PLS_REQUIRE(scan_of[b] >= 0 && scan_of[b] < S, "pls_kdmap_evaluate_poses: scan_of entries must lie in [0, S)");
    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    const std::vector<KdScan> regs = stage_scans(ctx, scans, n, S, scan_of, B);
    const float* T_dev = (const float*)to_device(ctx, T, (size_t)B * 16 * sizeof(float), ctx->stage_in[1]);
    OutArg o = out_arg(ctx, out_stats, (size_t)B * PLS_EVAL_STATS * sizeof(double), ctx->stage_out[0]);
    const double max_d2 = max_distance * max_distance;
    int last = 0;
    // no host synchronisation between the chunks: a buffer that grows waits for the stream itself (DBuf::reserve)
    for (int c0 = 0; c0 < B; c0 += PLS_MAX_SEQUENCES) {
        const int num = B - c0 < PLS_MAX_SEQUENCES ? B - c0 : PLS_MAX_SEQUENCES;
        int grid[KD_BATCH_GRID];
        FrameResult* frs = nullptr;
        uint32_t* words = nullptr;
        kdmap_hypotheses_begin(ctx, regs.data() + c0, num, st, grid, &frs, &words);
        hypotheses_begin_kernel<<<num, kMaxAlign, 0, st>>>(frs, T_dev + 16 * (size_t)c0, words);
        PLS_CHECK_LAUNCH();
        kdmap_evaluate_batch(ctx, num, st, grid, max_d2, (double*)o.dev + (size_t)PLS_EVAL_STATS * c0);
        last = num - 1;
    }
    kdmap_hypothesis_adopt(ctx, regs[(size_t)B - 1], last, st);
    fetch_result(ctx);
    ctx->icp_result = true;
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_API_END(ctx)
}


int pls_process_frame(pls_context* ctx, const void* data, int layout, int64_t n, const float* init_pose,
                      float* out_pose, float* out_params, int* out_has_pose, double* out_info) {
    PLS_API_BEGIN(ctx)  // (enqueues the last frame's map update first, unless this frame's grid-sample call already did)
    PLS_REQUIRE(data, "pls_process_frame: null data");
    if (const char* why = frame_refusal(ctx, layout & ~(PLS_PTR_DEVICE | PLS_PTR_HOST), n, 0.0))
        throw pls::Error{PLS_E_INVALID, why};
    const void* d = stage_frame_input(ctx, data, &layout, n);
    process_frame_device(ctx, d, layout, n, nullptr, init_pose, FrameOut{out_pose, out_params, out_has_pose, out_info, -1});
    PLS_API_END(ctx)
}

int pls_process_frame_grid_sample(pls_context* ctx, const float* raw_points, int64_t n, double voxel, int layout,
                                  const float* init_pose, float* out_pose, float* out_params, int* out_has_pose,
                                  double* out_info) {
    // (a map update still pending -- one the host decided -- is enqueued first here: with no host gap between the frames
    // the next ICP would otherwise wait for an index build that started a subsample's worth of launches later; an update
    // the device decided was enqueued with the last frame)
    g_trace.begin_call();
    PLS_API_BEGIN(ctx)
    g_trace.lap(4);
    PLS_REQUIRE(raw_points && n > 0 && voxel > 0.0, "pls_process_frame_grid_sample: bad arguments");
    if (const char* why = frame_refusal(ctx, layout, n, voxel)) throw pls::Error{PLS_E_INVALID, why};
    const void* d = to_device(ctx, raw_points, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    const GridSample g = frame_grid_sample(ctx, d, n, voxel);
    const FrameOut out{out_pose, out_params, out_has_pose, out_info, -1};
    // After a kd map's first frame, on one GPU, the fused input stage reads the sample count on the device (the raw row
    // count n bounds it): the frame is enqueued in one go, without waiting for the count.  The sharding decision of a
    // multi-GPU context and every other input stage size their launches from the count on the host.
    const bool deferred = ctx->frame_index > 0 && ctx->cfg.local_map_type == PLS_MAP_KDTREE && comm_size(ctx) == 1 &&
                          n <= SEL_MAX_N;
    if (deferred) {
        const FrameEntryState entry(ctx);
        grid_sample_enqueue(ctx, g, false);
        if (process_frame_device(ctx, ctx->gs_out_xyz.p, layout, n, scalar_u32(ctx, SC_GS_COUNT), init_pose, out)) return PLS_OK;
        // a hash overflowed the compact sort keys: the frame ran on a wrong sample and is run again from its entry state
        // on the raw keys (this frame's map update did nothing: its gate stayed closed; the cached normals stay valid for
        // the index)
        entry.restore(ctx);
    } else {
        grid_sample_enqueue(ctx, g);
        PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    // the sample count on the host, which sizes the frame; on overflowed compact keys, once more on the raw keys
    const int64_t S = grid_sample_finish(ctx, g);
    FrameOut sized = out;
    sized.samples = S;
    process_frame_device(ctx, ctx->gs_out_xyz.p, layout, S, nullptr, init_pose, sized);
    PLS_API_END(ctx)
}

// A read-only look at the host copy of the last ICP frame's result.  PLS_API_BEGIN_FRAME: a pending map update stays
// pending.
int pls_last_icp_sums(pls_context* ctx, double* out_sums, int* out_iters) {
    PLS_API_BEGIN_FRAME(ctx)
    PLS_REQUIRE(out_sums, "pls_last_icp_sums: null output");
    if (!ctx->icp_result) throw pls::Error{PLS_E_STATE, "pls_last_icp_sums: no ICP frame has run on this context"};
    const FrameResult* h = frame_result_host(ctx);
    memcpy(out_sums, h->last_sums, NACC * sizeof(double));
    if (out_iters) *out_iters = h->iters;
    PLS_API_END(ctx)
}

int pls_process_frames(pls_context* const* ctxs, int num, const void* const* data, const int* layouts, const int64_t* n,
                       double voxel, const float* const* init_poses, float* out_poses, float* out_params, int* out_has_pose,
                       double* out_info, int* out_status) {
    // ---- every argument is checked before anything is enqueued: a refused call changes no context
    const char* why = nullptr;
    if (!ctxs || num < 0 || num > PLS_MAX_SEQUENCES) why = "pls_process_frames: need 0 <= num <= PLS_MAX_SEQUENCES contexts";
    else if (num > 0 && (!data || !layouts || !n)) why = "pls_process_frames: data, layouts and n are required";
    for (int i = 0; !why && i < num; ++i) {
        const pls_context* c = ctxs[i];
        if (!c) { why = "pls_process_frames: null context"; break; }
        if (c->cfg.local_map_type != ctxs[0]->cfg.local_map_type)
            why = "pls_process_frames: batched sequences share one local map type: all kd-tree or all projective";
        else if (c->comm) why = "pls_process_frames: a context with a multi-GPU communicator cannot be batched";
        else if (c->cfg.device != ctxs[0]->cfg.device) why = "pls_process_frames: every context must be on one device";
        for (int j = 0; !why && j < i; ++j)
            if (ctxs[j] == c) why = "pls_process_frames: a context is listed twice";
        if (!why) why = frame_refusal(c, data[i] ? layouts[i] & ~(PLS_PTR_DEVICE | PLS_PTR_HOST) : -1, n[i], voxel);
    }
    if (why) {
        for (int i = 0; ctxs && i < num; ++i)
            if (ctxs[i]) ctxs[i]->err = why;
        return PLS_E_INVALID;
    }
    std::vector<int> active;
    for (int i = 0; i < num; ++i)
        if (data[i]) active.push_back(i);
    for (int i = 0; i < num; ++i)
        if (out_status) out_status[i] = PLS_OK;
    if (active.empty()) return PLS_OK;

    // profiling slots are not credited by a batched call
    struct ProfileOff {
        std::vector<std::pair<pls_context*, int>> off;
        ~ProfileOff() {
            for (auto& o : off) o.first->prof[o.second].enabled = true;
        }
    } prof_off;
    for (int i : active)
        for (int w = 0; w < kProfileSlots; ++w)
            if (ctxs[i]->prof[w].enabled) {
                ctxs[i]->prof[w].enabled = false;
                prof_off.off.push_back({ctxs[i], w});
            }

    pls_context* lead = ctxs[active[0]];
    int cur = active[0];  // the sequence a failure below belongs to
    std::vector<int> status((size_t)num, PLS_OK);
    std::vector<char> finished((size_t)num, 0);  // the sequence's frame is complete (or it was skipped)
    for (int i = 0; i < num; ++i) finished[i] = data[i] == nullptr;
    BatchTrace trace;
    try {
        PLS_CUDA(cudaSetDevice(lead->cfg.device));
        const cudaStream_t st = lead->stream;
        trace.begin(st);
        auto order_before_lead = [&](pls_context* ctx) {  // ctx's work so far happens-before lead's next work
            if (ctx == lead) return;
            if (!ctx->ev_batch) PLS_CUDA(cudaEventCreateWithFlags(&ctx->ev_batch, cudaEventDisableTiming));
            PLS_CUDA(cudaEventRecord(ctx->ev_batch, ctx->stream));
            PLS_CUDA(cudaStreamWaitEvent(st, ctx->ev_batch, 0));
        };
        // ---- input stage, per sequence on its own stream: the pending map update, the input on the device and, with
        // voxel > 0, the grid sample, whose counts are read back together
        std::vector<const void*> dev((size_t)num, nullptr);
        std::vector<int64_t> rows(n, n + num);
        std::vector<int> lay(layouts, layouts + num);
        std::vector<GridSample> gs((size_t)num);
        for (int i : active) {
            cur = i;
            pls_context* ctx = ctxs[i];
            flush_map_update(ctx);
            dev[i] = stage_frame_input(ctx, data[i], &lay[i], n[i]);
            if (voxel > 0.0) {
                gs[i] = frame_grid_sample(ctx, dev[i], n[i], voxel);
                grid_sample_enqueue(ctx, gs[i]);
                order_before_lead(ctx);
            }
        }
        if (voxel > 0.0) {
            PLS_CUDA(cudaStreamSynchronize(st));
            for (int i : active) {
                cur = i;
                rows[i] = grid_sample_finish(ctxs[i], gs[i]);
                dev[i] = ctxs[i]->gs_out_xyz.p;
            }
        }
        std::vector<FrameIn> in((size_t)num);
        std::vector<pls_context*> icp;
        std::vector<int> icp_seq;
        std::vector<int64_t> bounds;
        auto outputs = [&](int i) {
            return FrameOut{out_poses ? out_poses + 16 * i : nullptr, out_params ? out_params + 6 * i : nullptr,
                            out_has_pose ? out_has_pose + i : nullptr, out_info ? out_info + 12 * i : nullptr,
                            voxel > 0.0 ? rows[i] : -1};
        };
        for (int i : active) {
            cur = i;
            pls_context* ctx = ctxs[i];
            bool runs_icp = false;
            try {
                runs_icp = frame_input(ctx, dev[i], lay[i], rows[i], nullptr, init_poses ? init_poses[i] : nullptr, in[i],
                                       outputs(i));
            } catch (const pls::Error& e) {
                // an input the single path refuses (e.g. a grid sample of no point) is that sequence's error alone
                if (e.code != PLS_E_INVALID) throw;
                ctx->err = e.msg;
                status[i] = e.code;
                finished[i] = 1;
                continue;
            }
            if (!runs_icp) {
                finished[i] = 1;
                continue;
            }
            ctx->pm.zbuf_clean = false;
            icp.push_back(ctx);
            icp_seq.push_back(i);
            bounds.push_back(in[i].query_bound < 1 ? 1 : in[i].query_bound);
            order_before_lead(ctx);
        }
        // ---- the ICP of every sequence on the lead's stream, each kernel one launch for all of them
        const int m = (int)icp.size();
        trace.inputs_done(st, (int)active.size(), m);
        if (m > 0) {
            cur = icp_seq[0];
            int grid[KD_BATCH_GRID];
            const bool kd = lead->cfg.local_map_type == PLS_MAP_KDTREE;
            if (kd) kdmap_batch_begin(lead, icp.data(), bounds.data(), m, st, grid);
            else projmap_batch_begin(lead, icp.data(), bounds.data(), m, st, grid);
            auto enqueue = [&](int first, int last) {
                if (kd) kdmap_batch_iterations(lead, m, st, grid, first, last);
                else projmap_batch_iterations(lead, icp.data(), bounds.data(), m, st, grid, first, last);
            };
            auto read_done = [&](int* done) {
                if (kd) kdmap_batch_done(lead, m, st, done);
                else projmap_batch_done(lead, m, st, done);
            };
            trace.extra_rounds += icp_rounds(icp.data(), m, enqueue, read_done);
            for (pls_context* ctx : icp) enqueue_result_copy(ctx, st);
            trace.icp_done(st);
            PLS_CUDA(cudaStreamSynchronize(st));
            for (pls_context* ctx : icp) ctx->icp_result = true;
        }
        trace.epilogue_begin();
        // ---- epilogue, per sequence: a failed ICP is that sequence's error alone
        for (int j = 0; j < m; ++j) {
            const int i = icp_seq[j];
            cur = i;
            try {
                frame_epilogue(icp[j], in[i], outputs(i), false, nullptr);
            } catch (const pls::Error& e) {
                if (e.code != PLS_E_SINGULAR) throw;
                icp[j]->err = e.msg;
                status[i] = e.code;
            }
            finished[i] = 1;
        }
        trace.end();
    } catch (...) {
        // a failure no sequence can be blamed for alone (CUDA): every sequence whose frame did not complete reports it;
        // those that completed (a frame 0, a refused input) keep their status
        int code = PLS_E_INVALID;
        std::string msg;
        try {
            throw;
        } catch (const pls::Error& e) {
            code = e.code;
            msg = e.msg;
        } catch (const std::exception& e) {
            msg = e.what();
        }
        for (int i = 0; i < num; ++i) {
            if (!finished[i]) {
                status[i] = code;
                ctxs[i]->err = msg;
            }
            if (out_status) out_status[i] = status[i];
        }
        return code;
    }
    int first_error = PLS_OK;
    for (int i = 0; i < num; ++i) {
        if (out_status) out_status[i] = status[i];
        if (first_error == PLS_OK) first_error = status[i];
    }
    return first_error;
}

}  // extern "C"
