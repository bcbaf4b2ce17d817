// Context lifetime, host<->device argument staging, profiling slots.
#include <utility>

#include "internal.cuh"
#include "kdmap_device.cuh"

namespace pls {

long long g_kernel_launches = 0;

void DBuf::reserve(size_t bytes, cudaStream_t s, bool keep) {
    if (bytes <= cap) return;
    // growth is a stall (stream sync + cudaMalloc + cudaFree): callers that know their steady-state size reserve it
    // up front (kd map: kd_reserve_capacity); everything else grows by half so that a slowly growing buffer settles
    // after a few frames
    size_t want = bytes + bytes / 2 + 256;
    void* np = nullptr;
    PLS_CUDA(cudaStreamSynchronize(s));
    PLS_CUDA(cudaMalloc(&np, want));
    if (p) {
        if (keep) PLS_CUDA(cudaMemcpy(np, p, cap, cudaMemcpyDeviceToDevice));
        PLS_CUDA(cudaFree(p));
    }
    p = np;
    cap = want;
}

void DBuf::reserve_exact(size_t bytes, cudaStream_t s, bool keep) {
    if (bytes <= cap) return;
    void* np = nullptr;
    PLS_CUDA(cudaStreamSynchronize(s));
    PLS_CUDA(cudaMalloc(&np, bytes));
    if (p) {
        if (keep) PLS_CUDA(cudaMemcpy(np, p, cap, cudaMemcpyDeviceToDevice));
        PLS_CUDA(cudaFree(p));
    }
    p = np;
    cap = bytes;
}

void DBuf::release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
}

void HBuf::reserve(size_t bytes) {
    if (bytes <= cap) return;
    if (p) PLS_CUDA(cudaFreeHost(p));
    p = nullptr;
    cap = 0;
    // mapped + portable: kernels may write results straight into it (zero-copy over PCIe), any context may read it
    PLS_CUDA(cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable));
    cap = bytes;
}

void* HBuf::device_ptr() const {
    if (!p) return nullptr;
    void* d = nullptr;
    PLS_CUDA(cudaHostGetDevicePointer(&d, p, 0));
    return d;
}

void HBuf::release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
}

void map_stream_begin(pls_context* ctx) {
    ctx->stream = ctx->stream_map;
    std::swap(ctx->sort, ctx->sort_map);
}

void map_stream_end(pls_context* ctx) {
    cudaEventRecord(ctx->ev_map_done, ctx->stream_map);
    ctx->map_pending = true;
    std::swap(ctx->sort, ctx->sort_map);
    ctx->stream = ctx->stream_main;
}

void map_stream_wait(pls_context* ctx) {
    if (ctx->map_pending) {
        cudaStreamWaitEvent(ctx->stream_main, ctx->ev_map_done, 0);
        ctx->map_pending = false;
    }
}

void sync_all(pls_context* ctx) {
    PLS_CUDA(cudaStreamSynchronize(ctx->stream_map));
    PLS_CUDA(cudaStreamSynchronize(ctx->stream_main));
    ctx->map_pending = false;
}

// Classification cache: cudaPointerGetAttributes costs ~1 us per pointer and a frame passes half a dozen of them, the
// same ones every frame (the caller's pose / info arrays, pinned scan buffers).  Under unified addressing a virtual
// address never changes kind (device allocations live in the driver's reserved range), so the answer is cached per
// address; one host thread drives a context, the cache is thread-local.
namespace {
struct PtrCacheEntry {
    const void* p;
    bool dev;
};
thread_local PtrCacheEntry t_ptr_cache[64] = {};
}  // namespace

bool is_device_ptr(const void* p) {
    if (!p) return false;
    PtrCacheEntry& e = t_ptr_cache[(reinterpret_cast<uintptr_t>(p) >> 6) & 63u];
    if (e.p == p) return e.dev;
    const bool d = is_device_ptr_uncached(p);
    e.p = p;
    e.dev = d;
    return d;
}

bool is_device_ptr_uncached(const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

const void* to_device(pls_context* ctx, const void* p, size_t bytes, DBuf& stage) {
    if (!p || bytes == 0) return p;
    if (is_device_ptr(p)) return p;
    stage.reserve(bytes, ctx->stream);
    PLS_CUDA(cudaMemcpyAsync(stage.p, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return stage.p;
}

OutArg out_arg(pls_context* ctx, void* p, size_t bytes, DBuf& stage) {
    OutArg o;
    o.bytes = bytes;
    if (!p) return o;
    if (is_device_ptr(p)) {
        o.dev = p;
        return o;
    }
    stage.reserve(bytes, ctx->stream);
    o.host = p;
    o.dev = stage.p;
    return o;
}

void finish_out(pls_context* ctx, const OutArg& o, size_t bytes_used) {
    if (!o.host) return;
    size_t b = bytes_used == (size_t)-1 ? o.bytes : bytes_used;
    if (b) PLS_CUDA(cudaMemcpyAsync(o.host, o.dev, b, cudaMemcpyDeviceToHost, ctx->stream));
}

void put_out(void* dst, const void* src, size_t bytes) {
    if (!dst || !bytes) return;
    if (is_device_ptr(dst)) PLS_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    else memcpy(dst, src, bytes);
}

ProfileScope::ProfileScope(pls_context* c, int w, double bytes, bool count) : ctx(c), which(w) {
    ProfileSlot& s = ctx->prof[which];
    if (!s.enabled) return;
    if (s.used >= 4096) {
        cudaStreamSynchronize(ctx->stream_map);
        cudaStreamSynchronize(ctx->stream_main);
        profile_collect(ctx, which);
    }
    if (s.used + 2 > s.pool.size()) {
        for (int i = 0; i < 64; ++i) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return;
            s.pool.push_back(e);
        }
    }
    e0 = s.pool[s.used++];
    e1 = s.pool[s.used++];
    if (count) {
        s.bytes += bytes;
        s.launches += 1;
    }
    cudaEventRecord(e0, ctx->stream);
}

ProfileScope::~ProfileScope() {
    if (e1) cudaEventRecord(e1, ctx->stream);
}

void profile_collect(pls_context* ctx, int which) {
    ProfileSlot& s = ctx->prof[which];
    for (size_t i = 0; i + 1 < s.used; i += 2) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, s.pool[i], s.pool[i + 1]) == cudaSuccess) s.ms += ms;
    }
    s.used = 0;
}

}  // namespace pls

using namespace pls;

extern "C" {

const char* pls_version(void) { return "plslam_b200 0.1 (sm_90a)"; }

int pls_host_fingerprint(const void* host_ptr, int64_t num_bytes, uint64_t* out) {
    if (!host_ptr || !out || num_bytes < 0) return PLS_E_INVALID;
    const int64_t words = num_bytes / 8;
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (uint64_t)num_bytes;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(host_ptr);
    const int64_t step = words > 256 ? words / 256 : 1;
    for (int64_t i = 0; i < words; i += step) {
        uint64_t v;
        memcpy(&v, w + i, 8);
        h = (h ^ v) * 0x100000001B3ull;
        h ^= h >> 29;
    }
    if (words > 0) {
        uint64_t v;
        memcpy(&v, w + words - 1, 8);
        h = (h ^ v) * 0x100000001B3ull;
    }
    *out = h;
    return PLS_OK;
}

int pls_launch_count(int64_t* out) {
    if (!out) return PLS_E_INVALID;
    *out = (int64_t)pls::g_kernel_launches;
    return PLS_OK;
}

int pls_config_default(pls_config* c) {
    if (!c) return PLS_E_INVALID;
    memset(c, 0, sizeof(*c));
    c->height = 64;
    c->width = 2048;
    c->up_fov_deg = 3.0f;
    c->down_fov_deg = -24.0f;
    c->local_map_type = PLS_MAP_KDTREE;
    c->local_map_size = 20;
    c->num_neighbors_normals = 10;
    c->normals_kernel_size = 5;
    c->scheme = PLS_SCHEME_DEFAULT;
    c->sigma = 0.5f;
    c->gn_max_iters = 1;
    c->gn_norm_stop = 1e-3f;
    c->max_num_alignments = 100;
    c->threshold_delta_pose = 1e-4f;
    c->threshold_trans = 0.1f;
    c->threshold_rot = 0.3f;
    c->device = 0;
    c->stream = nullptr;
    return PLS_OK;
}

int pls_create(const pls_config* cfg, pls_context** out) {
    if (!cfg || !out) return PLS_E_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        cudaGetLastError();
        return PLS_E_CUDA;  // no CPU fallback: the product path needs the GPU
    }
    if (cfg->device < 0 || cfg->device >= ndev) return PLS_E_INVALID;
    if (cfg->height <= 0 || cfg->width <= 0 || cfg->local_map_size <= 0) return PLS_E_INVALID;
    if (cfg->max_num_alignments < 1 || cfg->max_num_alignments > kMaxAlign) return PLS_E_INVALID;
    if (cfg->num_neighbors_normals < 3 || cfg->num_neighbors_normals + 1 > KD_KMAX_WIDE) return PLS_E_INVALID;
    if (cfg->normals_kernel_size < 1 || cfg->normals_kernel_size > 9 || (cfg->normals_kernel_size % 2) == 0)
        return PLS_E_INVALID;
    pls_context* ctx = new pls_context();
    ctx->cfg = *cfg;
    try {
        PLS_CUDA(cudaSetDevice(cfg->device));
        if (cfg->stream) {
            ctx->stream = (cudaStream_t)cfg->stream;
        } else {
            // the frame's own work (subsample, ICP) is what the caller waits for: it outranks the local-map update that
            // runs beside it on the second stream (PLS_STREAM_PRIORITY=0: both at the default priority, for A/B runs)
            static const bool prio = !(getenv("PLS_STREAM_PRIORITY") && atoi(getenv("PLS_STREAM_PRIORITY")) == 0);
            int least = 0, greatest = 0;
            PLS_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
            PLS_CUDA(cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio ? greatest : 0));
            ctx->own_stream = true;
        }
        ctx->stream_main = ctx->stream;
        {
            static const bool prio = !(getenv("PLS_STREAM_PRIORITY") && atoi(getenv("PLS_STREAM_PRIORITY")) == 0);
            int least = 0, greatest = 0;
            PLS_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
            PLS_CUDA(cudaStreamCreateWithPriority(&ctx->stream_map, cudaStreamNonBlocking, prio ? least : 0));
        }
        PLS_CUDA(cudaEventCreateWithFlags(&ctx->ev_map_done, cudaEventDisableTiming));
        ctx->pinned.reserve(kScalarOffset + 256);  // FrameResult, then the host copy of the u32 scalars
        ctx->scalars.reserve(sizeof(FrameResult) + 4096, ctx->stream);
        PLS_CUDA(cudaMemsetAsync(ctx->scalars.p, 0, ctx->scalars.cap, ctx->stream));
        odometry_reset(ctx);
    } catch (const pls::Error& e) {
        fprintf(stderr, "pls_create: %s\n", e.msg.c_str());
        delete ctx;
        return e.code;
    }
    *out = ctx;
    return PLS_OK;
}

int pls_destroy(pls_context* ctx) {
    if (!ctx) return PLS_E_INVALID;
    cudaSetDevice(ctx->cfg.device);
    ctx->upd_pending = false;  // a map update that was never enqueued dies with the context
    cudaStreamSynchronize(ctx->stream_map);
    cudaStreamSynchronize(ctx->stream_main);
    comm_free(ctx);
    if (ctx->p2p_pending_xchg) cudaFree(ctx->p2p_pending_xchg);
    for (auto& b : ctx->stage_in) b.release();
    for (auto& b : ctx->stage_out) b.release();
    for (auto& b : ctx->tmp) b.release();
    for (auto& b : ctx->next_buf) b.release();
    ctx->pinned.release();
    ctx->scalars.release();
    ctx->sort.keys_alt.release(); ctx->sort.vals_alt.release(); ctx->sort.hist.release();
    ctx->sort.status.release(); ctx->sort.plan.release();
    ctx->sort_map.keys_alt.release(); ctx->sort_map.vals_alt.release(); ctx->sort_map.hist.release();
    ctx->sort_map.status.release(); ctx->sort_map.plan.release();
    ctx->scan.status.release();
    ctx->sel[0].status.release(); ctx->sel[1].status.release(); ctx->input_zbuf.release();
    for (auto& b : ctx->kd.store) b.release();
    ctx->kd.morton.release(); ctx->kd.order.release(); ctx->kd.sorted.release(); ctx->kd.sorted_prev.release(); ctx->kd.normals.release();
    ctx->kd.bbox.release(); ctx->kd.grid_hdr.release(); ctx->kd.cells.release(); ctx->kd.stats.release();
    ctx->kd_worklist.release(); ctx->kd_nn_state.release();
    ctx->pm.vmaps.release(); ctx->pm.nmaps.release(); ctx->pm.poses.release();
    ctx->pm.model_v.release(); ctx->pm.model_n.release(); ctx->pm.zbuf.release();
    for (auto& b : ctx->frame_vmap_buf) b.release();
    for (auto& b : ctx->frame_pts_buf) b.release();
    ctx->queries.release(); ctx->nn_prev.release();
    ctx->partials.release(); ctx->batch_buf.release(); ctx->hyp_buf.release(); ctx->degen_buf.release(); ctx->gs_keys.release(); ctx->gs_vals.release(); ctx->gs_out_xyz.release();
    ctx->gs_out_idx.release(); ctx->gs_bins.release(); ctx->gs_buckets.release();
    for (auto& s : ctx->prof)
        for (auto e : s.pool) cudaEventDestroy(e);
    if (ctx->ev_map_done) cudaEventDestroy(ctx->ev_map_done);
    if (ctx->ev_inputs) cudaEventDestroy(ctx->ev_inputs);
    if (ctx->ev_batch) cudaEventDestroy(ctx->ev_batch);
    if (ctx->ev_icp_done) cudaEventDestroy(ctx->ev_icp_done);
    ctx->gs_host_xyz.release(); ctx->gs_host_idx.release();
    if (ctx->stream_map) cudaStreamDestroy(ctx->stream_map);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream_main);
    delete ctx;
    return PLS_OK;
}

const char* pls_last_error(pls_context* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int pls_synchronize(pls_context* ctx) {
    PLS_API_BEGIN(ctx)
    sync_all(ctx);
    PLS_API_END(ctx)
}

int pls_wait_stream(pls_context* ctx, void* other_stream) {
    PLS_API_BEGIN(ctx)
    // work the caller enqueued on `other_stream` (e.g. PyTorch's current stream: the kernels that produced a CUDA
    // tensor handed to this library) happens-before everything this context launches from now on; no host sync
    cudaStream_t other = (cudaStream_t)other_stream;
    if (other != ctx->stream_main) {
        if (!ctx->ev_inputs) PLS_CUDA(cudaEventCreateWithFlags(&ctx->ev_inputs, cudaEventDisableTiming));
        PLS_CUDA(cudaEventRecord(ctx->ev_inputs, other));
        PLS_CUDA(cudaStreamWaitEvent(ctx->stream_main, ctx->ev_inputs, 0));
    }
    PLS_API_END(ctx)
}

int pls_profile_enable(pls_context* ctx, int which, int enable) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(which >= 0 && which < kProfileSlots, "pls_profile_enable: bad slot");
    ctx->prof[which].enabled = enable != 0;
    PLS_API_END(ctx)
}

int pls_profile_read(pls_context* ctx, int which, double* ms_total, int64_t* launches, double* bytes, int reset) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(which >= 0 && which < kProfileSlots, "pls_profile_read: bad slot");
    sync_all(ctx);
    profile_collect(ctx, which);
    ProfileSlot& s = ctx->prof[which];
    if (ms_total) *ms_total = s.ms;
    if (launches) *launches = s.launches;
    if (bytes) *bytes = s.bytes;
    if (reset) {
        s.ms = 0;
        s.launches = 0;
        s.bytes = 0;
    }
    PLS_API_END(ctx)
}

}  // extern "C"
