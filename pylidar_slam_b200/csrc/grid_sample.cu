// K1 -- voxel-grid subsample.
//
//   voxel_hash_kernel : voxel coordinate = int64(round_half_even(double(p) / voxel)) per axis
//                       and hash = 73856093 x + 19349669 y + 83492791 z in signed 64-bit
//                       (slam/common/pointcloud.py:13-23,40-79).  Also emits the sort key
//                       (hash with the sign bit flipped -> unsigned order == signed order).
//   radix sort        : stable, so equal hashes keep ascending point index.  The hashes of a LiDAR frame span ~2^38
//                       (|voxel coordinate| <~ 1000), so the sort runs on 40-bit biased keys -- 5 passes instead of the
//                       8 a raw int64 needs; a hash outside [-2^39, 2^39) stamps an overflow word and the caller,
//                       which reads the sample count back anyway, repeats the call on full 64-bit keys.
//   head flags + scan : first element of each run of equal hashes == np.unique(...,
//                       return_index=True)'s first occurrence (pointcloud.py:177,193).
//   gather            : sample_points / sample_indices in ascending-hash order.
#include "internal.cuh"
#include "select_device.cuh"

namespace pls {

namespace {

constexpr long long HX = 73856093ll, HY = 19349669ll, HZ = 83492791ll;

constexpr int GS_COMPACT_BITS = 40;

template <typename T>
__global__ void voxel_hash_kernel(const T* __restrict__ xyz, int64_t n, double voxel, long long* __restrict__ coords,
                                  long long* __restrict__ hashes, uint64_t* __restrict__ keys,
                                  uint32_t* __restrict__ vals, uint32_t* __restrict__ overflow = nullptr,
                                  uint32_t stamp = 0, double voxel_y = -1.0, double voxel_z = -1.0) {
    if (voxel_y < 0.0) voxel_y = voxel;   // voxelise's defaults (pointcloud.py:66-69)
    if (voxel_z < 0.0) voxel_z = voxel;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double x = (double)xyz[3 * i], y = (double)xyz[3 * i + 1], z = (double)xyz[3 * i + 2];
        long long cx = voxel_coord(x, voxel);
        long long cy = voxel_coord(y, voxel_y);
        long long cz = voxel_coord(z, voxel_z);
        // modulo 2^64 like numba's int64 arithmetic: signed overflow would be undefined behaviour
        const long long h = (long long)((uint64_t)HX * (uint64_t)cx + (uint64_t)HY * (uint64_t)cy + (uint64_t)HZ * (uint64_t)cz);
        if (coords) {
            coords[3 * i] = cx;
            coords[3 * i + 1] = cy;
            coords[3 * i + 2] = cz;
        }
        if (hashes) hashes[i] = h;
        if (keys) {
            if (overflow) {  // compact keys: h + 2^39 in 40 bits keeps the signed order
                const uint64_t hb = (uint64_t)h + (1ull << (GS_COMPACT_BITS - 1));  // modular: no signed overflow
                if (hb >> GS_COMPACT_BITS) *overflow = stamp;
                keys[i] = hb & ((1ull << GS_COMPACT_BITS) - 1ull);
            } else {
                keys[i] = (uint64_t)h ^ 0x8000000000000000ull;
            }
            vals[i] = (uint32_t)i;
        }
    }
}

__global__ void head_flags_kernel(const uint64_t* __restrict__ keys, int64_t n, uint8_t* __restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

template <typename T>
__global__ void gather_samples_kernel(const T* __restrict__ xyz, const uint32_t* __restrict__ vals,
                                      const uint8_t* __restrict__ flags, const uint32_t* __restrict__ pos, int64_t n,
                                      T* __restrict__ out_xyz, long long* __restrict__ out_idx) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[i]) continue;
        uint32_t src = vals[i];
        uint32_t dst = pos[i];
        const T x = xyz[3 * (size_t)src], y = xyz[3 * (size_t)src + 1], z = xyz[3 * (size_t)src + 2];
        if (out_idx) out_idx[dst] = (long long)src;
        out_xyz[3 * (size_t)dst] = x;
        out_xyz[3 * (size_t)dst + 1] = y;
        out_xyz[3 * (size_t)dst + 2] = z;
    }
}

// The host copy of a subsample: `count` (a device scalar -- the host does not know it yet) rows of two device arrays
// into mapped pinned host memory with 16-byte stores, a warp writing 512 contiguous bytes per instruction.  (Letting
// the selection kernel itself write its 4- and 8-byte results across PCIe made that kernel much slower; a DMA copy
// would need the count on the host first, i.e. a second round trip.)
__global__ void __launch_bounds__(256)
copy_counted_to_host_kernel(const unsigned char* __restrict__ src_a, unsigned char* __restrict__ dst_a, size_t elem_a,
                            const unsigned char* __restrict__ src_b, unsigned char* __restrict__ dst_b, size_t elem_b,
                            const uint32_t* __restrict__ count_dev) {
    const size_t na = (size_t)*count_dev * elem_a, nb = (size_t)*count_dev * elem_b;
    const size_t va = na / 16, vb = nb / 16;
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = gtid; i < va + vb; i += stride) {
        if (i < va) reinterpret_cast<uint4*>(dst_a)[i] = reinterpret_cast<const uint4*>(src_a)[i];
        else reinterpret_cast<uint4*>(dst_b)[i - va] = reinterpret_cast<const uint4*>(src_b)[i - va];
    }
    if (gtid < 16) {
        size_t o = va * 16 + gtid;
        if (o < na) dst_a[o] = src_a[o];
        o = vb * 16 + gtid;
        if (o < nb) dst_b[o] = src_b[o];
    }
}

// Run heads of the sorted keys -> samples, in ONE selection pass (select_device.cuh): element i is kept iff its key
// differs from its predecessor's; the kept element's original index is vals[i].
template <typename T>
struct GridSampleSelect {
    const uint64_t* keys;
    const uint32_t* vals;
    const T* xyz;
    T* out_xyz;
    long long* out_idx;
    struct State {};
    __device__ __forceinline__ uint32_t flags(int64_t i, State&) const { return (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u; }
    __device__ __forceinline__ void emit(int64_t i, int, uint32_t dst, const State&) const {
        const uint32_t src = vals[i];
        const T x = xyz[3 * (size_t)src], y = xyz[3 * (size_t)src + 1], z = xyz[3 * (size_t)src + 2];
        if (out_idx) out_idx[dst] = (long long)src;
        out_xyz[3 * (size_t)dst] = x;
        out_xyz[3 * (size_t)dst + 1] = y;
        out_xyz[3 * (size_t)dst + 2] = z;
    }
};

// ---- voxel statistics (Voxelization filter) ---------------------------------------------------------------
// After the same hash + stable sort as the subsample: rank of every run of equal hashes = voxel id
// (pointcloud.py:99-150 walks the sorted hashes the same way), scattered back to the points' original order.
__global__ void voxel_ids_kernel(const uint32_t* __restrict__ vals, const uint8_t* __restrict__ flags,
                                 const uint32_t* __restrict__ pos, int64_t n, long long* __restrict__ ids_out,
                                 uint32_t* __restrict__ starts) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t id = pos[i] + flags[i] - 1u;  // pos = number of run heads before i
        ids_out[vals[i]] = (long long)id;
        if (flags[i]) starts[id] = (uint32_t)i;
    }
}

// One warp per voxel: lanes stride over the voxel's points (gathered through the sorted index), float64 sums,
// fixed-order shuffle reduction (deterministic); two sweeps -- mean, then the scatter matrix
// sum (x - mean)(x - mean)^T, which the reference does NOT divide by the count (pointcloud.py:126-131).
template <typename T>
__global__ void __launch_bounds__(256)
voxel_stats_kernel(const T* __restrict__ xyz, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ starts,
                   const uint32_t* __restrict__ count_dev, int64_t n, long long* __restrict__ sizes,
                   T* __restrict__ means, T* __restrict__ covs) {
    const uint32_t V = *count_dev;
    const int lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < V; v += warps) {
        const uint32_t b = starts[v];
        const uint32_t e = (v + 1 < V) ? starts[v + 1] : (uint32_t)n;
        double sx = 0.0, sy = 0.0, sz = 0.0;
        for (uint32_t j = b + lane; j < e; j += 32) {
            const size_t src = vals[j];
            sx += (double)xyz[3 * src];
            sy += (double)xyz[3 * src + 1];
            sz += (double)xyz[3 * src + 2];
        }
        sx = warp_sum(sx); sy = warp_sum(sy); sz = warp_sum(sz);
        const double cnt = (double)(e - b);
        const double mx = sx / cnt, my = sy / cnt, mz = sz / cnt;
        double cxx = 0.0, cxy = 0.0, cxz = 0.0, cyy = 0.0, cyz = 0.0, czz = 0.0;
        for (uint32_t j = b + lane; j < e; j += 32) {
            const size_t src = vals[j];
            const double dx = (double)xyz[3 * src] - mx, dy = (double)xyz[3 * src + 1] - my, dz = (double)xyz[3 * src + 2] - mz;
            cxx += dx * dx; cxy += dx * dy; cxz += dx * dz;
            cyy += dy * dy; cyz += dy * dz; czz += dz * dz;
        }
        cxx = warp_sum(cxx); cxy = warp_sum(cxy); cxz = warp_sum(cxz);
        cyy = warp_sum(cyy); cyz = warp_sum(cyz); czz = warp_sum(czz);
        if (lane == 0) {
            sizes[v] = (long long)(e - b);
            means[3 * (size_t)v] = (T)mx; means[3 * (size_t)v + 1] = (T)my; means[3 * (size_t)v + 2] = (T)mz;
            T* c = covs + 9 * (size_t)v;
            c[0] = (T)cxx; c[1] = (T)cxy; c[2] = (T)cxz;
            c[3] = (T)cxy; c[4] = (T)cyy; c[5] = (T)cyz;
            c[6] = (T)cxz; c[7] = (T)cyz; c[8] = (T)czz;
        }
    }
}

inline int grid_for(int64_t n, int threads = 256) {
    int64_t b = (n + threads - 1) / threads;
    int64_t cap = 8 * kNumSMs;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

// Device-resident grid sample: xyz_dev [n,3] -> out_xyz_dev [<=n,3], out_idx_dev [<=n] (nullable);
// the sample count lands in the device scalar SC_GS_COUNT.  compact: sort on GS_COMPACT_BITS-bit keys, stamping gs_seq
// into SC_GS_OVERFLOW if a hash does not fit them.
template <typename T>
void grid_sample_device(pls_context* ctx, const T* xyz_dev, int64_t n, double voxel, T* out_xyz_dev,
                        long long* out_idx_dev, bool compact, T* host_xyz, long long* host_idx) {
    cudaStream_t st = ctx->stream;
    ProfileScope ps(ctx, 4, (double)n * 3 * sizeof(T));
    ctx->gs_keys.reserve((size_t)n * sizeof(uint64_t), st);
    ctx->gs_vals.reserve((size_t)n * sizeof(uint32_t), st);
    ctx->tmp[1].reserve((size_t)n, st);                    // head flags
    ctx->tmp[2].reserve((size_t)n * sizeof(uint32_t), st); // positions
    if (host_xyz && host_idx && !out_idx_dev) {            // the host copy is made from device arrays: indices too
        ctx->gs_out_idx.reserve((size_t)n * sizeof(long long), st);
        out_idx_dev = ctx->gs_out_idx.as<long long>();
    }
    auto copy_to_host = [&]() {
        if (!host_xyz || !host_idx) return;
        const size_t bytes = (size_t)n * (3 * sizeof(T) + sizeof(long long));
        copy_counted_to_host_kernel<<<grid_for((int64_t)(bytes / 16)), 256, 0, st>>>(
            reinterpret_cast<const unsigned char*>(out_xyz_dev), reinterpret_cast<unsigned char*>(host_xyz), 3 * sizeof(T),
            reinterpret_cast<const unsigned char*>(out_idx_dev), reinterpret_cast<unsigned char*>(host_idx), sizeof(long long),
            scalar_u32(ctx, SC_GS_COUNT));
        PLS_CHECK_LAUNCH();
    };
    if (compact) {
        ctx->gs_seq += 1;
        if (ctx->gs_seq == 0) ctx->gs_seq = 1;
    }
    voxel_hash_kernel<T><<<grid_for(n), 256, 0, st>>>(xyz_dev, n, voxel, nullptr, nullptr, ctx->gs_keys.as<uint64_t>(),
                                                      ctx->gs_vals.as<uint32_t>(),
                                                      compact ? scalar_u32(ctx, SC_GS_OVERFLOW) : nullptr, ctx->gs_seq);
    PLS_CHECK_LAUNCH();
    uint64_t* sk;
    uint32_t* sv;
    radix_sort_pairs(ctx, ctx->gs_keys.as<uint64_t>(), ctx->gs_vals.as<uint32_t>(), n, compact ? GS_COMPACT_BITS / 8 : 8, &sk, &sv);
    if (n <= SEL_MAX_N) {
        GridSampleSelect<T> op{sk, sv, xyz_dev, out_xyz_dev, out_idx_dev};
        select_launch(ctx, op, n, nullptr, scalar_u32(ctx, SC_GS_COUNT), nullptr);
        copy_to_host();
        return;
    }
    // clouds beyond the single-wave selection: flags, scan, gather
    head_flags_kernel<<<grid_for(n), 256, 0, st>>>(sk, n, ctx->tmp[1].as<uint8_t>());
    PLS_CHECK_LAUNCH();
    exclusive_scan_flags(ctx, ctx->tmp[1].as<uint8_t>(), n, ctx->tmp[2].as<uint32_t>(), scalar_u32(ctx, SC_GS_COUNT));
    gather_samples_kernel<T><<<grid_for(n), 256, 0, st>>>(xyz_dev, sv, ctx->tmp[1].as<uint8_t>(),
                                                          ctx->tmp[2].as<uint32_t>(), n, out_xyz_dev, out_idx_dev);
    PLS_CHECK_LAUNCH();
    copy_to_host();
}

// Voxelization.filter (preprocessing.py:71-97): coordinates, hashes and the per-voxel normal distribution.
template <typename T>
void voxel_statistics_device(pls_context* ctx, const T* xyz_dev, int64_t n, double voxel, long long* coords_dev,
                             long long* hashes_dev, long long* sizes_dev, T* means_dev, T* covs_dev, long long* ids_dev) {
    cudaStream_t st = ctx->stream;
    ctx->gs_keys.reserve((size_t)n * sizeof(uint64_t), st);
    ctx->gs_vals.reserve((size_t)n * sizeof(uint32_t), st);
    ctx->next_buf[1].reserve((size_t)n, st);                    // run-head flags
    ctx->next_buf[2].reserve((size_t)n * sizeof(uint32_t), st); // heads before i
    ctx->next_buf[3].reserve((size_t)n * sizeof(uint32_t), st); // first sorted position of every voxel
    voxel_hash_kernel<T><<<grid_for(n), 256, 0, st>>>(xyz_dev, n, voxel, coords_dev, hashes_dev, ctx->gs_keys.as<uint64_t>(),
                                                      ctx->gs_vals.as<uint32_t>());
    PLS_CHECK_LAUNCH();
    uint64_t* sk;
    uint32_t* sv;
    radix_sort_pairs(ctx, ctx->gs_keys.as<uint64_t>(), ctx->gs_vals.as<uint32_t>(), n, 8, &sk, &sv);
    uint8_t* flags = ctx->next_buf[1].as<uint8_t>();
    uint32_t* pos = ctx->next_buf[2].as<uint32_t>();
    uint32_t* starts = ctx->next_buf[3].as<uint32_t>();
    head_flags_kernel<<<grid_for(n), 256, 0, st>>>(sk, n, flags);
    PLS_CHECK_LAUNCH();
    exclusive_scan_flags(ctx, flags, n, pos, scalar_u32(ctx, SC_GS_COUNT));
    voxel_ids_kernel<<<grid_for(n), 256, 0, st>>>(sv, flags, pos, n, ids_dev, starts);
    PLS_CHECK_LAUNCH();
    voxel_stats_kernel<T><<<grid_for(n * 32), 256, 0, st>>>(xyz_dev, sv, starts, scalar_u32(ctx, SC_GS_COUNT), n, sizes_dev,
                                                           means_dev, covs_dev);
    PLS_CHECK_LAUNCH();
}

namespace {

void grid_sample_count_to_host(pls_context* ctx) {
    // into the pinned block behind the host FrameResult: a pageable destination would make the copy synchronous
    // through the driver's own staging buffer
    uint32_t* words = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(ctx->pinned.p) + kScalarOffset);
    static_assert(SC_GS_COUNT == 0 && SC_GS_OVERFLOW == 7, "one 32-byte copy covers the count and the overflow stamp");
    PLS_CUDA(cudaMemcpyAsync(words, scalar_u32(ctx, SC_GS_COUNT), 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
}

void grid_sample_launch(pls_context* ctx, const GridSample& g, bool compact) {
    if (!g.f64)
        grid_sample_device<float>(ctx, (const float*)g.xyz, g.n, g.voxel, (float*)g.out_xyz, g.out_idx, compact,
                                  (float*)g.host_xyz, g.host_idx);
    else
        grid_sample_device<double>(ctx, (const double*)g.xyz, g.n, g.voxel, (double*)g.out_xyz, g.out_idx, compact,
                                   (double*)g.host_xyz, g.host_idx);
}

}  // namespace

void grid_sample_enqueue(pls_context* ctx, const GridSample& g, bool count_to_host) {
    grid_sample_launch(ctx, g, true);
    if (count_to_host) grid_sample_count_to_host(ctx);
}

uint32_t grid_sample_host_count(pls_context* ctx, bool* overflowed) {
    const uint32_t* words = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(ctx->pinned.p) + kScalarOffset);
    *overflowed = ctx->gs_seq != 0 && words[SC_GS_OVERFLOW] == ctx->gs_seq;
    return words[SC_GS_COUNT];
}

uint32_t grid_sample_finish(pls_context* ctx, const GridSample& g) {
    bool overflowed = false;
    const uint32_t count = grid_sample_host_count(ctx, &overflowed);
    if (!overflowed) return count;
    // hashes beyond 40 bits: once more on the raw 64-bit keys
    grid_sample_launch(ctx, g, false);
    grid_sample_count_to_host(ctx);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    return grid_sample_host_count(ctx, &overflowed);
}

}  // namespace pls

using namespace pls;

extern "C" {

int pls_voxel_hash_xyz(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel_x, double voxel_y, double voxel_z,
                       int64_t* coords_out, int64_t* hashes_out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(xyz && n > 0 && voxel_x > 0.0 && voxel_y > 0.0 && voxel_z > 0.0, "pls_voxel_hash: need [n,3] points and voxel sizes > 0");
    const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
    const void* d_xyz = to_device(ctx, xyz, (size_t)n * 3 * esz, ctx->stage_in[0]);
    OutArg oc = out_arg(ctx, coords_out, (size_t)n * 3 * sizeof(int64_t), ctx->stage_out[0]);
    OutArg oh = out_arg(ctx, hashes_out, (size_t)n * sizeof(int64_t), ctx->stage_out[1]);
    if (is_f64)
        voxel_hash_kernel<double><<<grid_for(n), 256, 0, ctx->stream>>>((const double*)d_xyz, n, voxel_x, (long long*)oc.dev,
                                                                       (long long*)oh.dev, nullptr, nullptr, nullptr, 0, voxel_y,
                                                                       voxel_z);
    else
        voxel_hash_kernel<float><<<grid_for(n), 256, 0, ctx->stream>>>((const float*)d_xyz, n, voxel_x, (long long*)oc.dev,
                                                                      (long long*)oh.dev, nullptr, nullptr, nullptr, 0, voxel_y,
                                                                      voxel_z);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, oc);
    finish_out(ctx, oh);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_voxel_hash(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel, int64_t* coords_out,
                   int64_t* hashes_out) {
    return pls_voxel_hash_xyz(ctx, xyz, is_f64, n, voxel, voxel, voxel, coords_out, hashes_out);
}

int pls_grid_sample(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel, void* out_xyz,
                    int64_t* out_idx, int64_t* out_count) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(xyz && out_xyz && out_count && n > 0 && voxel > 0.0, "pls_grid_sample: bad arguments");
    const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
    const void* d_xyz = to_device(ctx, xyz, (size_t)n * 3 * esz, ctx->stage_in[0]);
    OutArg ox = out_arg(ctx, out_xyz, (size_t)n * 3 * esz, ctx->stage_out[0]);
    OutArg oi = out_arg(ctx, out_idx, (size_t)n * sizeof(int64_t), ctx->stage_out[1]);
    const GridSample g{d_xyz, is_f64 != 0, n, voxel, ox.dev, (long long*)oi.dev, nullptr, nullptr};
    grid_sample_enqueue(ctx, g);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    const uint32_t count = grid_sample_finish(ctx, g);
    *out_count = count;
    finish_out(ctx, ox, (size_t)count * 3 * esz);
    finish_out(ctx, oi, (size_t)count * sizeof(int64_t));
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_grid_sample_staged(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel,
                           const void** out_xyz_host, const int64_t** out_idx_host, const void** out_xyz_dev,
                           int64_t* out_count) {
    PLS_API_BEGIN_FRAME(ctx)
    PLS_REQUIRE(xyz && out_xyz_host && out_idx_host && out_count && n > 0 && voxel > 0.0, "pls_grid_sample_staged: bad arguments");
    const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
    const void* d_xyz = to_device(ctx, xyz, (size_t)n * 3 * esz, ctx->stage_in[0]);
    // one device-resident copy (what pls_process_frame consumes without a host hop) and one in mapped pinned memory,
    // written by the gather kernel itself; a single stream synchronisation ends the call
    DBuf& dev_xyz = is_f64 ? ctx->stage_out[0] : ctx->gs_out_xyz;
    dev_xyz.reserve((size_t)n * 3 * esz, ctx->stream);
    void* host_xyz = const_cast<void*>(*out_xyz_host);
    int64_t* host_idx = const_cast<int64_t*>(*out_idx_host);
    void *map_xyz = nullptr, *map_idx = nullptr;  // the device-side aliases the gather kernel writes through
    if (host_xyz && host_idx) {
        PLS_REQUIRE(cudaHostGetDevicePointer(&map_xyz, host_xyz, 0) == cudaSuccess &&
                        cudaHostGetDevicePointer(&map_idx, host_idx, 0) == cudaSuccess,
                    "pls_grid_sample_staged: caller-owned staging must come from pls_pinned_alloc");
    } else {
        ctx->gs_host_xyz.reserve((size_t)n * 3 * esz);
        ctx->gs_host_idx.reserve((size_t)n * sizeof(int64_t));
        host_xyz = ctx->gs_host_xyz.p;
        host_idx = ctx->gs_host_idx.as<int64_t>();
        map_xyz = ctx->gs_host_xyz.device_ptr();
        map_idx = ctx->gs_host_idx.device_ptr();
    }
    const GridSample g{d_xyz, is_f64 != 0, n, voxel, dev_xyz.p, nullptr, map_xyz, (long long*)map_idx};
    grid_sample_enqueue(ctx, g);
    flush_map_update(ctx);  // the last frame's local-map update is enqueued while the subsample runs
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    *out_count = grid_sample_finish(ctx, g);
    *out_xyz_host = host_xyz;
    *out_idx_host = host_idx;
    if (out_xyz_dev) *out_xyz_dev = dev_xyz.p;
    PLS_API_END(ctx)
}

int pls_pinned_alloc(int64_t num_bytes, void** out_ptr) {
    if (!out_ptr || num_bytes <= 0) return PLS_E_INVALID;
    void* p = nullptr;
    if (cudaHostAlloc(&p, (size_t)num_bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        return PLS_E_CUDA;
    }
    *out_ptr = p;
    return PLS_OK;
}

int pls_pinned_free(void* ptr) {
    if (!ptr) return PLS_OK;
    if (cudaFreeHost(ptr) != cudaSuccess) {
        cudaGetLastError();
        return PLS_E_CUDA;
    }
    return PLS_OK;
}

int pls_voxel_statistics(pls_context* ctx, const void* xyz, int is_f64, int64_t n, double voxel, int64_t* coords_out,
                         int64_t* hashes_out, int64_t* sizes_out, void* means_out, void* covs_out, int64_t* ids_out,
                         int64_t* out_count) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(xyz && sizes_out && means_out && covs_out && ids_out && out_count && n > 0 && voxel > 0.0,
                "pls_voxel_statistics: bad arguments");
    PLS_REQUIRE(n < (1ll << 31), "pls_voxel_statistics: too many points");
    const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
    const void* d_xyz = to_device(ctx, xyz, (size_t)n * 3 * esz, ctx->stage_in[0]);
    OutArg oc = out_arg(ctx, coords_out, (size_t)n * 3 * sizeof(int64_t), ctx->stage_out[0]);
    OutArg oh = out_arg(ctx, hashes_out, (size_t)n * sizeof(int64_t), ctx->stage_out[1]);
    OutArg os = out_arg(ctx, sizes_out, (size_t)n * sizeof(int64_t), ctx->stage_out[2]);
    OutArg om = out_arg(ctx, means_out, (size_t)n * 3 * esz, ctx->stage_out[3]);
    OutArg ov = out_arg(ctx, covs_out, (size_t)n * 9 * esz, ctx->stage_out[4]);
    OutArg oi = out_arg(ctx, ids_out, (size_t)n * sizeof(int64_t), ctx->stage_out[5]);
    if (is_f64)
        voxel_statistics_device<double>(ctx, (const double*)d_xyz, n, voxel, (long long*)oc.dev, (long long*)oh.dev,
                                        (long long*)os.dev, (double*)om.dev, (double*)ov.dev, (long long*)oi.dev);
    else
        voxel_statistics_device<float>(ctx, (const float*)d_xyz, n, voxel, (long long*)oc.dev, (long long*)oh.dev,
                                       (long long*)os.dev, (float*)om.dev, (float*)ov.dev, (long long*)oi.dev);
    uint32_t count = 0;
    PLS_CUDA(cudaMemcpyAsync(&count, scalar_u32(ctx, SC_GS_COUNT), sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    *out_count = count;
    finish_out(ctx, oc);
    finish_out(ctx, oh);
    finish_out(ctx, os, (size_t)count * sizeof(int64_t));
    finish_out(ctx, om, (size_t)count * 3 * esz);
    finish_out(ctx, ov, (size_t)count * 9 * esz);
    finish_out(ctx, oi);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

}  // extern "C"
