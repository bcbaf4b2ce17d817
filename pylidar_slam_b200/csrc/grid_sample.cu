// K1 -- voxel-grid subsample.
//
// Compact keys, n <= SEL_MAX_N (every frame of the kd path): three launches, no memset.
//   gs_hash_bins_kernel      : the hash below, composite key key40 << 24 | index, counts of 2^16 bins (top 16 key
//                              bits); the last block turns the occupied bins into offsets and cuts buckets of whole bins
//   gs_bucket_scatter_kernel : every key to its bin's cursor -- each bucket lands in its own slice
//   gs_bucket_select_kernel  : a block per bucket sorts it by composite key (the smallest index of a run sorts first),
//                              keeps the run heads and chains the buckets' counts to place them
// Larger clouds and the 64-bit replay after an overflow take the path below:
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

// ---- bucket grid sample (compact keys, n <= SEL_MAX_N) -------------------------------------------------------
// Composite key = key40 << 24 | point index: sorted, the head of every run of equal key40 is its smallest index, so no
// stable sort is needed.  Bins are the top 16 bits of key40 (2^24 hash units each): LiDAR hashes crowd around 0, and
// fine bins keep the buckets cut from them balanced.
constexpr int GS_BIN_BITS = 16;
constexpr int GS_BINS = 1 << GS_BIN_BITS;
constexpr int GS_IDX_BITS = 24;
constexpr uint64_t GS_IDX_MASK = (1ull << GS_IDX_BITS) - 1ull;
constexpr uint32_t GS_BUCKET_TARGET = 1024;  // bucket b: the bins whose first key ranks in [b, b + 1) * GS_BUCKET_TARGET
constexpr uint32_t GS_BUCKET_CAP = 4096;     // the largest bucket sorted in shared memory (32 KB of keys)
constexpr int GS_SELECT_THREADS = 512;
constexpr int GS_SCAN_ITEMS = 8;             // bins per thread and tile in the hash kernel's offset scan
constexpr uint32_t GS_FLAG_AGG = 1u << 30, GS_FLAG_PREFIX = 2u << 30, GS_VALUE_MASK = (1u << 30) - 1u;
// control words behind the bins: the hash kernel's last-block ticket, the occupied bin range while it is being taken
// (65535 - lowest bin, highest bin: both start at 0), that range for the select kernel, the select kernel's bucket ticket
enum { GSW_TICKET = 0, GSW_LO_INV, GSW_HI, GSW_RANGE_LO, GSW_RANGE_HI, GSW_BUCKET_TICKET, GSW_WORDS = 8 };

__device__ __forceinline__ uint32_t gs_ld_volatile(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void gs_st_volatile(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Exclusive scan of one value per thread over the block; `total` gets the sum.  Every thread of the block calls it.
__device__ __forceinline__ uint32_t gs_block_scan(uint32_t v, uint32_t* s_warp, uint32_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t before = 0, tot = 0;
    for (int w = 0; w < warps; ++w) {
        const uint32_t c = s_warp[w];
        before += w < warp ? c : 0u;
        tot += c;
    }
    __syncthreads();  // s_warp is free for the next scan
    total = tot;
    return before + inc - v;
}

// K1: the voxel hash of voxel_hash_kernel, the composite key with the overflow stamp, and the bin counts.  The block
// that finishes last turns the counts of the occupied bin range into exclusive offsets in place (the scatter's
// cursors) and cuts the buckets; it also resets the control words for the next call.
template <typename T>
__global__ void __launch_bounds__(256)
gs_hash_bins_kernel(const T* __restrict__ xyz, int64_t n, double voxel, uint64_t* __restrict__ keys, uint32_t* bins,
                    uint32_t* words, uint32_t* __restrict__ bucket_start, uint32_t* __restrict__ status, int num_buckets,
                    uint32_t* __restrict__ overflow, uint32_t stamp) {
    __shared__ uint32_t s_lo_inv, s_hi, s_warp[8];
    __shared__ int s_last;
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) s_lo_inv = s_hi = 0u;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // the select kernel's look-back words (the last call's select kernel has completed)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + tid; i <= num_buckets; i += stride) status[i] = 0u;
    // warp-uniform trip count: the match below needs every lane
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (tid & ~31); base < n; base += stride) {
        const int64_t i = base + lane;
        const bool valid = i < n;
        uint32_t bin = 0xffffffffu;
        if (valid) {
            const long long cx = voxel_coord((double)xyz[3 * i], voxel);
            const long long cy = voxel_coord((double)xyz[3 * i + 1], voxel);
            const long long cz = voxel_coord((double)xyz[3 * i + 2], voxel);
            const uint64_t h = (uint64_t)HX * (uint64_t)cx + (uint64_t)HY * (uint64_t)cy + (uint64_t)HZ * (uint64_t)cz;
            const uint64_t hb = h + (1ull << (GS_COMPACT_BITS - 1));
            if (hb >> GS_COMPACT_BITS) *overflow = stamp;
            const uint64_t k40 = hb & ((1ull << GS_COMPACT_BITS) - 1ull);
            keys[i] = (k40 << GS_IDX_BITS) | (uint64_t)i;
            bin = (uint32_t)(k40 >> (GS_COMPACT_BITS - GS_BIN_BITS));
        }
        // consecutive points of a scan often share a voxel: one atomic per bin and warp
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        if (valid && lane == __ffs(peers) - 1) atomicAdd(&bins[bin], (uint32_t)__popc(peers));
        const uint32_t lo_inv = __reduce_max_sync(0xffffffffu, valid ? (uint32_t)(GS_BINS - 1) - bin : 0u);
        const uint32_t hi = __reduce_max_sync(0xffffffffu, valid ? bin : 0u);
        if (lane == 0) {
            atomicMax(&s_lo_inv, lo_inv);
            atomicMax(&s_hi, hi);
        }
    }
    __syncthreads();
    if (tid == 0) {
        atomicMax(&words[GSW_LO_INV], s_lo_inv);
        atomicMax(&words[GSW_HI], s_hi);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(&words[GSW_TICKET], 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const uint32_t lo = (uint32_t)(GS_BINS - 1) - __ldcg(&words[GSW_LO_INV]), hi = __ldcg(&words[GSW_HI]);
    // tiles of GS_SCAN_ITEMS bins per thread, loaded together: one L2 round trip per tile, not one per bin
    uint32_t carry = 0;
    for (uint32_t t0 = lo; t0 <= hi; t0 += blockDim.x * GS_SCAN_ITEMS) {
        const uint32_t b0 = t0 + tid * GS_SCAN_ITEMS;
        uint32_t c[GS_SCAN_ITEMS], sum = 0;
#pragma unroll
        for (int j = 0; j < GS_SCAN_ITEMS; ++j) {
            c[j] = b0 + j <= hi ? __ldcg(&bins[b0 + j]) : 0u;
            sum += c[j];
        }
        uint32_t total;
        uint32_t p = carry + gs_block_scan(sum, s_warp, total);
        carry += total;
#pragma unroll
        for (int j = 0; j < GS_SCAN_ITEMS; ++j) {
            if (b0 + j > hi) break;
            bins[b0 + j] = p;
            // bucket k starts at the first bin offset >= k * target: the buckets whose k * target lies in (p, p + c]
            for (uint32_t k = p / GS_BUCKET_TARGET + 1; k * GS_BUCKET_TARGET <= p + c[j] && k < (uint32_t)num_buckets; ++k)
                bucket_start[k] = p + c[j];
            p += c[j];
        }
    }
    if (tid == 0) {
        bucket_start[0] = 0u;
        bucket_start[num_buckets] = (uint32_t)n;
        words[GSW_TICKET] = 0u;
        words[GSW_LO_INV] = 0u;
        words[GSW_HI] = 0u;
        words[GSW_RANGE_LO] = lo;
        words[GSW_RANGE_HI] = hi;
        words[GSW_BUCKET_TICKET] = 0u;
    }
}

// K2: every composite key to its bin's cursor.  The bins are contiguous key ranges in key order, so every bucket ends
// up in its own slice of `sorted`; the order inside a bin does not matter.
__global__ void __launch_bounds__(256)
gs_bucket_scatter_kernel(const uint64_t* __restrict__ keys, int64_t n, uint32_t* bins, uint64_t* __restrict__ sorted) {
    pls_grid_dependency_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
        const int64_t i = base + lane;
        const bool valid = i < n;
        const uint64_t k = valid ? keys[i] : 0ull;
        const uint32_t bin = valid ? (uint32_t)(k >> (GS_IDX_BITS + GS_COMPACT_BITS - GS_BIN_BITS)) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        const int leader = __ffs(peers) - 1;
        uint32_t pos = 0;
        if (valid && lane == leader) pos = atomicAdd(&bins[bin], (uint32_t)__popc(peers));
        pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(peers & ((1u << lane) - 1u));
        if (valid) sorted[pos] = k;
    }
}

// The output offset of bucket b (run by one warp): decoupled look-back over the buckets before it, 32 per round trip.
__device__ uint32_t gs_bucket_prefix(uint32_t* status, uint32_t b, uint32_t agg) {
    const int lane = threadIdx.x & 31;
    if (b == 0) {
        if (lane == 0) gs_st_volatile(status, GS_FLAG_PREFIX | agg);
        return 0u;
    }
    if (lane == 0) gs_st_volatile(status + b, GS_FLAG_AGG | agg);
    uint32_t excl = 0;
    for (int64_t t = (int64_t)b - 1;; t -= 32) {
        const int64_t j = t - lane;
        uint32_t v = j >= 0 ? gs_ld_volatile(status + j) : GS_FLAG_PREFIX;  // before bucket 0: a prefix of 0
        while (__any_sync(0xffffffffu, (v >> 30) == 0u))
            if ((v >> 30) == 0u) v = gs_ld_volatile(status + j);
        const int first = __ffs(__ballot_sync(0xffffffffu, (v & GS_FLAG_PREFIX) != 0u)) - 1;
        excl += __reduce_add_sync(0xffffffffu, (first < 0 || lane <= first) ? (v & GS_VALUE_MASK) : 0u);
        if (first >= 0) break;
    }
    if (lane == 0) gs_st_volatile(status + b, GS_FLAG_PREFIX | (excl + agg));
    return excl;
}

template <typename T>
__device__ __forceinline__ void gs_emit(const T* __restrict__ xyz, T* __restrict__ out_xyz, long long* __restrict__ out_idx,
                                        uint64_t key, uint32_t dst) {
    const uint32_t src = (uint32_t)(key & GS_IDX_MASK);
    const T x = xyz[3 * (size_t)src], y = xyz[3 * (size_t)src + 1], z = xyz[3 * (size_t)src + 2];
    if (out_idx) out_idx[dst] = (long long)src;
    out_xyz[3 * (size_t)dst] = x;
    out_xyz[3 * (size_t)dst + 1] = y;
    out_xyz[3 * (size_t)dst + 2] = z;
}

__device__ __forceinline__ bool gs_is_head(const uint64_t* k, uint32_t i) {
    // buckets hold whole bins, so the first key of a bucket always starts a run
    return i == 0 || (k[i] >> GS_IDX_BITS) != (k[i - 1] >> GS_IDX_BITS);
}

// K3: one block per bucket (in ticket order, for the look-back): sort the bucket by composite key, keep the run heads,
// write them at the bucket's output offset.  The last bucket writes the sample count.  The block also clears the bins
// the scatter used, for the next call.
template <typename T>
__global__ void __launch_bounds__(GS_SELECT_THREADS)
gs_bucket_select_kernel(uint64_t* sorted, uint64_t* scratch, const uint32_t* __restrict__ bucket_start, uint32_t* status,
                        uint32_t* words, uint32_t* bins, int num_buckets, const T* __restrict__ xyz, T* __restrict__ out_xyz,
                        long long* __restrict__ out_idx, uint32_t* __restrict__ count_out) {
    __shared__ uint64_t s_keys[GS_BUCKET_CAP];
    __shared__ uint32_t s_warp[GS_SELECT_THREADS / 32];
    __shared__ uint32_t s_bucket, s_excl;
    const int tid = threadIdx.x;
    pls_grid_dependency_wait();
    if (tid == 0) s_bucket = atomicAdd(&words[GSW_BUCKET_TICKET], 1u);
    {
        const uint32_t lo = words[GSW_RANGE_LO], hi = words[GSW_RANGE_HI];
        for (uint32_t b = lo + blockIdx.x * blockDim.x + tid; b <= hi; b += gridDim.x * blockDim.x) bins[b] = 0u;
    }
    __syncthreads();
    const uint32_t b = s_bucket;
    const uint32_t s = bucket_start[b], m = bucket_start[b + 1] - s;
    uint32_t total;
    if (m <= GS_BUCKET_CAP) {
        // bitonic sort in shared memory, padded to a power of two with keys above every composite key
        uint32_t P = 1;
        while (P < m) P <<= 1;
        for (uint32_t i = tid; i < P; i += blockDim.x) s_keys[i] = i < m ? sorted[s + i] : ~0ull;
        __syncthreads();
        for (uint32_t k = 2; k <= P; k <<= 1)
            for (uint32_t j = k >> 1; j > 0; j >>= 1) {
                for (uint32_t i = tid; i < P / 2; i += blockDim.x) {
                    const uint32_t lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo | j;
                    const uint64_t a = s_keys[lo], c = s_keys[hi];
                    if ((a > c) == ((lo & k) == 0)) {
                        s_keys[lo] = c;
                        s_keys[hi] = a;
                    }
                }
                __syncthreads();
            }
        // contiguous items per thread: heads, their block offsets, the bucket's offset, the samples
        const uint32_t per = (m + blockDim.x - 1) / blockDim.x;
        const uint32_t i0 = min(tid * per, m), i1 = min(i0 + per, m);
        uint32_t heads = 0;
        for (uint32_t i = i0; i < i1; ++i) heads += gs_is_head(s_keys, i);
        uint32_t dst = gs_block_scan(heads, s_warp, total);
        if (tid < 32) {
            const uint32_t e = gs_bucket_prefix(status, b, total);
            if (tid == 0) s_excl = e;
        }
        __syncthreads();
        dst += s_excl;
        for (uint32_t i = i0; i < i1; ++i)
            if (gs_is_head(s_keys, i)) gs_emit(xyz, out_xyz, out_idx, s_keys[i], dst++);
    } else {
        // A bucket beyond shared memory (more than GS_BUCKET_CAP - GS_BUCKET_TARGET points in one bin, e.g. many points
        // in one voxel): a stable LSD radix sort through global memory by this block alone, on the bits in which the
        // bucket's keys differ, one chunk of blockDim.x keys after the other.
        uint64_t* a = sorted + s;
        uint64_t* alt = scratch + s;
        uint32_t* hist = reinterpret_cast<uint32_t*>(s_keys);  // [256] digit offsets
        uint32_t* warp_cnt = hist + 256;                       // [warps][256] digit counts of a chunk
        uint64_t kmin = ~0ull, kmax = 0ull;
        for (uint32_t i = tid; i < m; i += blockDim.x) {
            const uint64_t k = a[i];
            kmin = min(kmin, k);
            kmax = max(kmax, k);
        }
        __shared__ unsigned long long s_min, s_max;
        if (tid == 0) {
            s_min = ~0ull;
            s_max = 0ull;
        }
        __syncthreads();
        atomicMin(&s_min, (unsigned long long)kmin);
        atomicMax(&s_max, (unsigned long long)kmax);
        __syncthreads();
        kmin = s_min;
        const int bits = 64 - __clzll((long long)(s_max - kmin));
        const int lane = tid & 31, warp = tid >> 5, warps = blockDim.x >> 5;
        for (int shift = 0; shift < bits; shift += 8) {
            for (int d = tid; d < 256; d += blockDim.x) hist[d] = 0u;
            __syncthreads();
            for (uint32_t i = tid; i < m; i += blockDim.x) atomicAdd(&hist[(uint32_t)((a[i] - kmin) >> shift) & 255u], 1u);
            __syncthreads();
            {
                const uint32_t c = tid < 256 ? hist[tid] : 0u;
                const uint32_t e = gs_block_scan(c, s_warp, total);
                if (tid < 256) hist[tid] = e;
                __syncthreads();
            }
            for (uint32_t c0 = 0; c0 < m; c0 += blockDim.x) {
                for (int w = tid; w < warps * 256; w += blockDim.x) warp_cnt[w] = 0u;
                __syncthreads();
                const uint32_t i = c0 + tid;
                const bool valid = i < m;
                const uint64_t k = valid ? a[i] : 0ull;
                const uint32_t d = valid ? ((uint32_t)((k - kmin) >> shift) & 255u) : 256u;
                const uint32_t peers = __match_any_sync(0xffffffffu, d);
                const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
                if (valid && lane == __ffs(peers) - 1) warp_cnt[warp * 256 + d] = __popc(peers);
                __syncthreads();
                if (tid < 256) {
                    uint32_t run = hist[tid];
                    for (int w = 0; w < warps; ++w) {
                        const uint32_t c = warp_cnt[w * 256 + tid];
                        warp_cnt[w * 256 + tid] = run;
                        run += c;
                    }
                    hist[tid] = run;
                }
                __syncthreads();
                if (valid) alt[warp_cnt[warp * 256 + d] + rank] = k;
                __syncthreads();
            }
            uint64_t* t = a;
            a = alt;
            alt = t;
        }
        uint32_t heads = 0;
        for (uint32_t i = tid; i < m; i += blockDim.x) heads += gs_is_head(a, i);
        gs_block_scan(heads, s_warp, total);
        if (tid < 32) {
            const uint32_t e = gs_bucket_prefix(status, b, total);
            if (tid == 0) s_excl = e;
        }
        __syncthreads();
        uint32_t carry = s_excl;
        for (uint32_t c0 = 0; c0 < m; c0 += blockDim.x) {
            const uint32_t i = c0 + tid;
            const bool head = i < m && gs_is_head(a, i);
            uint32_t chunk;
            const uint32_t dst = carry + gs_block_scan(head ? 1u : 0u, s_warp, chunk);
            if (head) gs_emit(xyz, out_xyz, out_idx, a[i], dst);
            carry += chunk;
        }
        total = carry - s_excl;
    }
    if (b == (uint32_t)num_buckets - 1 && tid == 0) *count_out = s_excl + total;
}

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

// The three launches of the bucket path; the count lands in SC_GS_COUNT, an overflow stamp in SC_GS_OVERFLOW.
template <typename T>
void grid_sample_buckets(pls_context* ctx, const T* xyz_dev, int64_t n, double voxel, T* out_xyz_dev, long long* out_idx_dev) {
    cudaStream_t st = ctx->stream;
    const int num_buckets = (int)((n + GS_BUCKET_TARGET - 1) / GS_BUCKET_TARGET);
    if (!ctx->gs_bins.p) {  // the bins and control words start at zero; every call leaves them so
        ctx->gs_bins.reserve_exact((GS_BINS + GSW_WORDS) * sizeof(uint32_t), st);
        PLS_CUDA(cudaMemsetAsync(ctx->gs_bins.p, 0, (GS_BINS + GSW_WORDS) * sizeof(uint32_t), st));
    }
    ctx->gs_buckets.reserve(2 * ((size_t)num_buckets + 1) * sizeof(uint32_t), st);
    ctx->sort.keys_alt.reserve((size_t)n * sizeof(uint64_t), st);
    uint32_t* bins = ctx->gs_bins.as<uint32_t>();
    uint32_t* words = bins + GS_BINS;
    uint32_t* bucket_start = ctx->gs_buckets.as<uint32_t>();
    uint32_t* status = bucket_start + num_buckets + 1;
    uint64_t* keys = ctx->gs_keys.as<uint64_t>();
    uint64_t* sorted = ctx->sort.keys_alt.as<uint64_t>();
    gs_hash_bins_kernel<T><<<grid_for(n), 256, 0, st>>>(xyz_dev, n, voxel, keys, bins, words, bucket_start, status,
                                                        num_buckets, scalar_u32(ctx, SC_GS_OVERFLOW), ctx->gs_seq);
    PLS_CHECK_LAUNCH();
    launch_dependent(gs_bucket_scatter_kernel, grid_for(n), 256, st, (const uint64_t*)keys, n, bins, sorted);
    launch_dependent(gs_bucket_select_kernel<T>, num_buckets, GS_SELECT_THREADS, st, sorted, keys,
                     (const uint32_t*)bucket_start, status, words, bins, num_buckets, xyz_dev, out_xyz_dev, out_idx_dev,
                     scalar_u32(ctx, SC_GS_COUNT));
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
    if (compact && n <= SEL_MAX_N) {
        grid_sample_buckets(ctx, xyz_dev, n, voxel, out_xyz_dev, out_idx_dev);
        copy_to_host();
        return;
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
