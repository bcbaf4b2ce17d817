// Device-wide primitives used by the hot path: a stable LSD radix sort of (u64,u32) pairs
// (one kernel per 8-bit digit, chained-scan decoupled look-back across tiles, histograms of
// all digits taken in one upfront pass) and a single-pass exclusive scan of 0/1 flags.
//
// They replace np.unique's stable sort (slam/common/pointcloud.py:177,193) and feed the
// cell-pyramid index build that stands in for the per-frame KD-tree build (local_map.py:365-369).
#include "internal.cuh"

namespace pls {

namespace {

constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_ITEMS = 8;
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;
constexpr int LOOKBACK = 8;
constexpr int RADIX = 256;
constexpr uint32_t FLAG_AGG = 1u << 30;
constexpr uint32_t FLAG_PREFIX = 2u << 30;
constexpr uint32_t VALUE_MASK = (1u << 30) - 1u;

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Digit histograms of all passes in one read of the keys; the block that finishes last turns them into
// exclusive bin offsets (one launch instead of histogram + scan).  Also clears the look-back words and tile counters
// of the passes that follow (status_words of them).  n_dev (nullable): the key count on the device, n a bound of it.
__global__ void __launch_bounds__(256) sort_hist_kernel(const uint64_t* __restrict__ keys, int64_t n,
                                                        int num_passes, uint32_t* __restrict__ hist,
                                                        uint32_t* __restrict__ done_counter, uint32_t* __restrict__ status,
                                                        int64_t status_words, const uint32_t* __restrict__ n_dev) {
    __shared__ uint32_t sh[8 * RADIX];
    __shared__ int s_last;
    pls_grid_dependency_wait();
    if (n_dev) n = *n_dev;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < status_words; i += (int64_t)gridDim.x * blockDim.x)
        status[i] = 0u;
    for (int i = threadIdx.x; i < num_passes * RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t k = keys[i];
        for (int p = 0; p < num_passes; ++p) atomicAdd(&sh[p * RADIX + (int)((k >> (8 * p)) & 255u)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < num_passes * RADIX; i += blockDim.x)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(done_counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // in-place exclusive scan of every pass's 256 bins (blockDim.x == RADIX)
    const int t = threadIdx.x;
    for (int p = 0; p < num_passes; ++p) {
        uint32_t* h = hist + p * RADIX;
        const uint32_t v = __ldcg(h + t);
        __syncthreads();
        sh[t] = v;
        __syncthreads();
        for (int o = 1; o < RADIX; o <<= 1) {
            const uint32_t a = (t >= o) ? sh[t - o] : 0u;
            __syncthreads();
            sh[t] += a;
            __syncthreads();
        }
        h[t] = sh[t] - v;
    }
}

// n_dev (nullable): the key count on the device, n a bound of it (the grid is sized for n).  Tiles are cut from 0 as
// for a host count; a tile past the count exits before it publishes a look-back word, and since tiles take their
// numbers in launch order, no tile within the count ever waits for one past it.
__global__ void __launch_bounds__(SORT_THREADS)
sort_pass_kernel(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin, uint64_t* __restrict__ kout,
                 uint32_t* __restrict__ vout, int64_t n, int shift, const uint32_t* __restrict__ base,
                 uint32_t* status, uint32_t* tile_counter, const uint32_t* __restrict__ n_dev) {
    __shared__ uint32_t warp_hist[SORT_WARPS][RADIX];
    __shared__ uint32_t tile_offset[RADIX];
    __shared__ uint32_t s_tile;
    __shared__ uint32_t tile_start[RADIX];     // first slot of digit d in the tile's digit-sorted staging order
    __shared__ uint32_t scan_warp[SORT_WARPS];
    __shared__ uint64_t s_keys[SORT_TILE];
    __shared__ uint32_t s_vals[SORT_TILE];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pls_grid_dependency_wait();
    if (tid == 0) s_tile = atomicAdd(tile_counter, 1u);
    for (int i = tid; i < SORT_WARPS * RADIX; i += SORT_THREADS) (&warp_hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    if (n_dev) {
        n = *n_dev;
        if ((int64_t)tile * SORT_TILE >= n) return;  // block-uniform
    }
    const int64_t seg = (int64_t)tile * SORT_TILE + (int64_t)warp * (32 * SORT_ITEMS);
    const uint32_t lt_mask = (1u << lane) - 1u;

    uint64_t key[SORT_ITEMS];
    uint32_t val[SORT_ITEMS];
    uint32_t rank[SORT_ITEMS];
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        int64_t idx = seg + i * 32 + lane;
        bool valid = idx < n;
        key[i] = valid ? kin[idx] : 0ull;
        val[i] = valid ? vin[idx] : 0u;
    }
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        int64_t idx = seg + i * 32 + lane;
        bool valid = idx < n;
        uint32_t d = valid ? (uint32_t)((key[i] >> shift) & 255u) : 0xffffu;
        uint32_t peers = __match_any_sync(0xffffffffu, d);
        uint32_t pre = valid ? warp_hist[warp][d] : 0u;
        __syncwarp();
        if (valid && lane == (__ffs(peers) - 1)) warp_hist[warp][d] = pre + __popc(peers);
        __syncwarp();
        rank[i] = pre + __popc(peers & lt_mask);
    }
    __syncthreads();
    {
        // thread d: exclusive prefix over the warps of this tile, then decoupled look-back
        const int d = tid;
        uint32_t sum = 0;
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) {
            uint32_t c = warp_hist[w][d];
            warp_hist[w][d] = sum;
            sum += c;
        }
        uint32_t excl = 0;
        uint32_t* st = status + (size_t)tile * RADIX + d;
        if (tile == 0) {
            st_volatile_u32(st, FLAG_PREFIX | sum);
        } else {
            st_volatile_u32(st, FLAG_AGG | sum);
            // windowed look-back: LOOKBACK predecessors are read per round trip (independent loads) and
            // consumed in order up to the first unpublished one.  With one predecessor per round trip the
            // inclusive prefix ripples through the tiles at one L2 latency per tile.
            int64_t t = (int64_t)tile - 1;
            bool done = false;
            while (!done) {
                uint32_t s[LOOKBACK];
#pragma unroll
                for (int k = 0; k < LOOKBACK; ++k)
                    s[k] = (t - k >= 0) ? ld_volatile_u32(status + (size_t)(t - k) * RADIX + d) : FLAG_PREFIX;
#pragma unroll
                for (int k = 0; k < LOOKBACK; ++k) {
                    if (done || (s[k] >> 30) == 0u) break;  // stop at the first unpublished predecessor
                    excl += s[k] & VALUE_MASK;
                    --t;
                    if (s[k] & FLAG_PREFIX) done = true;
                }
            }
            st_volatile_u32(st, FLAG_PREFIX | (excl + sum));
        }
        tile_offset[d] = base[d] + excl;
        // exclusive scan of the tile's digit counts over the 256 digits (thread d holds `sum`)
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) scan_warp[warp] = inc;
        __syncthreads();
        uint32_t before = 0;
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) before += (w < warp) ? scan_warp[w] : 0u;
        tile_start[d] = before + inc - sum;
    }
    __syncthreads();
    // stage the tile in shared memory in digit order (stable: warp, then item, then lane), then write it out
    // with consecutive threads on consecutive slots: elements of one digit land on consecutive global
    // addresses, so the low-digit passes no longer scatter one 8-byte key per 32-byte sector
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        int64_t idx = seg + i * 32 + lane;
        if (idx < n) {
            uint32_t d = (uint32_t)((key[i] >> shift) & 255u);
            uint32_t slot = tile_start[d] + warp_hist[warp][d] + rank[i];
            s_keys[slot] = key[i];
            s_vals[slot] = val[i];
        }
    }
    __syncthreads();
    const int64_t tile_base = (int64_t)tile * SORT_TILE;
    const int tile_n = (int)((n - tile_base) < (int64_t)SORT_TILE ? (n - tile_base) : (int64_t)SORT_TILE);
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; ++i) {
        const int j = i * SORT_THREADS + tid;
        if (j < tile_n) {
            const uint64_t k = s_keys[j];
            const uint32_t d = (uint32_t)((k >> shift) & 255u);
            const uint32_t pos = tile_offset[d] + ((uint32_t)j - tile_start[d]);
            kout[pos] = k;
            vout[pos] = s_vals[j];
        }
    }
}

// ---- single-pass exclusive scan of byte flags -------------------------------------------------
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__global__ void __launch_bounds__(SCAN_THREADS)
scan_flags_kernel(const uint8_t* __restrict__ flags, int64_t n, uint32_t* __restrict__ pos_out,
                  uint32_t* status, uint32_t* tile_counter, uint32_t* total_out) {
    __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint32_t s_tile, s_excl;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) s_tile = atomicAdd(tile_counter, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const int64_t base = (int64_t)tile * SCAN_TILE + (int64_t)tid * SCAN_ITEMS;
    uint32_t f[SCAN_ITEMS];
    uint32_t local = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        int64_t idx = base + i;
        f[i] = (idx < n && flags[idx]) ? 1u : 0u;
        local += f[i];
    }
    // block exclusive scan of `local`
    uint32_t inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = (lane < SCAN_THREADS / 32) ? warp_sums[lane] : 0u;
        uint32_t winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t v = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += v;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = winc - w;
        uint32_t tile_sum = __shfl_sync(0xffffffffu, winc, SCAN_THREADS / 32 - 1);
        if (lane == 0) {
            uint32_t excl = 0;
            if (tile == 0) {
                st_volatile_u32(status + tile, FLAG_PREFIX | tile_sum);
            } else {
                st_volatile_u32(status + tile, FLAG_AGG | tile_sum);
                int64_t t = (int64_t)tile - 1;
                bool done = false;
                while (!done) {
                    uint32_t s[LOOKBACK];
#pragma unroll
                    for (int k = 0; k < LOOKBACK; ++k) s[k] = (t - k >= 0) ? ld_volatile_u32(status + (t - k)) : FLAG_PREFIX;
#pragma unroll
                    for (int k = 0; k < LOOKBACK; ++k) {
                        if (done || (s[k] >> 30) == 0u) break;
                        excl += s[k] & VALUE_MASK;
                        --t;
                        if (s[k] & FLAG_PREFIX) done = true;
                    }
                }
                st_volatile_u32(status + tile, FLAG_PREFIX | (excl + tile_sum));
            }
            s_excl = excl;
            if ((int64_t)(tile + 1) * SCAN_TILE >= n) *total_out = excl + tile_sum;
        }
    }
    __syncthreads();
    uint32_t run = s_excl + warp_sums[warp] + (inc - local);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        int64_t idx = base + i;
        if (idx < n) pos_out[idx] = run;
        run += f[i];
    }
}

}  // namespace

void radix_sort_pairs(pls_context* ctx, uint64_t* keys, uint32_t* vals, int64_t n, int num_passes,
                      uint64_t** keys_out, uint32_t** vals_out, int64_t cap_n, const uint32_t* n_dev) {
    PLS_REQUIRE(num_passes >= 1 && num_passes <= 8, "radix_sort_pairs: 1..8 passes");
    PLS_REQUIRE(n < (1ll << 30), "radix_sort_pairs: n must be < 2^30");
    SortScratch& s = ctx->sort;
    cudaStream_t st = ctx->stream;
    if (n <= 0) {
        *keys_out = keys;
        *vals_out = vals;
        return;
    }
    const int64_t tiles = (n + SORT_TILE - 1) / SORT_TILE;
    if (cap_n < n) cap_n = n;
    const int64_t cap_tiles = (cap_n + SORT_TILE - 1) / SORT_TILE;
    s.keys_alt.reserve(cap_n * sizeof(uint64_t), st);
    s.vals_alt.reserve(cap_n * sizeof(uint32_t), st);
    const size_t hist_bytes = (8 * RADIX + 1) * sizeof(uint32_t);  // + the histogram kernel's last-block ticket
    const size_t status_words = (size_t)num_passes * tiles * RADIX + 8;
    s.hist.reserve(hist_bytes, st);
    s.status.reserve(((size_t)num_passes * cap_tiles * RADIX + 8) * sizeof(uint32_t), st);
    PLS_CUDA(cudaMemsetAsync(s.hist.p, 0, hist_bytes, st));
    // one block per SM at most: every block ends with num_passes * 256 global atomics
    int hist_blocks = (int)((n + 256 * 4 - 1) / (256 * 4));
    if (hist_blocks > kNumSMs) hist_blocks = kNumSMs;
    launch_dependent(sort_hist_kernel, hist_blocks, 256, st, keys, n, num_passes, s.hist.as<uint32_t>(),
                     s.hist.as<uint32_t>() + 8 * RADIX, s.status.as<uint32_t>(), (int64_t)status_words, n_dev);
    uint64_t* kin = keys;
    uint32_t* vin = vals;
    uint64_t* kout = s.keys_alt.as<uint64_t>();
    uint32_t* vout = s.vals_alt.as<uint32_t>();
    uint32_t* counters = s.status.as<uint32_t>() + (size_t)num_passes * tiles * RADIX;
    for (int p = 0; p < num_passes; ++p) {
        launch_dependent(sort_pass_kernel, (unsigned)tiles, SORT_THREADS, st, kin, vin, kout, vout, n, 8 * p,
                         s.hist.as<uint32_t>() + p * RADIX, s.status.as<uint32_t>() + (size_t)p * tiles * RADIX, counters + p,
                         n_dev);
        uint64_t* tk = kin; kin = kout; kout = tk;
        uint32_t* tv = vin; vin = vout; vout = tv;
    }
    *keys_out = kin;
    *vals_out = vin;
}

void exclusive_scan_flags(pls_context* ctx, const uint8_t* flags, int64_t n, uint32_t* pos_out,
                          uint32_t* total_dev) {
    cudaStream_t st = ctx->stream;
    if (n <= 0) {
        PLS_CUDA(cudaMemsetAsync(total_dev, 0, sizeof(uint32_t), st));
        return;
    }
    PLS_REQUIRE(n < (1ll << 30), "exclusive_scan_flags: n must be < 2^30");
    const int64_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    ctx->scan.status.reserve((tiles + 4) * sizeof(uint32_t), st);
    PLS_CUDA(cudaMemsetAsync(ctx->scan.status.p, 0, (tiles + 4) * sizeof(uint32_t), st));
    uint32_t* status = ctx->scan.status.as<uint32_t>();
    scan_flags_kernel<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(flags, n, pos_out, status, status + tiles, total_dev);
    PLS_CHECK_LAUNCH();
}

}  // namespace pls
