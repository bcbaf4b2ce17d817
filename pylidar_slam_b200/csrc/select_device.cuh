// Single-pass stream selection with up to TWO outputs (decoupled look-back over tiles).
//
// Several steps of the path are "keep the elements that satisfy a predicate, in their original order": the run heads
// of the sorted voxel hashes (np.unique's first occurrence, pointcloud.py:177), the NaN-free rows of a cloud
// (utils.py:169-184), the z-buffer winners that become the ICP queries (icp_odometry.py:301-308).  Round 1 ran each as
// flags kernel -> scan kernel -> gather kernel plus a memset; here ONE kernel evaluates the predicate(s), scans and
// writes, and two selections over the same elements (valid rows AND z-buffer winners of a frame's samples) share it.
//
//   Op::State                                  per-element scratch carried from flags() to emit()
//   uint32_t Op::flags(int64_t i, State&)      bit 0 / bit 1: element i goes to output 0 / 1
//   void     Op::emit(int64_t i, int which, uint32_t pos, const State&)
//
// Tiles are the blocks in launch order; a tile publishes (aggregate, then inclusive prefix) in one 64-bit status word
// tagged with the launch's epoch, so the status array is never cleared (words of other epochs read as "not
// published").  The callers keep the grid within one resident wave (n <= SEL_MAX_N), so a tile waiting for its
// predecessors can never keep them from running.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "internal.cuh"

namespace pls {

constexpr int SEL_THREADS = 256;
constexpr int SEL_ITEMS = 8;
constexpr int SEL_TILE = SEL_THREADS * SEL_ITEMS;
constexpr int64_t SEL_MAX_N = (int64_t)SEL_TILE * 4 * kNumSMs;  // <= 4 tiles per SM: every tile of a launch is resident
constexpr unsigned long long SEL_AGG = 1ull << 62, SEL_PREFIX = 2ull << 62;
constexpr int SEL_EPOCH_BITS = 10, SEL_COUNT_BITS = 26;
constexpr unsigned long long SEL_COUNT_MASK = (1ull << SEL_COUNT_BITS) - 1ull;

__device__ __forceinline__ unsigned long long sel_pack(unsigned long long flag, uint32_t epoch, uint32_t c0, uint32_t c1) {
    return flag | ((unsigned long long)epoch << (2 * SEL_COUNT_BITS)) | ((unsigned long long)c1 << SEL_COUNT_BITS) | c0;
}

// totals[0], totals[1] receive the sizes of the two outputs (n_dev, if given, overrides n with a device-side count).
template <typename Op>
__global__ void __launch_bounds__(SEL_THREADS, 4)   // four tiles per SM resident: what SEL_MAX_N counts on
select_kernel(Op op, int64_t n, const uint32_t* __restrict__ n_dev, unsigned long long* status, uint32_t epoch,
              uint32_t* __restrict__ total0, uint32_t* __restrict__ total1) {
    __shared__ uint32_t warp_sums[2][SEL_THREADS / 32];
    __shared__ uint32_t s_excl[2];
    pls_grid_dependency_wait();
    if (n_dev) n = min(n, (int64_t)*n_dev);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t tile = blockIdx.x;
    const int64_t base = (int64_t)tile * SEL_TILE + (int64_t)tid * SEL_ITEMS;
    typename Op::State st[SEL_ITEMS];
    uint32_t f[SEL_ITEMS];
    uint32_t local0 = 0, local1 = 0;
#pragma unroll
    for (int i = 0; i < SEL_ITEMS; ++i) {
        const int64_t idx = base + i;
        f[i] = idx < n ? op.flags(idx, st[i]) : 0u;
        local0 += f[i] & 1u;
        local1 += (f[i] >> 1) & 1u;
    }
    // block-wide exclusive scan of the two per-thread counts, packed in one word (a tile holds 2048 elements: 12 bits each)
    uint32_t inc = local0 | (local1 << 16);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) {
        warp_sums[0][warp] = inc & 0xffffu;
        warp_sums[1][warp] = inc >> 16;
    }
    __syncthreads();
    if (warp == 0) {
        const uint32_t w0 = lane < SEL_THREADS / 32 ? warp_sums[0][lane] : 0u;
        const uint32_t w1 = lane < SEL_THREADS / 32 ? warp_sums[1][lane] : 0u;
        uint32_t i0 = w0, i1 = w1;
#pragma unroll
        for (int o = 1; o < SEL_THREADS / 32; o <<= 1) {
            const uint32_t v0 = __shfl_up_sync(0xffffffffu, i0, o), v1 = __shfl_up_sync(0xffffffffu, i1, o);
            if (lane >= o) { i0 += v0; i1 += v1; }
        }
        if (lane < SEL_THREADS / 32) {
            warp_sums[0][lane] = i0 - w0;
            warp_sums[1][lane] = i1 - w1;
        }
        const uint32_t t0 = __shfl_sync(0xffffffffu, i0, SEL_THREADS / 32 - 1);
        const uint32_t t1 = __shfl_sync(0xffffffffu, i1, SEL_THREADS / 32 - 1);
        if (lane == 0) {
            uint32_t e0 = 0, e1 = 0;
            volatile unsigned long long* vs = status;
            if (tile == 0) {
                vs[0] = sel_pack(SEL_PREFIX, epoch, t0, t1);
            } else {
                vs[tile] = sel_pack(SEL_AGG, epoch, t0, t1);
                int64_t t = (int64_t)tile - 1;
                while (true) {
                    const unsigned long long w = vs[t];
                    const bool mine = ((w >> (2 * SEL_COUNT_BITS)) & ((1u << SEL_EPOCH_BITS) - 1u)) == epoch && (w >> 62) != 0ull;
                    if (!mine) continue;  // not published yet (or a word of another launch): poll again
                    e0 += (uint32_t)(w & SEL_COUNT_MASK);
                    e1 += (uint32_t)((w >> SEL_COUNT_BITS) & SEL_COUNT_MASK);
                    if ((w >> 62) == 2ull) break;
                    --t;
                }
                vs[tile] = sel_pack(SEL_PREFIX, epoch, e0 + t0, e1 + t1);
            }
            s_excl[0] = e0;
            s_excl[1] = e1;
            if ((int64_t)(tile + 1) * SEL_TILE >= n || tile + 1 == gridDim.x) {
                if (total0) *total0 = e0 + t0;
                if (total1) *total1 = e1 + t1;
            }
        }
    }
    __syncthreads();
    uint32_t run0 = s_excl[0] + warp_sums[0][warp] + ((inc & 0xffffu) - local0);
    uint32_t run1 = s_excl[1] + warp_sums[1][warp] + ((inc >> 16) - local1);
#pragma unroll
    for (int i = 0; i < SEL_ITEMS; ++i) {
        const int64_t idx = base + i;
        if (f[i] & 1u) op.emit(idx, 0, run0, st[i]);
        if (f[i] & 2u) op.emit(idx, 1, run1, st[i]);
        run0 += f[i] & 1u;
        run1 += (f[i] >> 1) & 1u;
    }
}

// Host side: one launch, no memset (the status words are epoch-tagged; the buffer is cleared when it is (re)allocated
// and when the 10-bit epoch wraps).
template <typename Op>
void select_launch(pls_context* ctx, const Op& op, int64_t n, const uint32_t* n_dev, uint32_t* total0, uint32_t* total1) {
    PLS_REQUIRE(n > 0 && n <= SEL_MAX_N, "select_launch: size outside the single-wave range");
    cudaStream_t st = ctx->stream;
    SelectScratch& s = ctx->sel[ctx->stream == ctx->stream_map ? 1 : 0];
    const int64_t tiles = (n + SEL_TILE - 1) / SEL_TILE;
    const size_t need = (size_t)(SEL_MAX_N / SEL_TILE) * sizeof(unsigned long long);
    if (s.status.cap < need) {
        s.status.reserve_exact(need, st);
        PLS_CUDA(cudaMemsetAsync(s.status.p, 0, need, st));
        s.epoch = 0;
    }
    if (++s.epoch >= (1u << SEL_EPOCH_BITS)) {
        PLS_CUDA(cudaMemsetAsync(s.status.p, 0, need, st));
        s.epoch = 1;
    }
    launch_dependent(select_kernel<Op>, (unsigned)tiles, SEL_THREADS, st, op, n, n_dev, s.status.as<unsigned long long>(), s.epoch,
                     total0, total1);
}

}  // namespace pls
