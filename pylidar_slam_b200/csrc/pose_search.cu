// Correlative pose search on the kd map (no reference counterpart): pls_kdmap_pose_search.
//
//   ps_box_kernel    : the base cell of every (base, valid scan row), float64 with explicit roundings, reduced to the
//                      min / max cell with 64-bit atomicMin / atomicMax (order-independent).  The host reads the box.
//   ps_occupy_kernel : one pass over the map's points sets the bit of every map cell inside the box (atomicOr), in a
//                      bit grid with x fastest, each (y, z) row padded to whole 32-bit words.
//   ps_score_kernel  : a block owns one base and a tile of 32 i x 8 j shifts, warp w at j0 + w, lane l at i0 + l.  The
//                      base's cells stream through shared memory; a lane tests one bit per point -- a warp's 32 bits
//                      lie in one or two words of one row -- and counts in a register: no atomics, exact integers.
//   ps_peak_kernel   : flags the candidates (score > 0, key strictly better than each 3x3x3 neighbour's).
//   compaction       : exclusive_scan_flags per chunk of < 2^30 flags, keys (~score << 32 | L) sorted ascending by
//                      radix_sort_pairs -- score descending, then L ascending -- and the first K read back.
#include <algorithm>
#include <climits>
#include <cmath>

#include "internal.cuh"

namespace pls {

namespace {

constexpr int PS_THREADS = 256;
constexpr int PS_ROWS = PS_THREADS / 32;  // j shifts per block, one per warp
constexpr int PS_CHUNK = 1024;            // base cells staged in shared memory per pass
constexpr uint32_t PS_SKIP = 0xffffffffu; // a dropped (non-finite) row in the staged cells
constexpr long long PS_MAX_CELL = 1ll << 40;
constexpr int64_t PS_SCAN_CHUNK = 1ll << 29;  // exclusive_scan_flags takes fewer than 2^30 flags

inline int blocks_for(int64_t n, int threads, int cap) {
    const int64_t b = (n + threads - 1) / threads;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// cell_a(p) as the header defines it: q = ((R0 x + R1 y) + R2 z) + t, every operation separately rounded, then
// voxel_coord.  False for a row with a non-finite coordinate.
__device__ __forceinline__ long long base_axis(const double* __restrict__ R, double x, double y, double z, double c) {
    return voxel_coord(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[0], x), __dmul_rn(R[1], y)), __dmul_rn(R[2], z)), R[3]), c);
}
__device__ __forceinline__ bool base_cell(const double* __restrict__ T, float x, float y, float z, double c,
                                          long long& cx, long long& cy, long long& cz) {
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
    cx = base_axis(T, x, y, z, c);
    cy = base_axis(T + 4, x, y, z, c);
    cz = base_axis(T + 8, x, y, z, c);
    return true;
}

// box[0..2] = min cell, box[3..5] = max cell over every base and valid row (initialised to LLONG_MAX / LLONG_MIN)
__global__ void __launch_bounds__(PS_THREADS) ps_box_kernel(const float* __restrict__ scan, int64_t n,
                                                            const double* __restrict__ bases, int A, double c,
                                                            long long* __restrict__ box) {
    long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
    const int64_t total = n * (int64_t)A;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = k / n, p = k - a * n;
        long long cell[3];
        if (!base_cell(bases + 16 * a, scan[3 * p], scan[3 * p + 1], scan[3 * p + 2], c, cell[0], cell[1], cell[2]))
            continue;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            lo[r] = min(lo[r], cell[r]);
            hi[r] = max(hi[r], cell[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[r] = min(lo[r], __shfl_xor_sync(0xffffffffu, lo[r], o));
            hi[r] = max(hi[r], __shfl_xor_sync(0xffffffffu, hi[r], o));
        }
    }
    if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0]) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            atomicMin(box + r, lo[r]);
            atomicMax(box + 3 + r, hi[r]);
        }
    }
}

// The bit grid over the box: origin o (min cell - (half_x, half_y, 0)), extent e, wx words per (y, z) row.
struct PsGrid {
    long long o[3];
    long long e[3];
    uint32_t wx;
};

__global__ void ps_occupy_kernel(const float4* __restrict__ pts, int64_t m, double c, PsGrid g, uint32_t* __restrict__ bits) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
        const float4 p = pts[k];
        // unsigned differences: a cell below the origin wraps to a large value and fails the extent test
        const uint64_t X = (uint64_t)voxel_coord((double)p.x, c) - (uint64_t)g.o[0];
        const uint64_t Y = (uint64_t)voxel_coord((double)p.y, c) - (uint64_t)g.o[1];
        const uint64_t Z = (uint64_t)voxel_coord((double)p.z, c) - (uint64_t)g.o[2];
        if (X >= (uint64_t)g.e[0] || Y >= (uint64_t)g.e[1] || Z >= (uint64_t)g.e[2]) continue;
        atomicOr(bits + (Z * (uint64_t)g.e[1] + Y) * g.wx + (X >> 5), 1u << (X & 31));
    }
}

// Block b: base a, shift tile (it, jt); lane i0 + lane, warp j0 + warp.  scores[(a*Wy + jj)*Wx + ii].
__global__ void __launch_bounds__(PS_THREADS) ps_score_kernel(const float* __restrict__ scan, int64_t n,
                                                              const double* __restrict__ bases, double c, PsGrid g,
                                                              const uint32_t* __restrict__ bits, int Wx, int Wy,
                                                              int tiles_x, int tiles_y, int32_t* __restrict__ scores) {
    __shared__ uint2 cells[PS_CHUNK];  // (word offset of the cell's row at shift (0, -half_y), x - origin at shift -half_x)
    __shared__ double T[16];
    const int64_t b = blockIdx.x;
    const int it = (int)(b % tiles_x);
    const int jt = (int)((b / tiles_x) % tiles_y);
    const int64_t a = b / ((int64_t)tiles_x * tiles_y);
    if (threadIdx.x < 16) T[threadIdx.x] = bases[16 * a + threadIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ii = it * 32 + lane, jj = jt * PS_ROWS + warp;
    const bool active = ii < Wx && jj < Wy;
    // inactive lanes test an in-box bit of the last shift, so that every lane runs the same loop
    const uint32_t di = (uint32_t)min(ii, Wx - 1), dj_words = (uint32_t)min(jj, Wy - 1) * g.wx;
    int32_t count = 0;
    for (int64_t k0 = 0; k0 < n; k0 += PS_CHUNK) {
        const int len = (int)min((int64_t)PS_CHUNK, n - k0);
        __syncthreads();
        for (int k = threadIdx.x; k < len; k += PS_THREADS) {
            const int64_t p = k0 + k;
            long long cx, cy, cz;
            uint2 v = make_uint2(PS_SKIP, 0u);
            if (base_cell(T, scan[3 * p], scan[3 * p + 1], scan[3 * p + 2], c, cx, cy, cz)) {
                // relative to the box's min cell, i.e. at shift (-half_x, -half_y): each lane adds its di, dj
                const uint32_t X = (uint32_t)(cx - g.o[0]) - (uint32_t)(Wx - 1) / 2u;
                const uint32_t Y = (uint32_t)(cy - g.o[1]) - (uint32_t)(Wy - 1) / 2u;
                const uint32_t Z = (uint32_t)(cz - g.o[2]);
                v = make_uint2((Z * (uint32_t)g.e[1] + Y) * g.wx, X);
            }
            cells[k] = v;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < len; ++k) {
            const uint2 v = cells[k];
            if (v.x == PS_SKIP) continue;
            const uint32_t X = v.y + di;
            count += (int32_t)((__ldg(bits + v.x + dj_words + (X >> 5)) >> (X & 31)) & 1u);
        }
    }
    if (active) scores[(a * Wy + jj) * (int64_t)Wx + ii] = count;
}

// flags[L] = 1 for a candidate: score > 0 and (score, -L) strictly greater than every neighbour's in the 3x3x3 block
__global__ void ps_peak_kernel(const int32_t* __restrict__ s, int A, int Wy, int Wx, uint8_t* __restrict__ flags) {
    const int64_t V = (int64_t)A * Wy * Wx;
    for (int64_t L = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; L < V; L += (int64_t)gridDim.x * blockDim.x) {
        const int ii = (int)(L % Wx);
        const int64_t t = L / Wx;
        const int jj = (int)(t % Wy);
        const int a = (int)(t / Wy);
        const int32_t sc = s[L];
        bool peak = sc > 0;
        for (int da = -1; da <= 1 && peak; ++da) {
            if (a + da < 0 || a + da >= A) continue;
            for (int dj = -1; dj <= 1; ++dj) {
                if (jj + dj < 0 || jj + dj >= Wy) continue;
                for (int dx = -1; dx <= 1; ++dx) {
                    if (ii + dx < 0 || ii + dx >= Wx || (da == 0 && dj == 0 && dx == 0)) continue;
                    const int64_t Ln = L + ((int64_t)da * Wy + dj) * Wx + dx;
                    const int32_t sn = s[Ln];
                    if (sn > sc || (sn == sc && Ln < L)) peak = false;
                }
            }
        }
        flags[L] = peak ? 1 : 0;
    }
}

// keys[base + pos[L]] = (~score << 32) | L for every flagged L; base = the candidates of the earlier scan chunks
__global__ void ps_compact_kernel(const int32_t* __restrict__ s, const uint8_t* __restrict__ flags,
                                  const uint32_t* __restrict__ pos, const uint32_t* __restrict__ chunk_totals, int64_t V,
                                  uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    for (int64_t L = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; L < V; L += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[L]) continue;
        uint32_t at = pos[L];
        for (int64_t ch = 0; ch < L / PS_SCAN_CHUNK; ++ch) at += chunk_totals[ch];
        keys[at] = ((uint64_t)(~(uint32_t)s[L]) << 32) | (uint64_t)L;
        vals[at] = (uint32_t)L;
    }
}

}  // namespace

}  // namespace pls

using namespace pls;

extern "C" int pls_kdmap_pose_search(pls_context* ctx, const float* scan, int64_t n, const double* bases, int A,
                                     double cell, int half_x, int half_y, int K, int32_t* out_scores, double* out_T,
                                     int32_t* out_score, int64_t* out_index, int* out_num) {
    PLS_API_BEGIN(ctx)
    // every argument is checked before anything is enqueued: a refused call changes nothing
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, "pls_kdmap_pose_search: needs a kd-tree local map");
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    PLS_REQUIRE(scan && bases, "pls_kdmap_pose_search: scan and bases must not be NULL");
    PLS_REQUIRE(n > 0 && n <= INT32_MAX, "pls_kdmap_pose_search: scan must be [n,3] with 0 < n < 2^31");
    PLS_REQUIRE(A > 0, "pls_kdmap_pose_search: bases must be [A,16] with A > 0");
    PLS_REQUIRE(half_x >= 0 && half_y >= 0, "pls_kdmap_pose_search: half_x and half_y must be >= 0");
    PLS_REQUIRE(K >= 0 && K <= PLS_POSE_SEARCH_MAX_K, "pls_kdmap_pose_search: K must lie in [0, 1024]");
    PLS_REQUIRE(std::isfinite(cell) && cell > 0.0, "pls_kdmap_pose_search: cell must be finite and > 0");
    PLS_REQUIRE(out_num && (K == 0 || (out_T && out_score && out_index)),
                "pls_kdmap_pose_search: out_num, and for K > 0 out_T, out_score and out_index, must not be NULL");
    const int Wx = 2 * half_x + 1, Wy = 2 * half_y + 1;  // half <= INT_MAX / 2 follows from the volume check below
    PLS_REQUIRE(half_x < (1 << 30) && half_y < (1 << 30) && (double)A * Wx * Wy < 2147483648.0,
                "pls_kdmap_pose_search: A*(2*half_x+1)*(2*half_y+1) must be < 2^31");
    const int64_t V = (int64_t)A * Wx * Wy;
    std::vector<double> Tb((size_t)A * 16);
    if (is_device_ptr(bases)) PLS_CUDA(cudaMemcpy(Tb.data(), bases, Tb.size() * sizeof(double), cudaMemcpyDeviceToHost));
    else memcpy(Tb.data(), bases, Tb.size() * sizeof(double));
    for (double v : Tb) PLS_REQUIRE(std::isfinite(v), "pls_kdmap_pose_search: every base must be finite");

    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    // scratch of this stateless call: next_buf, never a buffer the map or an ICP keeps state in
    DBuf* nb = ctx->next_buf;
    const float* scan_dev = (const float*)to_device(ctx, scan, (size_t)n * 3 * sizeof(float), nb[0]);
    nb[1].reserve((size_t)A * 16 * sizeof(double) + 8 * sizeof(long long) + 8 * sizeof(uint32_t), st);
    double* bases_dev = nb[1].as<double>();
    long long* box_dev = reinterpret_cast<long long*>(bases_dev + (size_t)A * 16);
    uint32_t* totals_dev = reinterpret_cast<uint32_t*>(box_dev + 8);
    const long long box_init[6] = {LLONG_MAX, LLONG_MAX, LLONG_MAX, LLONG_MIN, LLONG_MIN, LLONG_MIN};
    PLS_CUDA(cudaMemcpyAsync(bases_dev, Tb.data(), Tb.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    PLS_CUDA(cudaMemcpyAsync(box_dev, box_init, sizeof(box_init), cudaMemcpyHostToDevice, st));
    ps_box_kernel<<<blocks_for(n * (int64_t)A, PS_THREADS, 8 * kNumSMs), PS_THREADS, 0, st>>>(scan_dev, n, bases_dev, A,
                                                                                              cell, box_dev);
    PLS_CHECK_LAUNCH();
    long long box[6];
    PLS_CUDA(cudaMemcpyAsync(box, box_dev, sizeof(box), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));

    auto put = [&](void* dst, const void* src, size_t bytes) {  // host or device outputs
        if (!dst || !bytes) return;
        if (is_device_ptr(dst)) PLS_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
        else memcpy(dst, src, bytes);
    };
    if (box[0] > box[3]) {  // no valid row: every score is 0, no candidate
        if (out_scores) {
            if (is_device_ptr(out_scores)) PLS_CUDA(cudaMemset(out_scores, 0, (size_t)V * sizeof(int32_t)));
            else memset(out_scores, 0, (size_t)V * sizeof(int32_t));
        }
        *out_num = 0;
        return PLS_OK;
    }
    for (int r = 0; r < 6; ++r)
        PLS_REQUIRE(box[r] > -PS_MAX_CELL && box[r] < PS_MAX_CELL,
                    "pls_kdmap_pose_search: a base cell lies beyond +-2^40 cells of the origin");
    PsGrid g;
    const long long half[3] = {half_x, half_y, 0};
    for (int r = 0; r < 3; ++r) {
        g.o[r] = box[r] - half[r];
        g.e[r] = box[3 + r] - box[r] + 1 + 2 * half[r];
    }
    // the grid's bits: x rows padded to whole words
    const double box_bits = 32.0 * (double)((g.e[0] + 31) / 32) * (double)g.e[1] * (double)g.e[2];
    if (box_bits > (double)PLS_POSE_SEARCH_MAX_BITS) {
        char msg[256];
        snprintf(msg, sizeof(msg),
                 "pls_kdmap_pose_search: the occupancy box of %lld x %lld x %lld cells (%.0f bits with word-padded x "
                 "rows) exceeds PLS_POSE_SEARCH_MAX_BITS (2^31); use a larger cell or a smaller window",
                 g.e[0], g.e[1], g.e[2], box_bits);
        throw pls::Error{PLS_E_INVALID, msg};
    }
    g.wx = (uint32_t)((g.e[0] + 31) / 32);
    const size_t words = (size_t)g.wx * (size_t)g.e[1] * (size_t)g.e[2];

    // occupancy of the map's cells inside the box
    nb[2].reserve(words * sizeof(uint32_t), st);
    uint32_t* bits = nb[2].as<uint32_t>();
    PLS_CUDA(cudaMemsetAsync(bits, 0, words * sizeof(uint32_t), st));
    const int64_t M = ctx->kd.count;
    if (M > 0) {
        ps_occupy_kernel<<<blocks_for(M, 256, 16 * kNumSMs), 256, 0, st>>>(ctx->kd.store[ctx->kd.cur].as<float4>(), M,
                                                                           cell, g, bits);
        PLS_CHECK_LAUNCH();
    }
    // scores
    nb[3].reserve((size_t)V * sizeof(int32_t), st);
    int32_t* scores = nb[3].as<int32_t>();
    const int tiles_x = (Wx + 31) / 32, tiles_y = (Wy + PS_ROWS - 1) / PS_ROWS;
    const int64_t score_blocks = (int64_t)A * tiles_x * tiles_y;
    ps_score_kernel<<<(unsigned)score_blocks, PS_THREADS, 0, st>>>(scan_dev, n, bases_dev, cell, g, bits, Wx, Wy, tiles_x,
                                                                    tiles_y, scores);
    PLS_CHECK_LAUNCH();

    // candidates and their order
    std::vector<uint64_t> top;
    if (K > 0) {
        nb[4].reserve((size_t)V, st);
        nb[5].reserve((size_t)V * sizeof(uint32_t), st);
        uint8_t* flags = nb[4].as<uint8_t>();
        uint32_t* pos = nb[5].as<uint32_t>();
        ps_peak_kernel<<<blocks_for(V, 256, 16 * kNumSMs), 256, 0, st>>>(scores, A, Wy, Wx, flags);
        PLS_CHECK_LAUNCH();
        const int chunks = (int)((V + PS_SCAN_CHUNK - 1) / PS_SCAN_CHUNK);
        for (int ch = 0; ch < chunks; ++ch) {
            const int64_t off = (int64_t)ch * PS_SCAN_CHUNK;
            exclusive_scan_flags(ctx, flags + off, std::min(PS_SCAN_CHUNK, V - off), pos + off, totals_dev + ch);
        }
        uint32_t totals[8] = {};
        PLS_CUDA(cudaMemcpyAsync(totals, totals_dev, (size_t)chunks * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        int64_t num = 0;
        for (int ch = 0; ch < chunks; ++ch) num += totals[ch];
        if (num > 0) {
            nb[6].reserve((size_t)num * sizeof(uint64_t), st);
            nb[7].reserve((size_t)num * sizeof(uint32_t), st);
            ps_compact_kernel<<<blocks_for(V, 256, 16 * kNumSMs), 256, 0, st>>>(scores, flags, pos, totals_dev, V,
                                                                                nb[6].as<uint64_t>(), nb[7].as<uint32_t>());
            PLS_CHECK_LAUNCH();
            uint64_t* keys_out = nullptr;
            uint32_t* vals_out = nullptr;
            radix_sort_pairs(ctx, nb[6].as<uint64_t>(), nb[7].as<uint32_t>(), num, 8, &keys_out, &vals_out);
            top.resize((size_t)std::min<int64_t>(K, num));
            PLS_CUDA(cudaMemcpyAsync(top.data(), keys_out, top.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        }
    }
    if (out_scores)
        PLS_CUDA(cudaMemcpyAsync(out_scores, scores, (size_t)V * sizeof(int32_t), cudaMemcpyDefault, st));
    PLS_CUDA(cudaStreamSynchronize(st));

    const int k = (int)top.size();
    std::vector<double> T((size_t)k * 16);
    std::vector<int32_t> sc((size_t)k);
    std::vector<int64_t> idx((size_t)k);
    for (int c = 0; c < k; ++c) {
        const int64_t L = (int64_t)(top[(size_t)c] & 0xffffffffull);
        sc[(size_t)c] = (int32_t)~(uint32_t)(top[(size_t)c] >> 32);
        idx[(size_t)c] = L;
        const int i = (int)(L % Wx) - half_x, j = (int)((L / Wx) % Wy) - half_y;
        const int64_t a = L / ((int64_t)Wx * Wy);
        memcpy(&T[16 * (size_t)c], &Tb[16 * (size_t)a], 16 * sizeof(double));
        T[16 * (size_t)c + 3] += (double)i * cell;
        T[16 * (size_t)c + 7] += (double)j * cell;
    }
    put(out_T, T.data(), T.size() * sizeof(double));
    put(out_score, sc.data(), sc.size() * sizeof(int32_t));
    put(out_index, idx.data(), idx.size() * sizeof(int64_t));
    *out_num = k;
    PLS_API_END(ctx)
}
