// Correlative pose search on the kd map (no reference counterpart).  One exhaustive pipeline scores every pose of S
// scans in one pass: pls_kdmap_pose_search_scans, and pls_kdmap_pose_search as the batch of one scan.  Beside it,
// pls_kdmap_pose_search_pyramid finds the same candidates by branch and bound (kernels further down); it shares the box,
// occupancy and candidate-rule steps.
//
// The scans' rows are staged back to back and their volumes concatenated scan-major; every kernel finds its scan by
// binary search over per-scan offsets.  One occupancy grid serves every scan: the bounding box of the union of the scans'
// reachable boxes (base cells widened by the scan's window), so that every lookup of every scan lies inside it.
//   ps_box_kernel     : the base cell of every (scan, base, valid row), float64 with explicit roundings, reduced to each
//                       scan's min / max cell with 64-bit atomicMin / atomicMax (order-independent).  The host reads
//                       the boxes.
//   ps_occupy_kernel  : one pass over the map's points sets the bit of every map cell inside the grid (atomicOr), in a
//                       bit grid with x fastest, each (y, z) row padded to whole 32-bit words.
//   ps_score_kernel   : a block owns one (scan, base) and a tile of 32 i x 8 j shifts, warp w at j0 + w, lane l at
//                       i0 + l.  The base's cells stream through shared memory; a lane tests one bit per point -- a
//                       warp's 32 bits lie in one or two words of one row -- and counts in a register: exact integers.
//   ps_peak_kernel    : flags the candidates (score > 0, key strictly better than each 3x3x3 neighbour's in its scan).
//   ps_segment_kernel : the first compacted candidate of each scan, from the flag scan's positions.
//   ps_compact_kernel : keys (~score << 32) | L at exclusive_scan_flags positions (chunks of < 2^30 flags), values the
//                       scan.  radix_sort_pairs orders the keys -- score descending, then L ascending; with S > 1 a
//                       second, stable radix sort by scan brings each scan's candidates together in key order.
//   ps_top_kernel     : the first min(K, count) keys of each scan.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>

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

// Folds the warp's lo / hi into lane 0, which commits them to box[0..2] (atomicMin) and box[3..5] (atomicMax) when the
// warp saw a cell.  box starts at LLONG_MAX / LLONG_MIN.
__device__ __forceinline__ void commit_box(long long (&lo)[3], long long (&hi)[3], long long* __restrict__ box) {
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

// True when no neighbour of L = (a Wy + jj) Wx + ii in its 3x3x3 block of the A x Wy x Wx volume (no wrap-around) has
// a better key: a higher score, or the same score and a smaller L.  score(Ln, sn) sets sn to neighbour Ln's score and
// returns true, or returns false when Ln cannot compete.
template <typename Score, typename Lookup>
__device__ __forceinline__ bool beats_neighbours(int64_t L, Score sc, int64_t A, int Wy, int Wx, Lookup score) {
    const int ii = (int)(L % Wx);
    const int64_t t = L / Wx;
    const int jj = (int)(t % Wy);
    const int64_t a = t / Wy;
    for (int da = -1; da <= 1; ++da) {
        if (a + da < 0 || a + da >= A) continue;
        for (int dj = -1; dj <= 1; ++dj) {
            if (jj + dj < 0 || jj + dj >= Wy) continue;
            for (int dx = -1; dx <= 1; ++dx) {
                if (ii + dx < 0 || ii + dx >= Wx || (da == 0 && dj == 0 && dx == 0)) continue;
                const int64_t Ln = L + ((int64_t)da * Wy + dj) * Wx + dx;
                Score sn;
                if (score(Ln, sn) && (sn > sc || (sn == sc && Ln < L))) return false;
            }
        }
    }
    return true;
}

// The bit grid over a box: origin o (its min cell), extent e, wx words per (y, z) row.
struct PsGrid {
    long long o[3];
    long long e[3];
    uint32_t wx;
};

// One scan of a batch.
struct PsScan {
    int64_t row;   // first row in the staged scans
    int64_t n;
    int64_t base;  // first base in the concatenated bases
    int A, Wx, Wy, tiles_x, tiles_y;
};

// the s with off[s] <= x < off[s + 1], off [S + 1] ascending (scans with no entries are skipped)
__device__ __forceinline__ int ps_scan_of(const int64_t* __restrict__ off, int S, int64_t x) {
    int lo = 0, hi = S - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Scan s's box at box[6 s ..] from blocks [blk[s], blk[s+1]): min cell, then max cell, over every base and valid row
__global__ void __launch_bounds__(PS_THREADS) ps_box_kernel(const float* __restrict__ rows,
                                                            const double* __restrict__ bases,
                                                            const PsScan* __restrict__ sd,
                                                            const int64_t* __restrict__ blk, int S, double c,
                                                            long long* __restrict__ box) {
    const int s = ps_scan_of(blk, S, blockIdx.x);
    const PsScan d = sd[s];
    const float* scan = rows + 3 * d.row;
    const double* B = bases + 16 * d.base;
    const int64_t nblk = blk[s + 1] - blk[s], total = d.n * (int64_t)d.A;
    long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
    for (int64_t k = (blockIdx.x - blk[s]) * PS_THREADS + threadIdx.x; k < total; k += nblk * PS_THREADS) {
        const int64_t a = k / d.n, p = k - a * d.n;
        long long cell[3];
        if (!base_cell(B + 16 * a, scan[3 * p], scan[3 * p + 1], scan[3 * p + 2], c, cell[0], cell[1], cell[2])) continue;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            lo[r] = min(lo[r], cell[r]);
            hi[r] = max(hi[r], cell[r]);
        }
    }
    commit_box(lo, hi, box + 6 * s);
}

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

// Block b of scan s (blocks [blk[s], blk[s+1])): base a, shift tile (it, jt); lane i0 + lane, warp j0 + warp.
// scores[vol[s] + (a*Wy + jj)*Wx + ii].  Every scan's reachable box lies inside the grid g, so the cells need no bounds
// test.
__global__ void __launch_bounds__(PS_THREADS) ps_score_kernel(const float* __restrict__ rows,
                                                              const double* __restrict__ bases,
                                                              const PsScan* __restrict__ sd,
                                                              const int64_t* __restrict__ blk,
                                                              const int64_t* __restrict__ vol, int S, double c,
                                                              PsGrid g, const uint32_t* __restrict__ bits,
                                                              int32_t* __restrict__ scores) {
    __shared__ uint2 cells[PS_CHUNK];  // (word offset of the cell's row at shift (0, -half_y), x - origin at shift -half_x)
    __shared__ double T[16];
    const int s = ps_scan_of(blk, S, blockIdx.x);
    const PsScan d = sd[s];
    const int64_t b = blockIdx.x - blk[s];
    const int it = (int)(b % d.tiles_x);
    const int jt = (int)((b / d.tiles_x) % d.tiles_y);
    const int64_t a = b / ((int64_t)d.tiles_x * d.tiles_y);
    if (threadIdx.x < 16) T[threadIdx.x] = bases[16 * (d.base + a) + threadIdx.x];
    const float* scan = rows + 3 * d.row;
    const int64_t n = d.n;
    const int Wx = d.Wx, Wy = d.Wy;
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
                // relative to the grid's origin at shift (-half_x, -half_y): each lane adds its di, dj
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
    if (active) scores[vol[s] + (a * Wy + jj) * (int64_t)Wx + ii] = count;
}

// flags[G] = 1 for a candidate over the concatenated volumes, scan s's at [vol[s], vol[s+1]): score > 0 and a key
// strictly better than every neighbour's in its own scan's volume
__global__ void ps_peak_kernel(const int32_t* __restrict__ scores, const PsScan* __restrict__ sd,
                               const int64_t* __restrict__ vol, int S, uint8_t* __restrict__ flags) {
    const int64_t V = vol[S];
    for (int64_t G = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; G < V; G += (int64_t)gridDim.x * blockDim.x) {
        const int s_ = ps_scan_of(vol, S, G);
        const PsScan d = sd[s_];
        const int32_t* s = scores + vol[s_];
        const int64_t L = G - vol[s_];
        const int32_t sc = s[L];
        flags[G] = sc > 0 && beats_neighbours(L, sc, d.A, d.Wy, d.Wx, [&](int64_t Ln, int32_t& sn) {
                       sn = s[Ln];
                       return true;
                   });
    }
}

// seg[s] = the candidates of the scans before s (seg[S] = all of them): the compacted position at vol[s]
__global__ void ps_segment_kernel(const uint32_t* __restrict__ pos, const uint32_t* __restrict__ chunk_totals,
                                  int chunks, const int64_t* __restrict__ vol, int S, uint32_t* __restrict__ seg) {
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= S; s += gridDim.x * blockDim.x) {
        const int64_t L = vol[s];
        const int64_t full = s < S ? L / PS_SCAN_CHUNK : chunks;
        uint32_t at = s < S ? pos[L] : 0u;
        for (int64_t ch = 0; ch < full; ++ch) at += chunk_totals[ch];
        seg[s] = at;
    }
}

// keys[at] = (~score << 32) | L_local, vals[at] = s for every flagged entry; at adds the earlier flag chunks' totals
__global__ void ps_compact_kernel(const int32_t* __restrict__ scores, const uint8_t* __restrict__ flags,
                                  const uint32_t* __restrict__ pos, const uint32_t* __restrict__ chunk_totals,
                                  const int64_t* __restrict__ vol, int S, uint64_t* __restrict__ keys,
                                  uint32_t* __restrict__ vals) {
    const int64_t V = vol[S];
    for (int64_t G = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; G < V; G += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[G]) continue;
        uint32_t at = pos[G];
        for (int64_t ch = 0; ch < G / PS_SCAN_CHUNK; ++ch) at += chunk_totals[ch];
        const int s = ps_scan_of(vol, S, G);
        keys[at] = ((uint64_t)(~(uint32_t)scores[G]) << 32) | (uint64_t)(G - vol[s]);
        vals[at] = (uint32_t)s;
    }
}

// the second sort's input: key = the scan of the e-th candidate in key order, value = e
__global__ void ps_by_scan_kernel(const uint32_t* __restrict__ scan_of, int64_t num, uint64_t* __restrict__ keys,
                                  uint32_t* __restrict__ vals) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < num; e += (int64_t)gridDim.x * blockDim.x) {
        keys[e] = scan_of[e];
        vals[e] = (uint32_t)e;
    }
}

// top[s K + j] = the key of scan s's j-th candidate, j < min(K, seg[s+1] - seg[s]).  order: the key ranks sorted by
// scan, or NULL when the keys are already grouped by scan (one scan).
__global__ void ps_top_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ order,
                              const uint32_t* __restrict__ seg, int S, int K, uint64_t* __restrict__ top) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < (int64_t)S * K;
         c += (int64_t)gridDim.x * blockDim.x) {
        const int s = (int)(c / K), j = (int)(c % K);
        const uint32_t e = seg[s] + (uint32_t)j;
        if (e < seg[s + 1]) top[c] = keys[order ? order[e] : e];
    }
}

// ---- pls_kdmap_pose_search_pyramid: the same candidates by branch and bound over max-pooled bit grids --------------
//
// A node (a, I, J) at level k covers the shifts ii in [I 2^k, (I+1) 2^k), jj likewise, of base a (ii = i + half_x).
// Level k's grid B_k(X, Y, Z) is the OR of level 0 over [X, X + 2^k) x [Y, Y + 2^k), so #{p : B_k(cell_a(p) - half +
// (I 2^k, J 2^k)) set} bounds the score of every pose under the node.  Work lists hold int4 (a, I, J, bound), sorted
// by a: roots are made a-major and expansion keeps the parents' order.
constexpr int PY_THREADS = 256;
constexpr int PY_CHUNK = 512;  // staged cells per pass (24 B each)

// A (base, row)'s cell relative to the clipped grid at shift (-half_x, -half_y): x, y; row = Z * e[1], or -1 when Z
// lies outside the grid (the row then scores 0 at every shift) or the scan row is not finite.
struct PyCell {
    long long x, y, row;
};

// box[0..2] = min map cell, box[3..5] = max (pls_voxel_hash's coordinates; initialised to LLONG_MAX / LLONG_MIN)
__global__ void __launch_bounds__(PS_THREADS) ps_map_box_kernel(const float4* __restrict__ pts, int64_t m, double c,
                                                                long long* __restrict__ box) {
    long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
        const float4 p = pts[k];
        const long long cell[3] = {voxel_coord((double)p.x, c), voxel_coord((double)p.y, c), voxel_coord((double)p.z, c)};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            lo[r] = min(lo[r], cell[r]);
            hi[r] = max(hi[r], cell[r]);
        }
    }
    commit_box(lo, hi, box);
}

// dst = B_k from src = B_(k-1), s = 2^(k-1): each word ORs its own, its x + s bits (a funnel shift of the two words
// s bits on), and the same two at row y + s.  Bits past the grid's edge read 0.
__global__ void ps_pool_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, PsGrid g, long long s) {
    const long long wx = g.wx, words = wx * g.e[1] * g.e[2];
    const long long q = s >> 5;
    const uint32_t r = (uint32_t)(s & 31);
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < words; w += (long long)gridDim.x * blockDim.x) {
        const long long xw = w % wx, row = w / wx, y = row % g.e[1];
        auto pooled_x = [&](long long at) {  // the row's word xw | its bits x + s
            const long long rb = at - xw;
            const uint32_t lo = xw + q < wx ? src[rb + xw + q] : 0u;
            const uint32_t hi = xw + q + 1 < wx ? src[rb + xw + q + 1] : 0u;
            return src[at] | __funnelshift_r(lo, hi, r);
        };
        uint32_t v = pooled_x(w);
        if (y + s < g.e[1]) v |= pooled_x(w + s * wx);
        dst[w] = v;
    }
}

// cells[a n + p] for every base and scan row, computed once for every level and pass
__global__ void ps_pyr_cells_kernel(const float* __restrict__ scan, int64_t n, const double* __restrict__ bases, int A,
                                    double c, PsGrid g, int half_x, int half_y, PyCell* __restrict__ cells) {
    const int64_t total = n * (int64_t)A;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = k / n, p = k - a * n;
        long long cx, cy, cz;
        PyCell v = {0, 0, -1};
        if (base_cell(bases + 16 * a, scan[3 * p], scan[3 * p + 1], scan[3 * p + 2], c, cx, cy, cz)) {
            const long long Z = cz - g.o[2];
            if (Z >= 0 && Z < g.e[2]) v = {cx - half_x - g.o[0], cy - half_y - g.o[1], Z * g.e[1]};
        }
        cells[k] = v;
    }
}

// nodes[i].w = the node's bound at level k (its exact score at k = 0).  A block's lanes are 256 consecutive nodes;
// for each base among them, that base's cells stream through shared memory and its lanes count in a register.
// A block left or below the grid's edge that reaches into it reads B_k at the edge, which pools a superset: still a bound.
__global__ void __launch_bounds__(PY_THREADS) ps_pyr_score_kernel(const PyCell* __restrict__ cells, int64_t n,
                                                                  const uint32_t* __restrict__ bits, PsGrid g, int k,
                                                                  int4* __restrict__ nodes, int64_t count) {
    __shared__ PyCell staged[PY_CHUNK];
    const int64_t first = (int64_t)blockIdx.x * PY_THREADS, i = first + threadIdx.x;
    const int4 nd = i < count ? nodes[i] : make_int4(-1, 0, 0, 0);
    const int a_lo = nodes[first].x, a_hi = nodes[min(first + PY_THREADS, count) - 1].x;
    const long long span = 1ll << k, xs = (long long)nd.y << k, ys = (long long)nd.z << k;
    const unsigned long long ex = (unsigned long long)g.e[0], ey = (unsigned long long)g.e[1];
    int32_t ub = 0;
    for (int a = a_lo; a <= a_hi; ++a) {
        if (!__syncthreads_or(nd.x == a)) continue;
        const PyCell* src = cells + (int64_t)a * n;
        for (int64_t k0 = 0; k0 < n; k0 += PY_CHUNK) {
            const int len = (int)min((int64_t)PY_CHUNK, n - k0);
            __syncthreads();
            for (int t = threadIdx.x; t < len; t += PY_THREADS) staged[t] = src[k0 + t];
            __syncthreads();
            if (nd.x != a) continue;
#pragma unroll 4
            for (int t = 0; t < len; ++t) {
                const PyCell v = staged[t];
                if (v.row < 0) continue;
                long long X = v.x + xs, Y = v.y + ys;
                if (X < 0) X = X + span > 0 ? 0 : -1;
                if (Y < 0) Y = Y + span > 0 ? 0 : -1;
                if ((unsigned long long)X < ex && (unsigned long long)Y < ey)
                    ub += (int32_t)((__ldg(bits + (v.row + Y) * (long long)g.wx + (X >> 5)) >> (X & 31)) & 1u);
            }
        }
    }
    if (i < count) nodes[i].w = ub;
}

// flags[4 i + c] = 1 for child c = (dx, dy) = (c & 1, c >> 1) of node i at level k >= 1: bound >= tau and the child's
// first shift inside the window
__global__ void ps_pyr_branch_kernel(const int4* __restrict__ nodes, int64_t count, int k, int Wx, int Wy, int tau,
                                     uint8_t* __restrict__ flags) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < 4 * count; f += (int64_t)gridDim.x * blockDim.x) {
        const int4 nd = nodes[f >> 2];
        const long long I = 2ll * nd.y + (f & 1), J = 2ll * nd.z + ((f >> 1) & 1);
        flags[f] = nd.w >= tau && (I << (k - 1)) < Wx && (J << (k - 1)) < Wy;
    }
}

__global__ void ps_pyr_children_kernel(const int4* __restrict__ nodes, const uint8_t* __restrict__ flags,
                                       const uint32_t* __restrict__ pos, int64_t count, int4* __restrict__ out) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < 4 * count; f += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[f]) continue;
        const int4 nd = nodes[f >> 2];
        out[pos[f]] = make_int4(nd.x, 2 * nd.y + (int)(f & 1), 2 * nd.z + (int)((f >> 1) & 1), 0);
    }
}

// E_tau at level 0: flags[i] = score >= tau
__global__ void ps_pyr_keep_kernel(const int4* __restrict__ nodes, int64_t count, int tau, uint8_t* __restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        flags[i] = nodes[i].w >= tau;
}

__global__ void ps_pyr_exact_kernel(const int4* __restrict__ nodes, const uint8_t* __restrict__ flags,
                                    const uint32_t* __restrict__ pos, int64_t count, int Wx, int Wy,
                                    uint64_t* __restrict__ L, uint32_t* __restrict__ s) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[i]) continue;
        const int4 nd = nodes[i];
        L[pos[i]] = (uint64_t)(((int64_t)nd.x * Wy + nd.z) * Wx + nd.y);
        s[pos[i]] = (uint32_t)nd.w;
    }
}

// flags[e] = 1 for a candidate among E_tau sorted by L: no neighbour of its 3x3x3 block that is in E_tau has a better
// key.  A neighbour outside E_tau scores below tau <= s[e], so it cannot beat it.
__global__ void ps_pyr_peak_kernel(const uint64_t* __restrict__ L, const uint32_t* __restrict__ s, int64_t m, int A,
                                   int Wy, int Wx, uint8_t* __restrict__ flags) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
        flags[e] = beats_neighbours((int64_t)L[e], s[e], A, Wy, Wx, [&](int64_t Ln, uint32_t& sn) {
            int64_t lo = 0, hi = m;  // lower bound of Ln
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (L[mid] < (uint64_t)Ln) lo = mid + 1;
                else hi = mid;
            }
            if (lo == m || L[lo] != (uint64_t)Ln) return false;
            sn = s[lo];
            return true;
        });
    }
}

// keys[pos[e]] = (~score << 32) | e: sorted ascending, score descending, then e ascending, which is L ascending
__global__ void ps_pyr_rank_kernel(const uint32_t* __restrict__ s, const uint8_t* __restrict__ flags,
                                   const uint32_t* __restrict__ pos, int64_t m, uint64_t* __restrict__ keys,
                                   uint32_t* __restrict__ vals) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[e]) continue;
        keys[pos[e]] = ((uint64_t)(~s[e]) << 32) | (uint64_t)e;
        vals[pos[e]] = (uint32_t)e;
    }
}

// the first k candidates in key order: their L and score
__global__ void ps_pyr_top_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ L, int k,
                                  int64_t* __restrict__ out_L, int32_t* __restrict__ out_s) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= k) return;
    out_L[c] = (int64_t)L[keys[c] & 0xffffffffull];
    out_s[c] = (int32_t)~(uint32_t)(keys[c] >> 32);
}

// ---- host steps shared by the entry points ------------------------------------------------------------------------

// A refusal: PLS_E_INVALID with a printf-formatted message
[[noreturn]] __attribute__((format(printf, 1, 2))) void refuse(const char* fmt, ...) {
    char msg[384];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
    throw pls::Error{PLS_E_INVALID, msg};
}

// The refusals every search shares, fn naming the entry point: a kd map that holds points, and the cell size.
void require_search(const pls_context* ctx, const char* fn, double cell) {
    if (ctx->cfg.local_map_type != PLS_MAP_KDTREE) refuse("%s: needs a kd-tree local map", fn);
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    if (!(std::isfinite(cell) && cell > 0.0)) refuse("%s: cell must be finite and > 0", fn);
}

// count doubles of bases, host or device, in host memory
std::vector<double> host_bases(const double* bases, size_t count) {
    std::vector<double> Tb(count);
    if (is_device_ptr(bases)) PLS_CUDA(cudaMemcpy(Tb.data(), bases, count * sizeof(double), cudaMemcpyDeviceToHost));
    else memcpy(Tb.data(), bases, count * sizeof(double));
    return Tb;
}

// The bit grid over the cells lo..hi, both inclusive
PsGrid grid_over(const long long* lo, const long long* hi) {
    PsGrid g;
    for (int r = 0; r < 3; ++r) {
        g.o[r] = lo[r];
        g.e[r] = hi[r] - lo[r] + 1;
    }
    g.wx = (uint32_t)((g.e[0] + 31) / 32);
    return g;
}

// The grid's bits, x rows padded to whole words: what the bit limits bound
double grid_bits(const PsGrid& g) { return 32.0 * (double)((g.e[0] + 31) / 32) * (double)g.e[1] * (double)g.e[2]; }

size_t grid_words(const PsGrid& g) { return (size_t)g.wx * (size_t)g.e[1] * (size_t)g.e[2]; }

// The occupancy of the map's cells inside g in buf, cleared and filled; buf holds `levels` grids of g's size.
uint32_t* occupancy(pls_context* ctx, const PsGrid& g, double cell, DBuf& buf, int levels) {
    cudaStream_t st = ctx->stream;
    const size_t words = grid_words(g);
    buf.reserve(words * levels * sizeof(uint32_t), st);
    uint32_t* bits = buf.as<uint32_t>();
    PLS_CUDA(cudaMemsetAsync(bits, 0, words * sizeof(uint32_t), st));
    const int64_t M = ctx->kd.count;
    if (M > 0) {
        ps_occupy_kernel<<<blocks_for(M, 256, 16 * kNumSMs), 256, 0, st>>>(ctx->kd.store[ctx->kd.cur].as<float4>(), M,
                                                                           cell, g, bits);
        PLS_CHECK_LAUNCH();
    }
    return bits;
}

// T = the pose of entry L of a volume over `bases`: bases[a] moved by (i c, j c)
void pose_of(const double* bases, int64_t L, int half_x, int half_y, double cell, double* T) {
    const int Wx = 2 * half_x + 1, Wy = 2 * half_y + 1;
    const int i = (int)(L % Wx) - half_x, j = (int)((L / Wx) % Wy) - half_y;
    const int64_t a = L / ((int64_t)Wx * Wy);
    memcpy(T, bases + 16 * a, 16 * sizeof(double));
    T[3] += (double)i * cell;
    T[7] += (double)j * cell;
}

// Sub-arrays carved from one scratch buffer start on 256-byte boundaries, as whole allocations do.
size_t aligned(int64_t bytes) { return ((size_t)bytes + 255) & ~(size_t)255; }

PsScan describe(int64_t row, int64_t n, int64_t base, int A, int half_x, int half_y) {
    PsScan d;
    d.row = row;
    d.n = n;
    d.base = base;
    d.A = A;
    d.Wx = 2 * half_x + 1;
    d.Wy = 2 * half_y + 1;
    d.tiles_x = (d.Wx + 31) / 32;
    d.tiles_y = (d.Wy + PS_ROWS - 1) / PS_ROWS;
    return d;
}

// ps_box_kernel's blocks for one scan of n rows and A bases: 16 (base, row) pairs per thread, at most 8 per SM
int64_t box_blocks(int64_t n, int A) {
    return std::min<int64_t>((n * A + 16 * PS_THREADS - 1) / (16 * PS_THREADS), 8 * kNumSMs);
}

// the radix passes that order the scan ids 0..S-1
int scan_passes(int S) {
    int bytes = 1;
    while (bytes < 4 && (uint32_t)(S - 1) >> (8 * bytes)) ++bytes;
    return bytes;
}

// The exhaustive search of S scans, as the header defines pls_kdmap_pose_search_scans; pls_kdmap_pose_search is S = 1.
// fn names the entry point in refusals; with name_scans they also name the scan.
void search_scans(pls_context* ctx, const char* fn, bool name_scans, const float* const* scans, const int64_t* n, int S,
                  const double* bases, const int* num_bases, double cell, const int* half_x, const int* half_y, int K,
                  int32_t* out_scores, double* out_T, int32_t* out_score, int64_t* out_index, int* out_num) {
    // every argument is checked before anything is enqueued: a refused call changes nothing
    if (!(K >= 0 && K <= PLS_POSE_SEARCH_MAX_K)) refuse("%s: K must lie in [0, 1024]", fn);
    if (!(out_num && (K == 0 || (out_T && out_score && out_index))))
        refuse("%s: out_num, and for K > 0 out_T, out_score and out_index, must not be NULL", fn);
    char who_buf[96];
    auto who = [&](int s) {  // the prefix of scan s's refusals
        if (name_scans) snprintf(who_buf, sizeof(who_buf), "%s: scan %d", fn, s);
        else snprintf(who_buf, sizeof(who_buf), "%s", fn);
        return who_buf;
    };
    std::vector<PsScan> sd((size_t)S);
    std::vector<int64_t> off((size_t)3 * (S + 1));  // box blocks, score blocks, volumes: [S + 1] each
    int64_t* box_blk = off.data();
    int64_t* score_blk = box_blk + (S + 1);
    int64_t* vol = score_blk + (S + 1);
    int64_t rows = 0, A_total = 0;
    for (int s = 0; s < S; ++s) {
        if (!scans[s]) refuse("%s: the scan must not be NULL", who(s));
        if (!(n[s] > 0 && n[s] <= INT32_MAX)) refuse("%s: the scan must be [n,3] with 0 < n < 2^31", who(s));
        const int A = num_bases[s];
        if (A <= 0) refuse("%s: the bases must be [A,16] with A > 0", who(s));
        if (half_x[s] < 0 || half_y[s] < 0) refuse("%s: half_x and half_y must be >= 0", who(s));
        if (!(half_x[s] < (1 << 30) && half_y[s] < (1 << 30) &&
              (double)A * (2.0 * half_x[s] + 1) * (2.0 * half_y[s] + 1) < 2147483648.0))
            refuse("%s: A*(2*half_x+1)*(2*half_y+1) must be < 2^31", who(s));
        const PsScan d = sd[(size_t)s] = describe(rows, n[s], A_total, A, half_x[s], half_y[s]);
        box_blk[s + 1] = box_blk[s] + box_blocks(d.n, A);
        score_blk[s + 1] = score_blk[s] + (int64_t)A * d.tiles_x * d.tiles_y;
        vol[s + 1] = vol[s] + (int64_t)A * d.Wx * d.Wy;
        rows += d.n;
        A_total += A;
    }
    const int64_t V = vol[S];
    if (V >= (1ll << 31)) refuse("%s: the volumes together must hold fewer than 2^31 poses", fn);
    const std::vector<double> Tb = host_bases(bases, (size_t)A_total * 16);
    for (int s = 0; s < S; ++s)
        for (int64_t v = 16 * sd[(size_t)s].base; v < 16 * (sd[(size_t)s].base + sd[(size_t)s].A); ++v)
            if (!std::isfinite(Tb[(size_t)v])) refuse("%s: every base must be finite", who(s));

    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    // scratch of this stateless call: next_buf, never a buffer the map or an ICP keeps state in.  nb[1] holds, on
    // 256-byte boundaries: bases, boxes [S,6], chunk totals [8], segments [S+1], descriptors, offsets, top keys [S,K].
    DBuf* nb = ctx->next_buf;
    size_t at = 0;
    auto carve = [&](size_t bytes) { const size_t o = at; at += aligned((int64_t)bytes); return o; };
    const size_t o_bases = carve(Tb.size() * sizeof(double)), o_box = carve((size_t)S * 6 * sizeof(long long));
    const size_t o_tot = carve(8 * sizeof(uint32_t)), o_seg = carve((size_t)(S + 1) * sizeof(uint32_t));
    const size_t o_sd = carve(sd.size() * sizeof(PsScan)), o_off = carve(off.size() * sizeof(int64_t));
    const size_t o_top = carve((size_t)S * K * sizeof(uint64_t));
    // the inputs of the first launch, laid out as on the device up to the top keys, copied in one go
    std::vector<char> head(o_top);
    memcpy(head.data() + o_bases, Tb.data(), Tb.size() * sizeof(double));
    long long* box_init = reinterpret_cast<long long*>(head.data() + o_box);
    for (int s = 0; s < S; ++s)
        for (int r = 0; r < 3; ++r) box_init[6 * s + r] = LLONG_MAX, box_init[6 * s + 3 + r] = LLONG_MIN;
    memcpy(head.data() + o_sd, sd.data(), sd.size() * sizeof(PsScan));
    memcpy(head.data() + o_off, off.data(), off.size() * sizeof(int64_t));
    nb[1].reserve(at, st);
    char* blob = nb[1].as<char>();
    PLS_CUDA(cudaMemcpyAsync(blob, head.data(), head.size(), cudaMemcpyHostToDevice, st));
    const double* bases_dev = reinterpret_cast<const double*>(blob + o_bases);
    long long* box_dev = reinterpret_cast<long long*>(blob + o_box);
    uint32_t* totals_dev = reinterpret_cast<uint32_t*>(blob + o_tot);
    uint32_t* seg_dev = reinterpret_cast<uint32_t*>(blob + o_seg);
    const PsScan* sd_dev = reinterpret_cast<const PsScan*>(blob + o_sd);
    const int64_t* box_blk_dev = reinterpret_cast<const int64_t*>(blob + o_off);
    const int64_t* score_blk_dev = box_blk_dev + (S + 1);
    const int64_t* vol_dev = score_blk_dev + (S + 1);
    uint64_t* top_dev = reinterpret_cast<uint64_t*>(blob + o_top);
    // every scan's rows, back to back; one scan already on the device is read where it is
    const float* rows_dev;
    if (S == 1) {
        rows_dev = (const float*)to_device(ctx, scans[0], (size_t)n[0] * 3 * sizeof(float), nb[0]);
    } else {
        nb[0].reserve((size_t)rows * 3 * sizeof(float), st);
        for (int s = 0; s < S; ++s)
            PLS_CUDA(cudaMemcpyAsync(nb[0].as<float>() + 3 * sd[(size_t)s].row, scans[s], (size_t)n[s] * 3 * sizeof(float),
                                     cudaMemcpyDefault, st));
        rows_dev = nb[0].as<float>();
    }
    ps_box_kernel<<<(unsigned)box_blk[S], PS_THREADS, 0, st>>>(rows_dev, bases_dev, sd_dev, box_blk_dev, S, cell, box_dev);
    PLS_CHECK_LAUNCH();
    std::vector<long long> box((size_t)S * 6);
    PLS_CUDA(cudaMemcpyAsync(box.data(), box_dev, box.size() * sizeof(long long), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));

    // the shared grid: the union of the reachable boxes of the scans with a valid row
    long long lo[3], hi[3];
    bool any = false;
    for (int s = 0; s < S; ++s) {
        const long long* b = &box[(size_t)s * 6];
        if (b[0] > b[3]) continue;  // no valid row: every score 0, no candidate
        for (int r = 0; r < 6; ++r)
            if (!(b[r] > -PS_MAX_CELL && b[r] < PS_MAX_CELL))
                refuse("%s: a base cell lies beyond +-2^40 cells of the origin", who(s));
        const long long half[3] = {half_x[s], half_y[s], 0};
        long long own_lo[3], own_hi[3];
        for (int r = 0; r < 3; ++r) own_lo[r] = b[r] - half[r], own_hi[r] = b[3 + r] + half[r];
        const PsGrid own = grid_over(own_lo, own_hi);
        if (grid_bits(own) > (double)PLS_POSE_SEARCH_MAX_BITS)
            refuse("%s: the occupancy box of %lld x %lld x %lld cells (%.0f bits with word-padded x rows) exceeds "
                   "PLS_POSE_SEARCH_MAX_BITS (2^31); use a larger cell or a smaller window",
                   who(s), own.e[0], own.e[1], own.e[2], grid_bits(own));
        for (int r = 0; r < 3; ++r) {
            lo[r] = any ? std::min(lo[r], own_lo[r]) : own_lo[r];
            hi[r] = any ? std::max(hi[r], own_hi[r]) : own_hi[r];
        }
        any = true;
    }
    if (!any) {
        if (out_scores) {
            if (is_device_ptr(out_scores)) PLS_CUDA(cudaMemset(out_scores, 0, (size_t)V * sizeof(int32_t)));
            else memset(out_scores, 0, (size_t)V * sizeof(int32_t));
        }
        const std::vector<int> zeros((size_t)S, 0);
        put_out(out_num, zeros.data(), zeros.size() * sizeof(int));
        return;
    }
    const PsGrid g = grid_over(lo, hi);
    if (grid_bits(g) > (double)PLS_POSE_SEARCH_MAX_BITS)
        refuse("%s: the shared occupancy box of %lld x %lld x %lld cells (%.0f bits with word-padded x rows) exceeds "
               "PLS_POSE_SEARCH_MAX_BITS (2^31); search scans that lie far apart in separate calls",
               fn, g.e[0], g.e[1], g.e[2], grid_bits(g));

    const uint32_t* bits = occupancy(ctx, g, cell, nb[2], 1);
    nb[3].reserve((size_t)V * sizeof(int32_t), st);
    int32_t* scores = nb[3].as<int32_t>();
    ps_score_kernel<<<(unsigned)score_blk[S], PS_THREADS, 0, st>>>(rows_dev, bases_dev, sd_dev, score_blk_dev, vol_dev, S,
                                                                    cell, g, bits, scores);
    PLS_CHECK_LAUNCH();

    std::vector<uint32_t> seg((size_t)S + 1, 0u);
    std::vector<uint64_t> top;
    if (K > 0) {
        nb[4].reserve((size_t)V, st);
        nb[5].reserve((size_t)V * sizeof(uint32_t), st);
        uint8_t* flags = nb[4].as<uint8_t>();
        uint32_t* pos = nb[5].as<uint32_t>();
        ps_peak_kernel<<<blocks_for(V, 256, 16 * kNumSMs), 256, 0, st>>>(scores, sd_dev, vol_dev, S, flags);
        PLS_CHECK_LAUNCH();
        const int chunks = (int)((V + PS_SCAN_CHUNK - 1) / PS_SCAN_CHUNK);
        for (int ch = 0; ch < chunks; ++ch) {
            const int64_t o = (int64_t)ch * PS_SCAN_CHUNK;
            exclusive_scan_flags(ctx, flags + o, std::min(PS_SCAN_CHUNK, V - o), pos + o, totals_dev + ch);
        }
        ps_segment_kernel<<<blocks_for(S + 1, 256, 16 * kNumSMs), 256, 0, st>>>(pos, totals_dev, chunks, vol_dev, S,
                                                                                 seg_dev);
        PLS_CHECK_LAUNCH();
        PLS_CUDA(cudaMemcpyAsync(seg.data(), seg_dev, seg.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        const int64_t num = seg[(size_t)S];
        if (num > 0) {
            nb[6].reserve((size_t)num * sizeof(uint64_t), st);
            nb[7].reserve((size_t)num * sizeof(uint32_t), st);
            uint64_t* keys = nb[6].as<uint64_t>();
            uint32_t* vals = nb[7].as<uint32_t>();
            ps_compact_kernel<<<blocks_for(V, 256, 16 * kNumSMs), 256, 0, st>>>(scores, flags, pos, totals_dev, vol_dev,
                                                                                S, keys, vals);
            PLS_CHECK_LAUNCH();
            uint64_t* ko = nullptr;
            uint32_t* vo = nullptr;
            radix_sort_pairs(ctx, keys, vals, num, 8, &ko, &vo);  // eight passes: sorted back in keys, vals
            // one scan's candidates are already together in key order; more scans' are brought together by a stable
            // sort by scan, in the buffers of the spent flags and positions
            const uint32_t* order = nullptr;
            if (S > 1) {
                nb[4].reserve((size_t)num * sizeof(uint64_t), st);
                uint64_t* by_scan = nb[4].as<uint64_t>();
                uint32_t* ranks = nb[5].as<uint32_t>();
                ps_by_scan_kernel<<<blocks_for(num, 256, 16 * kNumSMs), 256, 0, st>>>(vals, num, by_scan, ranks);
                PLS_CHECK_LAUNCH();
                uint64_t* so = nullptr;
                uint32_t* oo = nullptr;
                radix_sort_pairs(ctx, by_scan, ranks, num, scan_passes(S), &so, &oo);
                order = oo;
            }
            ps_top_kernel<<<blocks_for((int64_t)S * K, 256, 16 * kNumSMs), 256, 0, st>>>(keys, order, seg_dev, S, K,
                                                                                         top_dev);
            PLS_CHECK_LAUNCH();
            top.resize((size_t)S * K);
            PLS_CUDA(cudaMemcpyAsync(top.data(), top_dev, top.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        }
    }
    if (out_scores)
        PLS_CUDA(cudaMemcpyAsync(out_scores, scores, (size_t)V * sizeof(int32_t), cudaMemcpyDefault, st));
    PLS_CUDA(cudaStreamSynchronize(st));

    std::vector<int> nums((size_t)S);
    std::vector<double> T((size_t)K * 16);
    std::vector<int32_t> sc((size_t)K);
    std::vector<int64_t> idx((size_t)K);
    for (int s = 0; s < S; ++s) {
        const int k = (int)std::min<int64_t>(K, (int64_t)seg[(size_t)s + 1] - seg[(size_t)s]);
        for (int c = 0; c < k; ++c) {
            const uint64_t key = top[(size_t)s * K + c];
            idx[(size_t)c] = (int64_t)(key & 0xffffffffull);
            sc[(size_t)c] = (int32_t)~(uint32_t)(key >> 32);
            pose_of(&Tb[16 * (size_t)sd[(size_t)s].base], idx[(size_t)c], half_x[s], half_y[s], cell, &T[16 * (size_t)c]);
        }
        if (k) {
            put_out(out_T + (size_t)s * K * 16, T.data(), (size_t)k * 16 * sizeof(double));
            put_out(out_score + (size_t)s * K, sc.data(), (size_t)k * sizeof(int32_t));
            put_out(out_index + (size_t)s * K, idx.data(), (size_t)k * sizeof(int64_t));
        }
        nums[(size_t)s] = k;
    }
    put_out(out_num, nums.data(), nums.size() * sizeof(int));
}

constexpr int PY_ROOT_SIDE = 16;  // kmax: the least level with at most 16 x 16 roots per base

// The next threshold of a pass that found fewer than K candidates: 3/4 of the last, at least one less, at least 1.
int next_tau(int tau) { return std::max(1, std::min(tau - 1, (int)((3ll * tau) / 4))); }

// The radix passes that order L < V: whole bytes, an even count, so that the sorted keys land back in place.
int l_passes(int64_t V) {
    int bytes = 1;
    while (bytes < 8 && (uint64_t)(V - 1) >> (8 * bytes)) ++bytes;
    return std::min(8, bytes + (bytes & 1));
}

}  // namespace

}  // namespace pls

using namespace pls;

extern "C" int pls_kdmap_pose_search(pls_context* ctx, const float* scan, int64_t n, const double* bases, int A,
                                     double cell, int half_x, int half_y, int K, int32_t* out_scores, double* out_T,
                                     int32_t* out_score, int64_t* out_index, int* out_num) {
    PLS_API_BEGIN(ctx)
    require_search(ctx, "pls_kdmap_pose_search", cell);
    PLS_REQUIRE(scan && bases, "pls_kdmap_pose_search: scan and bases must not be NULL");
    search_scans(ctx, "pls_kdmap_pose_search", false, &scan, &n, 1, bases, &A, cell, &half_x, &half_y, K, out_scores,
                 out_T, out_score, out_index, out_num);
    PLS_API_END(ctx)
}

extern "C" int pls_kdmap_pose_search_scans(pls_context* ctx, const float* const* scans, const int64_t* n, int S,
                                           const double* bases, const int* num_bases, double cell, const int* half_x,
                                           const int* half_y, int K, int32_t* out_scores, double* out_T,
                                           int32_t* out_score, int64_t* out_index, int* out_num) {
    PLS_API_BEGIN(ctx)
    require_search(ctx, "pls_kdmap_pose_search_scans", cell);
    PLS_REQUIRE(S > 0, "pls_kdmap_pose_search_scans: S must be > 0");
    PLS_REQUIRE(scans && n && bases && num_bases && half_x && half_y,
                "pls_kdmap_pose_search_scans: scans, n, bases, num_bases, half_x and half_y must not be NULL");
    search_scans(ctx, "pls_kdmap_pose_search_scans", true, scans, n, S, bases, num_bases, cell, half_x, half_y, K,
                 out_scores, out_T, out_score, out_index, out_num);
    PLS_API_END(ctx)
}

extern "C" int pls_kdmap_pose_search_pyramid(pls_context* ctx, const float* scan, int64_t n, const double* bases, int A,
                                             double cell, int half_x, int half_y, int K, double* out_T,
                                             int32_t* out_score, int64_t* out_index, int* out_num) {
    PLS_API_BEGIN(ctx)
    // every argument is checked before anything is enqueued: a refused call changes nothing
    require_search(ctx, "pls_kdmap_pose_search_pyramid", cell);
    PLS_REQUIRE(scan && bases, "pls_kdmap_pose_search_pyramid: scan and bases must not be NULL");
    PLS_REQUIRE(n > 0 && n <= INT32_MAX, "pls_kdmap_pose_search_pyramid: scan must be [n,3] with 0 < n < 2^31");
    PLS_REQUIRE(A > 0, "pls_kdmap_pose_search_pyramid: bases must be [A,16] with A > 0");
    PLS_REQUIRE(half_x >= 0 && half_y >= 0 && half_x < (1 << 30) && half_y < (1 << 30),
                "pls_kdmap_pose_search_pyramid: half_x and half_y must lie in [0, 2^30)");
    PLS_REQUIRE(K >= 1 && K <= PLS_POSE_SEARCH_MAX_K, "pls_kdmap_pose_search_pyramid: K must lie in [1, 1024]");
    PLS_REQUIRE(out_num && out_T && out_score && out_index,
                "pls_kdmap_pose_search_pyramid: out_T, out_score, out_index and out_num must not be NULL");
    const int Wx = 2 * half_x + 1, Wy = 2 * half_y + 1;
    PLS_REQUIRE((unsigned __int128)A * (unsigned)Wx * (unsigned)Wy < ((unsigned __int128)1 << 62),
                "pls_kdmap_pose_search_pyramid: A*(2*half_x+1)*(2*half_y+1) must be < 2^62");
    const int64_t V = (int64_t)A * Wx * Wy;
    if ((double)n * A * sizeof(PyCell) > (double)PLS_POSE_SEARCH_PYRAMID_MAX_CELL_BYTES)
        refuse("pls_kdmap_pose_search_pyramid: the cells of %lld rows x %d bases (%zu bytes each) exceed "
               "PLS_POSE_SEARCH_PYRAMID_MAX_CELL_BYTES (2^33); use fewer bases or a sparser scan",
               (long long)n, A, sizeof(PyCell));
    const std::vector<double> Tb = host_bases(bases, (size_t)A * 16);
    for (double v : Tb) PLS_REQUIRE(std::isfinite(v), "pls_kdmap_pose_search_pyramid: every base must be finite");

    cudaStream_t st = ctx->stream;
    map_stream_wait(ctx);
    // scratch of this stateless call: next_buf, never a buffer the map or an ICP keeps state in
    DBuf* nb = ctx->next_buf;
    const float* scan_dev = (const float*)to_device(ctx, scan, (size_t)n * 3 * sizeof(float), nb[0]);
    // nb[1]: the head (the base box, then the map box; ps_box_kernel's block offsets and the scan's descriptor), the
    // bases, the counts read back, the top K
    struct Head {
        long long box[12];
        int64_t blk[2];
        PsScan d;
    };
    const Head head = {{LLONG_MAX, LLONG_MAX, LLONG_MAX, LLONG_MIN, LLONG_MIN, LLONG_MIN,
                        LLONG_MAX, LLONG_MAX, LLONG_MAX, LLONG_MIN, LLONG_MIN, LLONG_MIN},
                       {0, box_blocks(n, A)},
                       describe(0, n, 0, A, half_x, half_y)};
    const size_t tail = sizeof(Head) + (size_t)A * 16 * sizeof(double) + 8 * sizeof(uint32_t);
    nb[1].reserve(tail + (size_t)PLS_POSE_SEARCH_MAX_K * (sizeof(int64_t) + sizeof(int32_t)), st);
    Head* head_dev = nb[1].as<Head>();
    double* bases_dev = reinterpret_cast<double*>(head_dev + 1);
    long long* box_dev = head_dev->box;
    uint32_t* total_dev = reinterpret_cast<uint32_t*>(bases_dev + (size_t)A * 16);
    int64_t* top_L = reinterpret_cast<int64_t*>(nb[1].as<char>() + tail);
    int32_t* top_s = reinterpret_cast<int32_t*>(top_L + PLS_POSE_SEARCH_MAX_K);
    PLS_CUDA(cudaMemcpyAsync(head_dev, &head, sizeof(head), cudaMemcpyHostToDevice, st));
    PLS_CUDA(cudaMemcpyAsync(bases_dev, Tb.data(), Tb.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    ps_box_kernel<<<(unsigned)head.blk[1], PS_THREADS, 0, st>>>(scan_dev, bases_dev, &head_dev->d, head_dev->blk, 1, cell,
                                                                box_dev);
    PLS_CHECK_LAUNCH();
    const int64_t M = ctx->kd.count;
    if (M > 0) {
        ps_map_box_kernel<<<blocks_for(M, PS_THREADS, 8 * kNumSMs), PS_THREADS, 0, st>>>(
            ctx->kd.store[ctx->kd.cur].as<float4>(), M, cell, box_dev + 6);
        PLS_CHECK_LAUNCH();
    }
    long long box[12];
    PLS_CUDA(cudaMemcpyAsync(box, box_dev, sizeof(box), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));
    *out_num = 0;
    if (box[0] > box[3]) return PLS_OK;  // no valid row: every score is 0, no candidate
    for (int r = 0; r < 6; ++r)
        PLS_REQUIRE(box[r] > -PS_MAX_CELL && box[r] < PS_MAX_CELL,
                    "pls_kdmap_pose_search_pyramid: a base cell lies beyond +-2^40 cells of the origin");
    // the grid: the reachable box (base cells widened by the window) clipped to the map's own cells
    const long long half[3] = {half_x, half_y, 0};
    long long lo[3], hi[3];
    for (int r = 0; r < 3; ++r) {
        lo[r] = std::max(box[r] - half[r], box[6 + r]);
        hi[r] = std::min(box[3 + r] + half[r], box[9 + r]);
        if (M == 0 || hi[r] < lo[r]) return PLS_OK;  // no map cell is reachable: every score is 0
    }
    const PsGrid g = grid_over(lo, hi);
    int kmax = 0;
    while (((int64_t)std::max(Wx, Wy) + (1ll << kmax) - 1) >> kmax > PY_ROOT_SIDE) ++kmax;
    const int levels = kmax + 1;
    if (grid_bits(g) * levels > (double)PLS_POSE_SEARCH_PYRAMID_MAX_BITS)
        refuse("pls_kdmap_pose_search_pyramid: %d pooled levels of the clipped occupancy grid of %lld x %lld x %lld "
               "cells (%.0f bits with word-padded x rows) exceed PLS_POSE_SEARCH_PYRAMID_MAX_BITS (2^36); use a "
               "larger cell or a smaller window",
               levels, g.e[0], g.e[1], g.e[2], grid_bits(g) * levels);
    const size_t words = grid_words(g);

    // B_0: occupancy of the map's cells inside the clipped grid; B_k pooled from B_(k-1), one launch per level
    uint32_t* bits = occupancy(ctx, g, cell, nb[2], levels);
    for (int k = 1; k <= kmax; ++k) {
        ps_pool_kernel<<<blocks_for((int64_t)words, 256, 16 * kNumSMs), 256, 0, st>>>(
            bits + (k - 1) * words, bits + k * words, g, 1ll << (k - 1));
        PLS_CHECK_LAUNCH();
    }
    nb[3].reserve((size_t)n * A * sizeof(PyCell), st);
    PyCell* cells = nb[3].as<PyCell>();
    ps_pyr_cells_kernel<<<blocks_for(n * (int64_t)A, 256, 16 * kNumSMs), 256, 0, st>>>(scan_dev, n, bases_dev, A, cell,
                                                                                        g, half_x, half_y, cells);
    PLS_CHECK_LAUNCH();

    auto over_capacity = [&](int level, int64_t count) {
        if (count > PLS_POSE_SEARCH_PYRAMID_MAX_NODES)
            refuse("pls_kdmap_pose_search_pyramid: %lld nodes survive at level %d, more than "
                   "PLS_POSE_SEARCH_PYRAMID_MAX_NODES (2^26)",
                   (long long)count, level);
    };
    auto score = [&](int4* nodes, int64_t count, int k) {
        ps_pyr_score_kernel<<<(unsigned)((count + PY_THREADS - 1) / PY_THREADS), PY_THREADS, 0, st>>>(
            cells, n, bits + (size_t)k * words, g, k, nodes, count);
        PLS_CHECK_LAUNCH();
    };
    auto read_total = [&]() {
        uint32_t t = 0;
        PLS_CUDA(cudaMemcpyAsync(&t, total_dev, sizeof(t), cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        return (int64_t)t;
    };

    // roots: every (a, I, J) at level kmax, a-major, scored once for every pass; their bounds come back for the first tau
    const int rx = (int)(((int64_t)Wx + (1ll << kmax) - 1) >> kmax), ry = (int)(((int64_t)Wy + (1ll << kmax) - 1) >> kmax);
    const int64_t R = (int64_t)A * rx * ry;
    over_capacity(kmax, R);
    std::vector<int4> roots((size_t)R);
    for (int64_t r = 0; r < R; ++r)
        roots[(size_t)r] = make_int4((int)(r / ((int64_t)rx * ry)), (int)(r % rx), (int)((r / rx) % ry), 0);
    nb[4].reserve((size_t)R * sizeof(int4), st);
    int4* roots_dev = nb[4].as<int4>();
    PLS_CUDA(cudaMemcpyAsync(roots_dev, roots.data(), (size_t)R * sizeof(int4), cudaMemcpyHostToDevice, st));
    score(roots_dev, R, kmax);
    PLS_CUDA(cudaMemcpyAsync(roots.data(), roots_dev, (size_t)R * sizeof(int4), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));

    DBuf* work[2] = {&nb[5], &nb[6]};
    int top_bound = 1;
    for (const int4& r : roots) top_bound = std::max(top_bound, r.w);

    // threshold passes: tau from the largest root bound (no pose scores more) down by next_tau until K candidates
    // score >= tau, or tau = 1.  A high tau prunes hard, so the early passes are cheap.
    std::vector<int64_t> hL;
    std::vector<int32_t> hs;
    for (int tau = top_bound;; tau = next_tau(tau)) {
        int4* cur = roots_dev;
        int64_t count = R;
        int wi = 0;  // the work buffer the next level goes to
        for (int k = kmax; k > 0 && count > 0; --k) {
            nb[7].reserve((size_t)count * 4 * (sizeof(uint32_t) + 1), st);
            uint32_t* pos = nb[7].as<uint32_t>();
            uint8_t* flags = reinterpret_cast<uint8_t*>(pos + (size_t)count * 4);
            ps_pyr_branch_kernel<<<blocks_for(4 * count, 256, 16 * kNumSMs), 256, 0, st>>>(cur, count, k, Wx, Wy, tau,
                                                                                            flags);
            PLS_CHECK_LAUNCH();
            exclusive_scan_flags(ctx, flags, 4 * count, pos, total_dev);
            const int64_t next = read_total();
            over_capacity(k - 1, next);
            if (next > 0) {
                work[wi]->reserve((size_t)next * sizeof(int4), st);
                int4* out = work[wi]->as<int4>();
                ps_pyr_children_kernel<<<blocks_for(4 * count, 256, 16 * kNumSMs), 256, 0, st>>>(cur, flags, pos, count,
                                                                                                  out);
                PLS_CHECK_LAUNCH();
                score(out, next, k - 1);
                cur = out;
                wi ^= 1;
            }
            count = next;
        }
        int64_t num = 0;
        if (count > 0) {
            // E_tau, sorted by L, in the work buffer cur is not in; the candidates' keys in the other one
            DBuf* eb = work[wi];
            DBuf* cb = work[wi ^ 1];
            nb[7].reserve((size_t)count * (sizeof(uint32_t) + 1), st);
            uint32_t* pos = nb[7].as<uint32_t>();  // 4-byte words first: flags need no alignment
            uint8_t* flags = reinterpret_cast<uint8_t*>(pos + count);
            ps_pyr_keep_kernel<<<blocks_for(count, 256, 16 * kNumSMs), 256, 0, st>>>(cur, count, tau, flags);
            PLS_CHECK_LAUNCH();
            exclusive_scan_flags(ctx, flags, count, pos, total_dev);
            const int64_t m = read_total();
            if (m > 0) {
                eb->reserve(aligned(m * sizeof(uint64_t)) + (size_t)m * sizeof(uint32_t), st);
                uint64_t* L = eb->as<uint64_t>();
                uint32_t* s = reinterpret_cast<uint32_t*>(eb->as<char>() + aligned(m * sizeof(uint64_t)));
                ps_pyr_exact_kernel<<<blocks_for(count, 256, 16 * kNumSMs), 256, 0, st>>>(cur, flags, pos, count, Wx, Wy,
                                                                                           L, s);
                PLS_CHECK_LAUNCH();
                uint64_t* ko = nullptr;
                uint32_t* vo = nullptr;
                radix_sort_pairs(ctx, L, s, m, l_passes(V), &ko, &vo);  // an even pass count: sorted in place
                ps_pyr_peak_kernel<<<blocks_for(m, 256, 16 * kNumSMs), 256, 0, st>>>(L, s, m, A, Wy, Wx, flags);
                PLS_CHECK_LAUNCH();
                exclusive_scan_flags(ctx, flags, m, pos, total_dev);
                num = read_total();
                if (num > 0 && (num >= K || tau == 1)) {
                    cb->reserve(aligned(num * sizeof(uint64_t)) + (size_t)num * sizeof(uint32_t), st);
                    uint64_t* keys = cb->as<uint64_t>();
                    uint32_t* vals = reinterpret_cast<uint32_t*>(cb->as<char>() + aligned(num * sizeof(uint64_t)));
                    ps_pyr_rank_kernel<<<blocks_for(m, 256, 16 * kNumSMs), 256, 0, st>>>(s, flags, pos, m, keys, vals);
                    PLS_CHECK_LAUNCH();
                    radix_sort_pairs(ctx, keys, vals, num, 8, &ko, &vo);
                    const int k = (int)std::min<int64_t>(K, num);
                    ps_pyr_top_kernel<<<(k + 255) / 256, 256, 0, st>>>(keys, L, k, top_L, top_s);
                    PLS_CHECK_LAUNCH();
                    hL.resize((size_t)k);
                    hs.resize((size_t)k);
                    PLS_CUDA(cudaMemcpyAsync(hL.data(), top_L, k * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
                    PLS_CUDA(cudaMemcpyAsync(hs.data(), top_s, k * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
                    PLS_CUDA(cudaStreamSynchronize(st));
                }
            }
        }
        if (num >= K || tau == 1) break;
    }

    const int k = (int)hL.size();
    std::vector<double> T((size_t)k * 16);
    for (int c = 0; c < k; ++c) pose_of(Tb.data(), hL[(size_t)c], half_x, half_y, cell, &T[16 * (size_t)c]);
    put_out(out_T, T.data(), T.size() * sizeof(double));
    put_out(out_score, hs.data(), hs.size() * sizeof(int32_t));
    put_out(out_index, hL.data(), hL.size() * sizeof(int64_t));
    *out_num = k;
    PLS_API_END(ctx)
}
