// Exact nearest-neighbour search over the kd local map (replaces the pykdtree queries of
// slam/odometry/local_map.py:385,405): a pyramid of hashed cell tables over ONE array of map points sorted by
// the Morton code of their level-0 cell, searched by WHOLE WARPS.  Device side only.
//
// Index layout (HBM; largely served from L2 at the BASELINE map sizes):
//   sorted[M]   float4  map points ordered by level-0 cell id (insertion order inside a cell); .w = bit-cast
//                       insertion index
//   normals[M]  float4  lazily computed unit normal of each map point; .w carries a state word:
//                       2 gen = claimed (queued for computation), 2 gen + 1 = valid, anything else = stale
//   table[l]    uint4   open-addressing hash table of level l: {cell id, gen, first, last}.  A level-l cell is the
//                       Morton prefix id0 >> 3 l (cube of side cell0 * 2^l) and owns a CONTIGUOUS range of `sorted`,
//                       so one sorted array serves every level.  Entries of older generations count as empty: no
//                       table is ever cleared.  Level `top` is a single cell holding the whole map.
//
// Search.  A warp owns a query.  Lanes 0..26 each probe one cell of the 3x3x3 block around the query (27 independent
// table loads = one L2 round trip); the candidate ranges are flattened with a warp scan and read 32 at a time, lane t
// taking candidate t -- consecutive lanes read consecutive float4 of a range, so a round is a handful of full 128-byte
// lines instead of 32 scattered sectors (the thread-per-cell scans of round 1 spent their time in L1 wavefronts).
// Every point closer than (cell side - margin) lies inside the block, so a best (or k-th best) distance below that is
// exact; otherwise the next coarser level is scanned (cells pruned by their box distance), up to the level that holds
// everything.  No tree, no stack, no divergent descent.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "eigen_device.cuh"

namespace pls {

constexpr int KD_COORD_BITS = 13;                       // quantisation bits per axis
constexpr int KD_COORD_MAX = (1 << KD_COORD_BITS) - 1;
constexpr int KD_MIN_B0 = 3;                            // level-0 cell ids then fit 30 bits (4 radix passes)
constexpr int KD_MAX_LEVELS = KD_COORD_BITS - KD_MIN_B0 + 1;  // levels 0 .. top, top <= 10
constexpr float KD_CELL_TARGET = 0.20f;   // default level-0 cell side, metres (PLS_KD_CELL overrides)
constexpr float KD_CELL_MARGIN = 2e-3f;   // quantisation slack, metres
constexpr int KD_KMAX = 32;               // k + 1 <= 32: warp_knn, one key per lane
constexpr int KD_KMAX_WIDE = 256;         // k + 1 <= 256: warp_knn_wide, up to 8 keys per lane
constexpr unsigned FULL = 0xffffffffu;

struct KdGridHeader {
    float mn[3];
    float scale;      // quantisation units per metre
    int b0;           // bits dropped per axis at level 0
    float cell0;      // level-0 cell side, metres
    int top;          // coarsest level = KD_COORD_BITS - b0 (one cell)
    int overflow[KD_MAX_LEVELS];
};

struct KdIndex {
    const float4* sorted;
    float4* normals;
    int M;
    uint32_t gen;                      // generation of this build (tables, normal states)
    const KdGridHeader* grid;
    const uint4* table[KD_MAX_LEVELS];
    uint32_t mask[KD_MAX_LEVELS];
    unsigned long long* stats;         // optional debug counters (PLS_KD_STATS=1), else null
};
// stats slots: 0 nn queries, 1 nn exact at level 0, 2 nn needing coarser levels, 3 nn candidates,
//              4 knn queries, 5 knn exact at level 0, 6 knn needing coarser levels, 7 knn candidates
__device__ __forceinline__ void kd_stat(const KdIndex& ix, int slot, unsigned long long v = 1ull) {
    if (ix.stats) atomicAdd(ix.stats + slot, v);
}

__device__ __forceinline__ uint32_t kd_spread10(uint32_t x) {  // 10 bits -> every third bit
    x &= 0x3ffu;
    x = (x | (x << 16)) & 0x030000ffu;
    x = (x | (x << 8)) & 0x0300f00fu;
    x = (x | (x << 4)) & 0x030c30c3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}
__device__ __forceinline__ uint32_t kd_cell_id(uint32_t cx, uint32_t cy, uint32_t cz) {
    return kd_spread10(cx) | (kd_spread10(cy) << 1) | (kd_spread10(cz) << 2);
}
__device__ __forceinline__ uint32_t kd_hash(uint32_t id) { return (id * 0x9E3779B1u) ^ (id >> 15); }

__device__ __forceinline__ float dist2_point(float x, float y, float z, const float4& p) {
    const float dx = x - p.x, dy = y - p.y, dz = z - p.z;
    return dx * dx + dy * dy + dz * dz;
}

// The grid header in registers (warp-uniform values).
struct KdGridLocal {
    float mnx, mny, mnz, scale, inv_scale;
    int b0, top;
};
__device__ __forceinline__ KdGridLocal kd_load_grid(const KdIndex& ix) {
    KdGridLocal g;
    g.mnx = __ldg(&ix.grid->mn[0]); g.mny = __ldg(&ix.grid->mn[1]); g.mnz = __ldg(&ix.grid->mn[2]);
    g.scale = __ldg(&ix.grid->scale);
    g.inv_scale = 1.f / g.scale;
    g.b0 = __ldg(&ix.grid->b0);
    g.top = __ldg(&ix.grid->top);
    return g;
}

// The cell of the 3x3x3 block (at `level`, around the query) owned by this lane: its point range [start, start+count)
// or count = 0 (lanes >= 27, cells outside the grid, empty cells).  `box2` receives the squared distance from the
// query to the cell's box, shrunk by the quantisation slack (a lower bound for every point binned into it): the caller
// drops cells farther than its current best.  The probe itself does not depend on any bound, so it can be in flight
// together with the load of the previous match.
// Returns the squared exactness radius of the block -- cell side + the query's clearance inside its own cell, minus the
// quantisation slack -- (FLT_MAX at the top level: the block then holds every point;
// negative if the level is unusable).  A query outside the grid is clamped to the border cell: all points lie on one
// side of it along that axis, so the block still holds everything within one cell side.
__device__ __forceinline__ float warp_probe_block(const KdIndex& ix, const KdGridLocal& g, int level, float x, float y,
                                                  float z, int lane, int& start, int& count, float& box2) {
    start = 0;
    count = 0;
    box2 = FLT_MAX;
    const int b = g.b0 + level;
    const int cmax = KD_COORD_MAX >> b;
    const float side_u = (float)(1 << b);                      // cell side in quantisation units
    const float fx = fminf(fmaxf((x - g.mnx) * g.scale, -1.0e6f), 1.0e6f);
    const float fy = fminf(fmaxf((y - g.mny) * g.scale, -1.0e6f), 1.0e6f);
    const float fz = fminf(fmaxf((z - g.mnz) * g.scale, -1.0e6f), 1.0e6f);
    const int cx = min(max(((int)floorf(fx)) >> b, 0), cmax);
    const int cy = min(max(((int)floorf(fy)) >> b, 0), cmax);
    const int cz = min(max(((int)floorf(fz)) >> b, 0), cmax);
    const bool usable = level >= g.top || !__ldg(&ix.grid->overflow[level]);
    if (lane < 27 && usable) {
        const int dz = lane / 9, rem = lane - dz * 9, dy = rem / 3, dx = rem - dy * 3;
        const int xx = cx + dx - 1, yy = cy + dy - 1, zz = cz + dz - 1;
        if (xx >= 0 && xx <= cmax && yy >= 0 && yy <= cmax && zz >= 0 && zz <= cmax) {
            const uint32_t id = kd_cell_id((uint32_t)xx, (uint32_t)yy, (uint32_t)zz);
            const uint4* __restrict__ table = ix.table[level];
            const uint32_t mask = ix.mask[level];
            uint32_t h = kd_hash(id) & mask;
            uint4 e = __ldg(table + h);
            // box distance while the probe is in flight
            const float lox = ((float)xx * side_u - fx), hix = (fx - (float)(xx + 1) * side_u);
            const float loy = ((float)yy * side_u - fy), hiy = (fy - (float)(yy + 1) * side_u);
            const float loz = ((float)zz * side_u - fz), hiz = (fz - (float)(zz + 1) * side_u);
            const float ax = fmaxf(fmaxf(lox, hix) * g.inv_scale - KD_CELL_MARGIN, 0.f);
            const float ay = fmaxf(fmaxf(loy, hiy) * g.inv_scale - KD_CELL_MARGIN, 0.f);
            const float az = fmaxf(fmaxf(loz, hiz) * g.inv_scale - KD_CELL_MARGIN, 0.f);
            box2 = ax * ax + ay * ay + az * az;
            for (int probe = 0; probe < 64; ++probe) {
                if (e.y != ix.gen) break;              // empty (or stale generation): the cell holds no point
                if (e.x == id) {
                    start = (int)e.z;
                    count = (int)e.w - (int)e.z + 1;
                    break;
                }
                h = (h + 1) & mask;
                e = __ldg(table + h);
            }
        }
    }
    if (level >= g.top) return FLT_MAX;
    if (!usable) return -1.f;  // this level's table was too small: nothing scanned, nothing proven
    // every point outside the block is at least one cell side PLUS the query's distance to the nearest face of its
    // own cell away (zero for a query clamped in from outside the grid)
    const float ox = fminf(fx - (float)cx * side_u, (float)(cx + 1) * side_u - fx);
    const float oy = fminf(fy - (float)cy * side_u, (float)(cy + 1) * side_u - fy);
    const float oz = fminf(fz - (float)cz * side_u, (float)(cz + 1) * side_u - fz);
    const float own = fmaxf(fminf(fminf(ox, oy), oz), 0.f);
    const float cell = (side_u + own) * g.inv_scale - KD_CELL_MARGIN;
    return cell > 0.f ? cell * cell : -1.f;
}


// arg-min of (d, i) over the warp with two REDUX instructions (d >= 0, so the float's bit pattern orders like its
// value; ties: smaller index).  The result lands in every lane; (FLT_MAX, -1) if no lane holds a candidate.
__device__ __forceinline__ void warp_argmin(float& d, int& i) {
    const unsigned bits = __float_as_uint(d);
    const unsigned m = __reduce_min_sync(FULL, bits);
    const unsigned wi = __reduce_min_sync(FULL, bits == m ? (unsigned)i : 0xffffffffu);
    d = __uint_as_float(m);
    i = (int)wi;
}

// Inclusive warp scan of the per-lane range sizes; returns the total.
__device__ __forceinline__ int warp_scan_counts(int count, int lane, int& incl) {
    incl = count;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += v;
    }
    return __shfl_sync(FULL, incl, 31);
}

// Index (into `sorted`) of the t-th candidate of the concatenated ranges: the owner cell is the number of lanes whose
// inclusive prefix is <= t (the prefixes are non-decreasing), found by a 5-step search over lane registers.
__device__ __forceinline__ int warp_candidate(int incl, int adj /* = start - exclusive prefix */, int t) {
    int c = 0;
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const int v = __shfl_sync(FULL, incl, c + s - 1);
        if (v <= t) c += s;
    }
    return __shfl_sync(FULL, adj, c) + t;
}

// The squared distance of a transformed query p to its match q in float64, every operation rounded on its own (no
// contraction): ((dx dx + dy dy) + dz dz), dx = (double)p_x - (double)q_x -- numpy's element-wise float64 bits.
__device__ __forceinline__ double match_d2_f64(const float* p, const float4& q) {
    const double dx = __dsub_rn((double)p[0], (double)q.x);
    const double dy = __dsub_rn((double)p[1], (double)q.y);
    const double dz = __dsub_rn((double)p[2], (double)q.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// The correspondence gate of a gated registration (pls_register_scans_gated): a query p whose exact 1-NN q has
// match_d2_f64(p, q) <= max_d2 is an inlier; every other query is an outlier and has no match.
//   g2    G, the float32 bound of the search: every inlier's float32 d^2 (dist2_point) is strictly below it.
//         Derivation (u = 2^-24, s = the exact squared distance of the two float32 points):
//           float64: dx = (p_x - q_x)(1 + e), |e| <= 2^-53, then three products and two sums, each rounded once, so
//                    match_d2_f64 >= s (1 - 2^-53)^5 and an inlier has s <= max_d2 (1 + 6 2^-53);
//           float32: the difference of two floats is rounded once (exact when subnormal); dist2_point squares and sums
//                    with at most three more roundings whatever the FMA contraction, so
//                    dist2_point <= s (1 + u)^5 + 3 2^-150 (underflow) <= s (1 + 5.01 u) + 2^-147;
//           together dist2_point < max_d2 (1 + 2^-20) + 2^-126, with room: 5.01 u + 6 2^-53 < 2^-20 / 3.
//         kd_gate_of rounds that bound up to float32 (+inf once it passes FLT_MAX: the search is never cut short).
//   dmax  max_distance rounded up to float32 (+inf above FLT_MAX): the outlier proof of match_proven<true>.
struct KdGate {
    double max_d2;
    float g2;
    float dmax;
};

// Exact 1-NN of (x, y, z) by the whole warp; every lane returns the same sorted position (-1 if the map is empty).
// `hint` (a sorted position or -1, warp-uniform) only seeds the pruning bound; its load overlaps the level-0 probes.
// *cand_out (optional) accumulates the number of candidates tested.
// *second_out receives a lower bound of the squared distance from the query to every map point OTHER than the winner
// (the runner-up inside the scanned block, the boxes of the cells that were pruned, the block's exactness radius):
// as long as the query moves by less than the gap between the two, the winner stays the nearest neighbour -- the next
// ICP iterations verify that instead of searching again (kd_icp_refine_kernel).
// GATE (a gated registration, KdGate): the climb also stops at the first level whose exactness radius r2 is at least
// G = gate.g2.  Every inlier's float32 d^2 is below G, so an inlier lies inside that block and the search ends at the
// very level -- with the very match and runner-up bound -- of the ungated search; a winner beyond r2 is then an outlier,
// and so is every point outside the block.  An outlier (no candidate, or match_d2_f64 > max_d2) returns -1, and
// *second_out becomes a lower bound of the squared distance to EVERY map point: min(best, runner-up bound).  A level
// whose table overflowed (r2 < 0) proves nothing and never stops the climb.
template <bool GATE = false>
__device__ __forceinline__ int warp_nearest(const KdIndex& ix, const KdGridLocal& g, float x, float y, float z, int hint,
                                            int lane, int* cand_out, float* second_out, KdGate gate = KdGate{}) {
    float best = FLT_MAX, second = FLT_MAX;
    int best_i = -1;
    float4 hp = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool has_hint = hint >= 0 && hint < ix.M;
    if (has_hint) hp = __ldg(ix.sorted + hint);
    if (lane == 0) kd_stat(ix, 0);
    for (int level = 0; level <= g.top; ++level) {
        int start, count;
        float box2;
        const float r2 = warp_probe_block(ix, g, level, x, y, z, lane, start, count, box2);
        if (level == 0 && has_hint) {
            best = dist2_point(x, y, z, hp);
            best_i = hint;
        }
        float l2 = FLT_MAX;          // this lane's bound for points other than its own best
        if (box2 > best) {           // nothing in that cell can beat (or tie) the bound ...
            if (count > 0) l2 = box2;  // ... but its points may be the runner-up
            count = 0;
        }
        int incl;
        const int total = warp_scan_counts(count, lane, incl);
        const int adj = start - (incl - count);
        float ld = best;
        int li = best_i;
        for (int base = 0; base < total; base += 32) {
            const int t = base + lane;
            const bool active = t < total;
            const int idx = warp_candidate(incl, adj, active ? t : total - 1);
            if (active) {
                const float d = dist2_point(x, y, z, __ldg(ix.sorted + idx));
                if (d < ld || (d == ld && (unsigned)idx < (unsigned)li)) {
                    l2 = fminf(l2, ld);
                    ld = d;
                    li = idx;
                } else if (idx != li) {
                    l2 = fminf(l2, d);
                }
            }
        }
        float wd = ld;
        int wi = li;
        warp_argmin(wd, wi);
        if (li != wi) l2 = fminf(l2, ld);  // this lane's best lost: it is a runner-up candidate
        const float inner = __uint_as_float(__reduce_min_sync(FULL, __float_as_uint(l2)));  // runner-up inside the block
        second = r2 >= 0.f ? fminf(inner, r2) : inner;  // anything outside the block is at least r2 away
        best = wd;
        best_i = wi;
        if (cand_out) *cand_out += total;
        if (ix.stats && lane == 0) {
            kd_stat(ix, 3, (unsigned long long)total);
            if (level == 0) kd_stat(ix, (best_i >= 0 && best <= r2) ? 1 : 2);
        }
        if (best_i >= 0 && best <= r2) break;
        if constexpr (GATE)
            if (r2 >= gate.g2) break;
    }
    if constexpr (GATE) {
        const float p[3] = {x, y, z};
        if (best_i < 0 || !(match_d2_f64(p, __ldg(ix.sorted + best_i)) <= gate.max_d2)) {
            second = fminf(best, second);
            best_i = -1;
        }
    }
    if (second_out) *second_out = second;
    return best_i;
}

// K-NN candidates compare as ONE 64-bit key: the bits of d^2 (>= 0, so they order like the value) above the sorted
// position -- the order (distance, then position) of the neighbour lists.  KNN_NONE: no candidate.
constexpr unsigned long long KNN_NONE = ~0ull;
__device__ __forceinline__ unsigned long long knn_key(float d, int idx) {
    return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
}

// The warp's smallest key (two REDUX: the distance bits, then the position among the lanes that hold that distance).
__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long k) {
    const unsigned hi = __reduce_min_sync(FULL, (unsigned)(k >> 32));
    const unsigned lo = __reduce_min_sync(FULL, (unsigned)(k >> 32) == hi ? (unsigned)k : 0xffffffffu);
    return ((unsigned long long)hi << 32) | lo;
}

// Level 0, at most 32 R candidates: lane r < K returns the r-th smallest key (KNN_NONE past the last candidate).
//   * every lane sorts its R candidates (t = s * 32 + lane) ascending (a small compare-exchange network);
//   * K rounds: the warp's minimum over the lane heads, the owner pops its head (a register shift).
template <int R>
__device__ __forceinline__ unsigned long long knn_select_small(const KdIndex& ix, float x, float y, float z, int K, int lane,
                                                               int incl, int adj, int total) {
    unsigned long long s[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
        const int t = j * 32 + lane;
        const bool active = t < total;
        const int idx = warp_candidate(incl, adj, active ? t : total - 1);
        s[j] = active ? knn_key(dist2_point(x, y, z, __ldg(ix.sorted + idx)), idx) : KNN_NONE;
    }
    // insertion network: after pass p the first p + 1 entries are ordered
#pragma unroll
    for (int p = 1; p < R; ++p) {
#pragma unroll
        for (int q = p; q >= 1; --q) {
            const unsigned long long lo = min(s[q - 1], s[q]), hi = max(s[q - 1], s[q]);
            s[q - 1] = lo;
            s[q] = hi;
        }
    }
    unsigned long long out = KNN_NONE;
    for (int r = 0; r < K; ++r) {
        const unsigned long long m = warp_min_key(s[0]);
        if (m == KNN_NONE) break;  // nothing left anywhere
        if (s[0] == m) {           // keys are unique: exactly one lane pops
#pragma unroll
            for (int j = 0; j + 1 < R; ++j) s[j] = s[j + 1];
            s[R - 1] = KNN_NONE;
        }
        if (lane == r) out = m;
    }
    return out;
}

// Bitonic sort of one key per lane, ascending with the lane index (15 compare-exchange stages over shuffles).
__device__ __forceinline__ unsigned long long warp_sort_keys(unsigned long long v, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const unsigned long long o = __shfl_xor_sync(FULL, v, j);
            v = (((lane & j) == 0) == ((lane & k) == 0)) ? min(v, o) : max(v, o);
        }
    }
    return v;
}

// The 32 smallest of two ascending lane-sorted lists, ascending: the element-wise minimum of one list and the other
// reversed is a bitonic sequence holding them, which five merge stages sort.
__device__ __forceinline__ unsigned long long warp_merge_keys(unsigned long long a, unsigned long long b, int lane) {
    unsigned long long v = min(a, __shfl_sync(FULL, b, 31 - lane));
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) {
        const unsigned long long o = __shfl_xor_sync(FULL, v, j);
        v = (lane & j) ? max(v, o) : min(v, o);
    }
    return v;
}

// Exact K-NN (K <= 32, warp-uniform) of (x, y, z): on return lane r < found holds the sorted position of the r-th
// nearest point (ascending by (distance, position)), other lanes -1; returns the number found (min(K, M)).
// `stage` is a warp-private shared buffer of KNN_STAGE keys.
//   * Level 0 (a 27-cell block of the BASELINE maps holds 30-80 points): up to 128 candidates are selected by
//     knn_select_small.
//   * Every coarser level (and a denser level-0 block) streams its candidates through a filter: the K-th key of the
//     previous level bounds this level's K-th from above (its block is a superset), so only keys <= that bound survive.
//     Survivors are compacted into `stage` with a ballot; every 32 of them are sorted and merged into the running 32
//     best.  If exactly K survive, they are the previous level's K: the list stands as it is.  A level whose table
//     overflowed is skipped: it scans nothing and leaves the list and its bound alone.
constexpr int KNN_STAGE = 64;
__device__ __forceinline__ int warp_knn(const KdIndex& ix, const KdGridLocal& g, float x, float y, float z, int K, int lane,
                                        int& out_i, int* cand_out, unsigned long long* stage) {
    unsigned long long kept = KNN_NONE;   // lane r < K: r-th smallest key so far
    unsigned long long bound = KNN_NONE;  // K-th key of the previous (finer) level
    float bound_d = FLT_MAX;              // ... its distance
    int found = 0;
    if (lane == 0) kd_stat(ix, 4);
    const unsigned lanes_below = (1u << lane) - 1u;
    for (int level = 0; level <= g.top; ++level) {
        int start, count;
        float box2;
        const float r2 = warp_probe_block(ix, g, level, x, y, z, lane, start, count, box2);
        if (r2 < 0.f) {  // this level's table overflowed: nothing scanned, the list of the finer level stands
            if (ix.stats && lane == 0 && level == 0) kd_stat(ix, 6);
            continue;
        }
        if (box2 > bound_d) count = 0;
        int incl;
        const int total = warp_scan_counts(count, lane, incl);
        const int adj = start - (incl - count);
        if (cand_out) *cand_out += total;
        if (ix.stats && lane == 0) kd_stat(ix, 7, (unsigned long long)total);
        if (bound == KNN_NONE && total <= 64) {
            kept = knn_select_small<2>(ix, x, y, z, K, lane, incl, adj, total);
        } else if (bound == KNN_NONE && total <= 128) {
            kept = knn_select_small<4>(ix, x, y, z, K, lane, incl, adj, total);
        } else {
            unsigned long long best = KNN_NONE;
            int staged = 0, survivors = 0;
            bool merged = false;
            for (int base = 0; base < total; base += 32) {
                const int t = base + lane;
                const bool active = t < total;
                const int idx = warp_candidate(incl, adj, active ? t : total - 1);
                unsigned long long key = KNN_NONE;
                if (active) key = knn_key(dist2_point(x, y, z, __ldg(ix.sorted + idx)), idx);
                const bool keep = active && key <= bound;
                const unsigned b = __ballot_sync(FULL, keep);
                if (keep) stage[staged + __popc(b & lanes_below)] = key;
                staged += __popc(b);
                survivors += __popc(b);
                if (staged >= 32) {
                    __syncwarp();
                    const unsigned long long c = warp_sort_keys(stage[lane], lane);
                    best = merged ? warp_merge_keys(best, c, lane) : c;
                    merged = true;
                    __syncwarp();
                    if (lane < staged - 32) stage[lane] = stage[32 + lane];
                    staged -= 32;
                    __syncwarp();
                }
            }
            // `kept` still holds the K keys that set `bound` (found == K): if exactly K survive, they are those K
            if (found != K || survivors != K) {
                if (staged > 0) {
                    __syncwarp();
                    const unsigned long long c = warp_sort_keys(lane < staged ? stage[lane] : KNN_NONE, lane);
                    best = merged ? warp_merge_keys(best, c, lane) : c;
                }
                kept = lane < K ? best : KNN_NONE;
            }
            __syncwarp();  // `stage` is reused by the next level
        }
        found = __popc(__ballot_sync(FULL, kept != KNN_NONE));
        const unsigned long long kth = __shfl_sync(FULL, kept, K - 1);
        const bool exact = (found == K && __uint_as_float((unsigned)(kth >> 32)) <= r2) || level >= g.top;
        if (ix.stats && lane == 0 && level == 0) kd_stat(ix, exact ? 5 : 6);
        if (exact) break;
        if (found == K) {
            bound = kth;
            bound_d = __uint_as_float((unsigned)(kth >> 32));
        }
    }
    out_i = kept != KNN_NONE ? (int)(unsigned)kept : -1;
    return found;
}

// Second moments about map point c of its k nearest OTHER map points (entry 0 of the (k+1)-NN list is the point
// itself): float32 sums taken sequentially in ascending-distance order and divided by k, as numpy's
// `.mean(axis=1)` forms them (slam/odometry/local_map.py:411-413).  Lane j holds neighbour j (nb_i); every lane
// returns the same six moments.
__device__ __forceinline__ void warp_second_moments(const KdIndex& ix, const float4& c, int k, int found, int nb_i, int lane,
                                                    float* cov) {
    float dx = 0.f, dy = 0.f, dz = 0.f;
    if (lane >= 1 && lane < found) {
        const float4 q = __ldg(ix.sorted + nb_i);
        dx = __fsub_rn(q.x, c.x);
        dy = __fsub_rn(q.y, c.y);
        dz = __fsub_rn(q.z, c.z);
    }
    float sxx = 0.f, sxy = 0.f, sxz = 0.f, syy = 0.f, syz = 0.f, szz = 0.f;
    for (int j = 1; j < found; ++j) {
        const float bx = __shfl_sync(FULL, dx, j), by = __shfl_sync(FULL, dy, j), bz = __shfl_sync(FULL, dz, j);
        sxx = __fadd_rn(sxx, __fmul_rn(bx, bx));
        sxy = __fadd_rn(sxy, __fmul_rn(bx, by));
        sxz = __fadd_rn(sxz, __fmul_rn(bx, bz));
        syy = __fadd_rn(syy, __fmul_rn(by, by));
        syz = __fadd_rn(syz, __fmul_rn(by, bz));
        szz = __fadd_rn(szz, __fmul_rn(bz, bz));
    }
    const float kk = (float)k;
    cov[0] = __fdiv_rn(sxx, kk); cov[1] = __fdiv_rn(sxy, kk); cov[2] = __fdiv_rn(sxz, kk);
    cov[3] = __fdiv_rn(syy, kk); cov[4] = __fdiv_rn(syz, kk); cov[5] = __fdiv_rn(szz, kk);
}

// ---- wide lists: K = k + 1 in 33 ... 256 ---------------------------------------------------------------------------
// A list of 32 R keys lives in R registers per lane, entry e = r * 32 + lane in register r: entry j of a neighbour list is
// in lane j % 32, register j / 32.  Keys are unique (they carry the sorted position), so the order is total.

// The key of entry r * 32 + sel_lane, every lane (r warp-uniform; a select chain keeps the list in registers).
template <int R>
__device__ __forceinline__ unsigned long long wide_entry(const unsigned long long (&a)[R], int r, int sel_lane) {
    unsigned long long v = a[0];
#pragma unroll
    for (int j = 1; j < R; ++j)
        if (j == r) v = a[j];
    return __shfl_sync(FULL, v, sel_lane);
}

// The 32 R smallest of an ascending list `a` of 32 R keys and an ascending 32-key list b (one per lane), ascending in a.
// Padded with KNN_NONE to 32 R entries and reversed, b is non-increasing; its element-wise minimum with a is a bitonic
// sequence holding the 32 R smallest, which log2(32 R) merge stages sort: the strides of 32 and more pair registers of
// one lane, the shorter ones lanes of one register.
template <int R>
__device__ __forceinline__ void warp_merge_wide(unsigned long long (&a)[R], unsigned long long b, int lane) {
    a[R - 1] = min(a[R - 1], __shfl_sync(FULL, b, 31 - lane));
#pragma unroll
    for (int j = R / 2; j > 0; j >>= 1) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if ((r & j) == 0) {
                const unsigned long long lo = min(a[r], a[r + j]), hi = max(a[r], a[r + j]);
                a[r] = lo;
                a[r + j] = hi;
            }
        }
    }
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const unsigned long long o = __shfl_xor_sync(FULL, a[r], j);
            a[r] = (lane & j) ? max(a[r], o) : min(a[r], o);
        }
    }
}

// Exact K-NN for 32 < K <= 32 R (warp-uniform): the same list as warp_knn would give with room for K keys -- the order
// (float32 d^2, sorted position), the cell-pyramid walk, the overflowed-level rule and the bound of the finer level's
// K-th key.  On return entry j < found of `kept` (lane j % 32, register j / 32) holds the key of the j-th nearest point,
// entries past it KNN_NONE; returns found = min(K, M).  `stage` is a warp-private shared buffer of KNN_STAGE keys.
// Every level streams its candidates: the keys at or below the bound are compacted into `stage`, and every 32 of them
// are sorted (warp_sort_keys) and merged into the level's running list (warp_merge_wide).  Once that list holds K keys,
// its K-th key bounds the level's remaining candidates too.  No level keeps the finer level's list: each rebuilds its
// own from its block.
template <int R>
__device__ __forceinline__ int warp_knn_wide(const KdIndex& ix, const KdGridLocal& g, float x, float y, float z, int K,
                                             int lane, unsigned long long (&kept)[R], int* cand_out,
                                             unsigned long long* stage) {
#pragma unroll
    for (int r = 0; r < R; ++r) kept[r] = KNN_NONE;
    unsigned long long bound = KNN_NONE;  // K-th key of the previous (finer) level
    float bound_d = FLT_MAX;              // ... its distance
    int found = 0;
    const int kr = (K - 1) >> 5, kl = (K - 1) & 31;  // where entry K - 1 lives
    if (lane == 0) kd_stat(ix, 4);
    const unsigned lanes_below = (1u << lane) - 1u;
    for (int level = 0; level <= g.top; ++level) {
        int start, count;
        float box2;
        const float r2 = warp_probe_block(ix, g, level, x, y, z, lane, start, count, box2);
        if (r2 < 0.f) {  // this level's table overflowed: nothing scanned, the list of the finer level stands
            if (ix.stats && lane == 0 && level == 0) kd_stat(ix, 6);
            continue;
        }
        if (box2 > bound_d) count = 0;
        int incl;
        const int total = warp_scan_counts(count, lane, incl);
        const int adj = start - (incl - count);
        if (cand_out) *cand_out += total;
        if (ix.stats && lane == 0) kd_stat(ix, 7, (unsigned long long)total);
        unsigned long long best[R];
#pragma unroll
        for (int r = 0; r < R; ++r) best[r] = KNN_NONE;
        unsigned long long cut = bound;  // keys above it cannot enter this level's K
        int staged = 0;
        for (int base = 0; base < total; base += 32) {
            const int t = base + lane;
            const bool active = t < total;
            const int idx = warp_candidate(incl, adj, active ? t : total - 1);
            unsigned long long key = KNN_NONE;
            if (active) key = knn_key(dist2_point(x, y, z, __ldg(ix.sorted + idx)), idx);
            const bool keep = active && key <= cut;
            const unsigned b = __ballot_sync(FULL, keep);
            if (keep) stage[staged + __popc(b & lanes_below)] = key;
            staged += __popc(b);
            if (staged >= 32) {
                __syncwarp();
                warp_merge_wide<R>(best, warp_sort_keys(stage[lane], lane), lane);
                __syncwarp();
                if (lane < staged - 32) stage[lane] = stage[32 + lane];
                staged -= 32;
                __syncwarp();
                cut = min(cut, wide_entry<R>(best, kr, kl));
            }
        }
        if (staged > 0) {
            __syncwarp();
            warp_merge_wide<R>(best, warp_sort_keys(lane < staged ? stage[lane] : KNN_NONE, lane), lane);
        }
        __syncwarp();  // `stage` is reused by the next level
        found = 0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            kept[r] = r * 32 + lane < K ? best[r] : KNN_NONE;
            found += __popc(__ballot_sync(FULL, kept[r] != KNN_NONE));
        }
        const unsigned long long kth = wide_entry<R>(kept, kr, kl);
        const bool exact = (found == K && __uint_as_float((unsigned)(kth >> 32)) <= r2) || level >= g.top;
        if (ix.stats && lane == 0 && level == 0) kd_stat(ix, exact ? 5 : 6);
        if (exact) break;
        if (found == K) {
            bound = kth;
            bound_d = __uint_as_float((unsigned)(kth >> 32));
        }
    }
    return found;
}

// warp_second_moments over a wide list: the same float32 arithmetic, neighbours 1 .. found - 1 summed sequentially in
// list order (entry j in lane j % 32, register j / 32) and divided by k.  Every lane returns the same six moments.
template <int R>
__device__ __forceinline__ void warp_second_moments_wide(const KdIndex& ix, const float4& c, int k, int found,
                                                         const unsigned long long (&kept)[R], int lane, float* cov) {
    float dx[R], dy[R], dz[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int j = r * 32 + lane;
        dx[r] = dy[r] = dz[r] = 0.f;
        if (j >= 1 && j < found) {
            const float4 q = __ldg(ix.sorted + (int)(unsigned)kept[r]);
            dx[r] = __fsub_rn(q.x, c.x);
            dy[r] = __fsub_rn(q.y, c.y);
            dz[r] = __fsub_rn(q.z, c.z);
        }
    }
    float sxx = 0.f, sxy = 0.f, sxz = 0.f, syy = 0.f, syz = 0.f, szz = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int n = min(found - r * 32, 32);
        for (int l = r == 0 ? 1 : 0; l < n; ++l) {
            const float bx = __shfl_sync(FULL, dx[r], l), by = __shfl_sync(FULL, dy[r], l), bz = __shfl_sync(FULL, dz[r], l);
            sxx = __fadd_rn(sxx, __fmul_rn(bx, bx));
            sxy = __fadd_rn(sxy, __fmul_rn(bx, by));
            sxz = __fadd_rn(sxz, __fmul_rn(bx, bz));
            syy = __fadd_rn(syy, __fmul_rn(by, by));
            syz = __fadd_rn(syz, __fmul_rn(by, bz));
            szz = __fadd_rn(szz, __fmul_rn(bz, bz));
        }
    }
    const float kk = (float)k;
    cov[0] = __fdiv_rn(sxx, kk); cov[1] = __fdiv_rn(sxy, kk); cov[2] = __fdiv_rn(sxz, kk);
    cov[3] = __fdiv_rn(syy, kk); cov[4] = __fdiv_rn(syz, kk); cov[5] = __fdiv_rn(szz, kk);
}

// Does k normal neighbours take the wide list (k + 1 > KD_KMAX)?  Its keys per lane for K = k + 1 entries: 2, 4 or 8.
__host__ __device__ constexpr bool kd_wide_k(int k) { return k + 1 > KD_KMAX; }
__host__ __device__ constexpr int kd_wide_regs(int K) { return K <= 64 ? 2 : (K <= 128 ? 4 : 8); }

// State words of the normal cache.
__device__ __forceinline__ uint32_t kd_normal_claimed(uint32_t gen) { return 2u * gen; }
__device__ __forceinline__ uint32_t kd_normal_valid(uint32_t gen) { return 2u * gen + 1u; }

}  // namespace pls
