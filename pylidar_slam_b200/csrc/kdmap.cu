// K5/K8 -- the kd local map on the GPU (replaces KdTreeLocalMap, slam/odometry/local_map.py:254-427).
//
// Per update (local_map.py:302-369): the whole map is moved by inverse(relative_pose) in float32, the new frame's
// points are appended, the oldest frame is dropped beyond local_map_size, the search index is rebuilt and the normal
// cache invalidated -- exactly the reference's life cycle, with the pykdtree build replaced by a cell-pyramid build:
//   kd_move_append_kernel   move + append + bounding box (block reduce, ordered-int atomics)
//   kd_grid_header_kernel   quantisation of the new bounding box
//   kd_cell_key_kernel      Morton id of every point's level-0 cell
//   radix sort (4 passes)   primitives.cu (stable: insertion order inside a cell)
//   kd_finalize_kernel      sorted float4 copy + the hashed cell tables of all levels
// Tables and cached normals carry the build's generation number: nothing is cleared between frames.
// Search (local_map.py:372-422): whole warps per query, see kdmap_device.cuh.  The kernels of one ICP iteration are
// listed below, under "one ICP iteration on the kd map".
#include <stdlib.h>

#include <vector>

#include "gn_device.cuh"
#include "internal.cuh"
#include "icp_device.cuh"
#include "kdmap_device.cuh"
#include "pose_device.cuh"
#include "projection_device.cuh"

namespace pls {

namespace {

inline int grid_for(int64_t n, int threads, int cap_blocks) {
    int64_t b = (n + threads - 1) / threads;
    return (int)(b < 1 ? 1 : (b > cap_blocks ? cap_blocks : b));
}

__global__ void kd_bbox_init_kernel(int* bbox) {
    if (threadIdx.x < 3) bbox[threadIdx.x] = 0x7fffffff;        // min (ordered int)
    else if (threadIdx.x < 6) bbox[threadIdx.x] = (int)0x80000000;  // max
}

struct Rigid {
    float R[9];
    float t[3];
};

// dst[k] = R src[k + skip] + t for k < kept;  dst[kept + j] = fresh[j] for j < num_new (from a
// device count);  bounding box of everything written.  upd: the device decided the update (kd_update_decision_kernel):
// skip, kept, num_new and the move come from it (all counts 0 when its gate is closed).
__global__ void __launch_bounds__(256)
kd_move_append_kernel(const float4* __restrict__ src, int64_t skip, int64_t kept, Rigid X,
                      const float4* __restrict__ fresh, const uint32_t* __restrict__ num_new_dev, int64_t num_new_cap,
                      float4* __restrict__ dst, int* __restrict__ bbox, const KdUpdateWords* __restrict__ upd) {
    int64_t num_new = num_new_dev ? (int64_t)*num_new_dev : num_new_cap;
    if (upd) {
        skip = upd->skip;
        kept = upd->kept;
        num_new = upd->num_new;
#pragma unroll
        for (int i = 0; i < 9; ++i) X.R[i] = upd->X[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) X.t[i] = upd->X[9 + i];
    }
    const int64_t total = kept + num_new;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
        float4 p;
        if (k < kept) {
            float4 s = src[k + skip];
            p.x = X.R[0] * s.x + X.R[1] * s.y + X.R[2] * s.z + X.t[0];
            p.y = X.R[3] * s.x + X.R[4] * s.y + X.R[5] * s.z + X.t[1];
            p.z = X.R[6] * s.x + X.R[7] * s.y + X.R[8] * s.z + X.t[2];
            p.w = 0.f;
        } else {
            p = fresh[k - kept];
        }
        dst[k] = p;
        mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
        mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
    }
    __shared__ float smn[8][3], smx[8][3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { smn[warp][a] = mn[a]; smx[warp][a] = mx[a]; }
    }
    __syncthreads();
    if (threadIdx.x < 3) {  // one atomic pair per axis per block
        const int a = threadIdx.x;
        float lo = smn[0][a], hi = smx[0][a];
        for (int w = 1; w < 8; ++w) { lo = fminf(lo, smn[w][a]); hi = fmaxf(hi, smx[w][a]); }
        if (lo != FLT_MAX) atomicMin(&bbox[a], float_to_ordered(lo));
        if (hi != -FLT_MAX) atomicMax(&bbox[3 + a], float_to_ordered(hi));
    }
}

// [n,3] raw points -> float4, dropping rows containing NaN (utils.py:169-184); flags only.
// T = double: the reference rounds a float64 cloud to float32 first (`_tgt_pc = pc_data.to(torch.float32)`,
// icp_odometry.py:352) and removes NaN rows afterwards; NaN survives the rounding, so the order does not matter.
template <typename T>
__global__ void kd_valid_rows_kernel(const T* __restrict__ pts, int64_t n, uint8_t* __restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        T x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        flags[i] = (x == x && y == y && z == z) ? 1 : 0;
    }
}
template <typename T>
__global__ void kd_pack_rows_kernel(const T* __restrict__ pts, int64_t n, const uint8_t* __restrict__ flags,
                                    const uint32_t* __restrict__ pos, float4* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (flags[i]) out[pos[i]] = make_float4((float)pts[3 * i], (float)pts[3 * i + 1], (float)pts[3 * i + 2], 0.f);
}
// pls_register_scans: block s packs scans[s] into its own slice of the query buffer, with the rows and the count
// pack_valid_rows gives for that scan alone: the rows without a NaN coordinate (kd_valid_rows_kernel's test), in input
// order (the positions of the exclusive scan).  The block walks its scan in tiles of KD_PACK_ROWS rows per thread.
constexpr int KD_PACK_THREADS = 1024, KD_PACK_ROWS = 4;
__global__ void __launch_bounds__(KD_PACK_THREADS) kd_pack_scans_kernel(const KdScanRows* __restrict__ scans) {
    __shared__ uint32_t s_warp[KD_PACK_ROWS][32];  // per sub-tile: valid rows of the warps before, then of the sub-tile
    __shared__ uint32_t s_sub[KD_PACK_ROWS];
    const KdScanRows sc = scans[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t below = (1u << lane) - 1u;
    uint32_t base = 0;
    for (int64_t t0 = 0; t0 < sc.n; t0 += (int64_t)KD_PACK_THREADS * KD_PACK_ROWS) {
        float4 v[KD_PACK_ROWS];
        bool ok[KD_PACK_ROWS];
        uint32_t rank[KD_PACK_ROWS];
#pragma unroll
        for (int j = 0; j < KD_PACK_ROWS; ++j) {
            const int64_t i = t0 + (int64_t)j * KD_PACK_THREADS + threadIdx.x;
            ok[j] = false;
            if (i < sc.n) {
                const float x = sc.rows[3 * i], y = sc.rows[3 * i + 1], z = sc.rows[3 * i + 2];
                ok[j] = x == x && y == y && z == z;
                v[j] = make_float4(x, y, z, 0.f);
            }
            const unsigned b = __ballot_sync(0xffffffffu, ok[j]);
            rank[j] = __popc(b & below);
            if (lane == 0) s_warp[j][warp] = __popc(b);
        }
        __syncthreads();
        if (warp < KD_PACK_ROWS) {  // warp j: exclusive prefix over the 32 warps of sub-tile j
            const uint32_t c = s_warp[warp][lane];
            uint32_t inc = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            s_warp[warp][lane] = inc - c;
            if (lane == 31) s_sub[warp] = inc;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < KD_PACK_ROWS; ++j) {
            if (ok[j]) sc.out[base + s_warp[j][warp] + rank[j]] = v[j];
            base += s_sub[j];
        }
        __syncthreads();  // s_warp and s_sub are rewritten by the next tile
    }
    if (threadIdx.x == 0) *sc.count = base;
}

// pls_kdmap_set_points: counts the rows with a NaN or an infinite coordinate once rounded to float32.
template <typename T>
__global__ void kd_nonfinite_rows_kernel(const T* __restrict__ pts, int64_t n, uint32_t* __restrict__ count) {
    uint32_t bad = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        bad += !(isfinite((float)pts[3 * i]) && isfinite((float)pts[3 * i + 1]) && isfinite((float)pts[3 * i + 2]));
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(count, bad);
}
// vertex map [3,H,W] -> pixels with |p| > min_norm and no NaN
__global__ void kd_valid_pixels_kernel(const float* __restrict__ vmap, int64_t hw, float min_norm,
                                       uint8_t* __restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x) {
        float x = vmap[i], y = vmap[hw + i], z = vmap[2 * hw + i];
        flags[i] = (sqrtf(x * x + y * y + z * z) > min_norm) ? 1 : 0;  // NaN compares false
    }
}
__global__ void kd_pack_pixels_kernel(const float* __restrict__ vmap, int64_t hw, const uint8_t* __restrict__ flags,
                                      const uint32_t* __restrict__ pos, float4* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x)
        if (flags[i]) out[pos[i]] = make_float4(vmap[i], vmap[hw + i], vmap[2 * hw + i], 0.f);
}

// Quantisation of the map.  A level-0 cell is always 2^KD_MIN_B0 = 8 quantisation units, so its id (10 bits per axis,
// Morton-interleaved) fits 30 bits and the sort needs four 8-bit passes whatever the extent; the unit is chosen so
// that the cell side equals the target -- or, for maps wider than 1024 cells, so that the 13-bit range just covers the
// extent (coarser cells).  The coarsest level (top = 10) is a single cell.
// gate (nullable): a device-decided update whose gate is closed leaves the header (which the ICP reads) as it is.
__global__ void kd_grid_header_kernel(int* __restrict__ bbox, KdGridHeader* __restrict__ hdr, float cell_target,
                                      const uint32_t* __restrict__ gate) {
    if (threadIdx.x != 0 || (gate && !*gate)) return;
    const float mnx = ordered_to_float(bbox[0]), mny = ordered_to_float(bbox[1]), mnz = ordered_to_float(bbox[2]);
    const float ex = ordered_to_float(bbox[3]) - mnx, ey = ordered_to_float(bbox[4]) - mny,
                ez = ordered_to_float(bbox[5]) - mnz;
    const float ext = fmaxf(fmaxf(ex, ey), fmaxf(ez, 1e-6f));
    const int b0 = KD_MIN_B0;
    const float scale = fminf((float)(1 << b0) / cell_target, (float)KD_COORD_MAX / ext);
    hdr->mn[0] = mnx; hdr->mn[1] = mny; hdr->mn[2] = mnz;
    hdr->scale = scale;
    hdr->b0 = b0;
    hdr->cell0 = (float)(1 << b0) / scale;
    hdr->top = KD_COORD_BITS - b0;
    for (int l = 0; l < KD_MAX_LEVELS; ++l) hdr->overflow[l] = 0;
    // leave the box empty for the next update (saves that update an init launch)
    bbox[0] = bbox[1] = bbox[2] = 0x7fffffff;
    bbox[3] = bbox[4] = bbox[5] = (int)0x80000000;
}

// Sort key of a map point = the Morton id of its level-0 cell (<= 30 bits); the order inside a cell is the
// insertion order (stable sort), nothing finer is needed: every level's cell is a prefix of this id.
// n_dev (nullable): the point count on the device, n a bound of it.
__global__ void kd_cell_key_kernel(const float4* __restrict__ pts, int64_t n, const KdGridHeader* __restrict__ hdr,
                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, const uint32_t* __restrict__ n_dev) {
    pls_grid_dependency_wait();
    if (n_dev) n = *n_dev;
    const float mnx = hdr->mn[0], mny = hdr->mn[1], mnz = hdr->mn[2];
    const float scale = hdr->scale;
    const int b0 = hdr->b0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        const uint32_t qx = (uint32_t)fminf(fmaxf((p.x - mnx) * scale, 0.f), (float)KD_COORD_MAX);
        const uint32_t qy = (uint32_t)fminf(fmaxf((p.y - mny) * scale, 0.f), (float)KD_COORD_MAX);
        const uint32_t qz = (uint32_t)fminf(fmaxf((p.z - mnz) * scale, 0.f), (float)KD_COORD_MAX);
        keys[i] = (uint64_t)kd_cell_id(qx >> b0, qy >> b0, qz >> b0);
        vals[i] = (uint32_t)i;
    }
}

struct CellTables {
    uint4* table[KD_MAX_LEVELS];
    uint32_t mask[KD_MAX_LEVELS];
};

// Finds or claims the slot of cell `id` in this generation's table.  Slots of older generations are free.
__device__ __forceinline__ int cell_claim(uint4* table, uint32_t mask, uint32_t id, uint32_t gen) {
    const unsigned long long want = (unsigned long long)id | ((unsigned long long)gen << 32);
    uint32_t h = kd_hash(id) & mask;
    for (int probe = 0; probe < 64; ++probe) {
        unsigned long long* word = reinterpret_cast<unsigned long long*>(&table[h]);
        unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(word);
        while (true) {
            if (old == want) return (int)h;
            if ((uint32_t)(old >> 32) == gen) break;  // another cell of this generation lives here
            const unsigned long long prev = atomicCAS(word, old, want);
            if (prev == old) return (int)h;
            old = prev;
        }
        h = (h + 1) & mask;
    }
    return -1;
}

// One pass over the sorted order finishes the index: the Morton-ordered float4 copy of the points and the cell
// tables of ALL levels -- element i is the head of a level-l cell run if its id prefix differs from element i-1's,
// i.e. for every level up to (highest differing bit) / 3, and the tail likewise against element i+1; heads store
// `first`, tails store `last` into the slot they find-or-claim.
__global__ void __launch_bounds__(256)
kd_finalize_kernel(const float4* __restrict__ pts, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ order,
                   int64_t n, CellTables T, KdGridHeader* hdr, uint32_t gen, float4* __restrict__ sorted,
                   const uint32_t* __restrict__ n_dev) {
    pls_grid_dependency_wait();
    if (n_dev) n = *n_dev;
    const int top = hdr->top;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t src = order[i];
        float4 p = pts[src];
        p.w = __uint_as_float(src);
        sorted[i] = p;
        const uint32_t k = (uint32_t)keys[i];
        // number of levels (from 0) at which this element starts / ends a run
        int nh = top + 1, nt = top + 1;
        if (i > 0) {
            const uint32_t d = k ^ (uint32_t)keys[i - 1];
            nh = d ? min((31 - __clz((int)d)) / 3 + 1, top + 1) : 0;
        }
        if (i + 1 < n) {
            const uint32_t d = k ^ (uint32_t)keys[i + 1];
            nt = d ? min((31 - __clz((int)d)) / 3 + 1, top + 1) : 0;
        }
        const int nl = max(nh, nt);
        for (int l = 0; l < nl; ++l) {
            const int slot = cell_claim(T.table[l], T.mask[l], k >> (3 * l), gen);
            if (slot < 0) {
                hdr->overflow[l] = 1;
            } else {
                if (l < nh) T.table[l][slot].z = (uint32_t)i;
                if (l < nt) T.table[l][slot].w = (uint32_t)i;
            }
        }
    }
}

__global__ void kd_export_kernel(const float4* __restrict__ pts, int64_t n, float* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float4 p = pts[i];
        out[3 * i] = p.x; out[3 * i + 1] = p.y; out[3 * i + 2] = p.z;
    }
}

// ---- one ICP iteration on the kd map (icp_odometry.py:275-284 + alignment.py:91-127 at x0 = 0) -----------------------
//   p = T p0; q = NN(p); n = normal(q); r = n.(p - q); J = [n, p x n]; w; reduce
// A frame's first iteration is three launches: kd_nn_warp_kernel, kd_normals_warp_kernel and kd_residual_kernel, which
// also runs the solve in its last block.  Every later iteration is one launch, kd_icp_refine_kernel, or, on maps of
// KD_COLD_MAP_POINTS or more and for k > 31 normal neighbours (kd_later_four_launch), four: kd_nn_verify_kernel and the
// same three on the queries it could not prove.
// KD_THREADS is the block size of the kernels that own a thread per query, and the number of query slots of a
// kd_icp_refine_kernel block: both striding and block partials follow from it.
constexpr int KD_THREADS = 256;
constexpr int KD_WARPS = KD_THREADS / 32;

// counters of the search kernels (u64, behind the u32 scalar slots): candidates tested by the 1-NN searches, by the
// k-NN searches, normals computed -- the inputs of SURVEY 8d's algorithmic-bytes formulas
enum { KDC_NN_CAND = 0, KDC_KNN_CAND = 1, KDC_NORMALS = 2 };
// per-iteration work-list counters (u32 words at SC_KD_LISTS), one pair per list, indexed by the iteration's parity:
// the first kernel of iteration `it` zeroes the words of parity (it + 1) & 1 -- consumed by the previous iteration,
// filled by the next -- so no list is ever reset by a separate launch
enum { KDL_PENDING = 0, KDL_HARD_NN = 2, KDL_WORDS = 4 };

#ifdef PLS_KD_SPLIT
// Stamp records of the residual-and-solve phase (tools/kd_residual_split.py): one per block of the launch of ICP
// iteration 0..KD_SPLIT_ITERS-1, and one for a launch that found ICP converged (a no-op).  Stamps: 0 start, 1 start of
// the residual phase, 2 / 3 the block's last thread done with its loads / its accumulation, 4 block partial stored,
// 5 ticket taken; last block only: 6 rows summed, 7 solve done, 8 pose written.
constexpr int KD_SPLIT_ITERS = 8;
constexpr int KD_SPLIT_BLOCKS = 8 * kNumSMs;
constexpr int KD_SPLIT_WORDS = (KD_SPLIT_ITERS + 1) * KD_SPLIT_BLOCKS * 2 * KD_SPLIT_STAMPS;
__device__ unsigned long long g_kd_split[KD_SPLIT_WORDS];
__device__ unsigned long long g_kd_split_normals_end;  // the last warp of kd_normals_warp_kernel to finish

__device__ __forceinline__ unsigned long long* kd_split_record(const FrameResult* fr) {
    const int slot = fr->done ? KD_SPLIT_ITERS : fr->iters;
    if ((!fr->done && slot >= KD_SPLIT_ITERS) || blockIdx.x >= KD_SPLIT_BLOCKS) return nullptr;
    return g_kd_split + ((size_t)slot * KD_SPLIT_BLOCKS + blockIdx.x) * 2 * KD_SPLIT_STAMPS;
}
#define KD_SPLIT_BEGIN()                             \
    unsigned long long* split = kd_split_record(fr); \
    __shared__ unsigned long long s_split[2];        \
    if (threadIdx.x == 0) {                          \
        PLS_SPLIT(0);                                \
        s_split[0] = s_split[1] = 0;                 \
        unsigned sm;                                 \
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm)); \
        if (split) split[11] = sm + 1;               \
    }
#define KD_SPLIT_MAX(k, dep) atomicMax(&s_split[k], split_now(dep))
#define KD_SPLIT_BLOCK_MAX()         \
    if (threadIdx.x == 0 && split) { \
        split[2] = s_split[0];       \
        split[3] = s_split[1];       \
    }
// the record and the block's shared maxima, into the device helpers that stamp
#define KD_SPLIT_ARG , unsigned long long* split, unsigned long long* s_split
#define KD_SPLIT_PASS , split, s_split
#else
#define KD_SPLIT_BEGIN()
#define KD_SPLIT_MAX(k, dep) \
    do {                     \
    } while (0)
#define KD_SPLIT_BLOCK_MAX()
#define KD_SPLIT_ARG
#define KD_SPLIT_PASS
#endif

// The block count of a residual or refine launch.  bound_dev null: the launched grid.  Else the host launched for the
// bound `bound` of a query count the device knows, *bound_dev: the count is that of the grid the host would launch for
// min(bound, *bound_dev) queries (grid_for), so that the striding, the block partials and the solve ticket -- and with
// them the bits -- are those of a launch sized on the host; blocks past it return at once.
__device__ __forceinline__ unsigned kd_logical_blocks(int64_t bound, const uint32_t* __restrict__ bound_dev) {
    if (!bound_dev) return gridDim.x;
    const int64_t n = min(bound, (int64_t)*bound_dev);
    const int64_t b = (n + KD_THREADS - 1) / KD_THREADS;
    return (unsigned)(b < 1 ? 1 : (b > 8 * kNumSMs ? 8 * kNumSMs : b));
}

// Appends this block's entries (collected in shared memory by any of its threads) to a global list: one atomic per block.
__device__ __forceinline__ void block_flush_list(const int* s_list, int n, int* __restrict__ list, uint32_t* count, int* s_base) {
    if (n == 0) return;  // block-uniform
    if (threadIdx.x == 0) *s_base = (int)atomicAdd(count, (uint32_t)n);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) list[*s_base + i] = s_list[i];
}

// Claims the normal of map point `pos` for computation if it is neither cached nor already claimed.
__device__ __forceinline__ bool claim_normal(const KdIndex& ix, int pos) {
    const uint32_t claimed = kd_normal_claimed(ix.gen), valid = kd_normal_valid(ix.gen);
    uint32_t* w = reinterpret_cast<uint32_t*>(&ix.normals[pos].w);
    const uint32_t cur = __ldcg(w);
    return cur != valid && cur != claimed && atomicCAS(w, cur, claimed) == cur;
}

// 1-NN of ICP iterations after a frame's first: VERIFY instead of searching.  The full search stored in `state` where
// the query stood (xyz, its transformed position) and in .w a lower bound of the squared distance to every map point
// other than its match.  If the query, now at p, has moved by eps since then and its match `pos` is now at distance d,
// every other point is still at least (bound - eps) away, so d + eps < bound proves the match unchanged -- one point
// load and a dozen flops per query.  False when there is no match (pos < 0).
// GATE: no match is a gated search's outlier, whose state holds a lower bound of the squared distance to EVERY map
// point (warp_nearest<true>).  It stays an outlier, with no search, while (bound - eps) > max_distance is proven in
// float32 with match_proven's own slack; otherwise it is searched again.  A proven match is kept whatever its distance:
// the residual pass tests it against the gate in every iteration.
template <bool GATE = false>
__device__ __forceinline__ bool match_proven(const KdIndex& ix, const float* p, int pos, const float4& state,
                                             float dmax = 0.f) {
    if constexpr (GATE)
        if (pos < 0) return (sqrtf(dist2_point(p[0], p[1], p[2], state)) + dmax) * 1.00001f + 1e-6f < sqrtf(state.w);
    if (pos < 0) return false;
    const float4 s = state;
    const float d = sqrtf(dist2_point(p[0], p[1], p[2], __ldg(ix.sorted + pos)));
    const float eps = sqrtf(dist2_point(p[0], p[1], p[2], s));
    return (d + eps) * 1.00001f + 1e-6f < sqrtf(s.w);
}

// Second moments of map point c's k nearest OTHER map points, from its exact (k+1)-NN by the whole warp.  R = 1: k <= 31
// (warp_knn); else the wide list of R keys per lane, k + 1 <= 32 R (warp_knn_wide).
template <int R = 1>
__device__ __forceinline__ void warp_normal_moments(const KdIndex& ix, const KdGridLocal& g, const float4& c, int k, int lane,
                                                    int* cand, unsigned long long* stage, float* cov) {
    if constexpr (R == 1) {
        int ni;
        const int found = warp_knn(ix, g, c.x, c.y, c.z, k + 1, lane, ni, cand, stage);
        warp_second_moments(ix, c, k, found, ni, lane, cov);
    } else {
        unsigned long long kept[R];
        const int found = warp_knn_wide<R>(ix, g, c.x, c.y, c.z, k + 1, lane, kept, cand, stage);
        warp_second_moments_wide<R>(ix, c, k, found, kept, lane, cov);
    }
}

// The normal of map point `pos` from its second moments, stored with `valid`, the state word kd_normal_valid(ix.gen).
__device__ __forceinline__ void store_normal(const KdIndex& ix, int pos, const float* cov, uint32_t valid) {
    float nn[3];
    smallest_eigenvector(cov, nn);
    __stcg(ix.normals + pos, make_float4(nn[0], nn[1], nn[2], __uint_as_float(valid)));
}

// A matched query's (p = T p0, match `pos`) share of the normal equations: residual, Jacobian, robust weight, fp64
// accumulation.
__device__ __forceinline__ void accumulate_match(double* acc, const KdIndex& ix, const float* p, int pos, int scheme,
                                                 float sigma KD_SPLIT_ARG) {
    const float4 qq = __ldg(ix.sorted + pos);
    const float4 nv = __ldcg(ix.normals + pos);
    float q[3] = {qq.x, qq.y, qq.z};
    float nn[3] = {nv.x, nv.y, nv.z};
    float J[6];
    const float r = p2plane_residual_jacobian_identity(p, q, nn, J);
    KD_SPLIT_MAX(0, r);
    const float w = ls_weight<float>(scheme, sigma, r, p, q);
    accumulate_normal_equations<float>(acc, J, w, r * w, r);
}

// The end of a residual phase, called by every thread of a THREADS-thread block whose first KD_WARPS warps hold
// accumulators: the block partial row `block` of W accumulators, then (NACC-wide rows, fuse_threshold >= 0) the
// fixed-order sum of the `grid` rows and the solve in the last block to arrive.  DEGEN: that solve is
// icp_solve_and_update<true> with dg.
template <int THREADS, int W = NACC, bool DEGEN = false>
__device__ __forceinline__ void block_partial_and_finish(double* acc, FrameResult* fr, double* __restrict__ partials,
                                                         float fuse_threshold, unsigned block, unsigned grid KD_SPLIT_ARG,
                                                         IcpDegen dg = IcpDegen{}) {
    KD_SPLIT_MAX(1, acc[0] + acc[29]);
    // The shuffle tree must start on a converged warp.  The grid's last block holds a warp whose lanes left the query
    // loop at different iterations; without this it took the divergent-warp path of the 30 x 5 shuffles, 35 us on H100
    // (profiles/h100_kd_residual_split_before.log) while every other block took 1.2 us -- and the solve waits for it.
    __syncwarp();
    block_reduce_store<THREADS, KD_WARPS, W>(acc, partials + (size_t)block * W);
    KD_SPLIT_BLOCK_MAX()
    if constexpr (W == NACC)
        if (fuse_threshold >= 0.f)
            icp_finish_in_last_block<THREADS, DEGEN>(fr, partials, (int)grid, fuse_threshold PLS_SPLIT_PASS, dg);
}

// Iterations after a frame's first on maps of KD_COLD_MAP_POINTS or more: a thread per query keeps its previous match
// if match_proven; the few others are queued for kd_nn_warp_kernel.  GATE: match_proven<true> with gate.dmax.
template <bool GATE = false>
__device__ __forceinline__ void kd_nn_verify_body(const KdIndex& ix, const float4* __restrict__ queries,
                                                  const uint32_t* __restrict__ nq_dev, int64_t q_begin, int64_t q_stride,
                                                  const float* __restrict__ T, const int* __restrict__ done,
                                                  const int* __restrict__ match, const float4* __restrict__ nn_state,
                                                  int* __restrict__ hard, uint32_t* lists, int parity, unsigned block,
                                                  float dmax = 0.f) {
    if (done && *done) return;
    __shared__ float sT[12];
    __shared__ int s_hard[KD_THREADS];
    __shared__ int s_nh, s_base;
    if (threadIdx.x < 12) sT[threadIdx.x] = T[threadIdx.x];
    if (threadIdx.x == 0) {
        s_nh = 0;
        if (block == 0)
            for (int l = 0; l < KDL_WORDS; l += 2) lists[l + (parity ^ 1)] = 0;
    }
    __syncthreads();
    const int64_t nq = (int64_t)*nq_dev;
    const int64_t qi = q_begin + ((int64_t)block * KD_THREADS + threadIdx.x) * q_stride;
    if (qi < nq) {
        float p[3];
        transform_point(sT, queries[qi], p);
        if (!match_proven<GATE>(ix, p, match[qi], nn_state[qi], dmax)) s_hard[atomicAdd(&s_nh, 1)] = (int)qi;
    }
    __syncthreads();
    block_flush_list(s_hard, s_nh, hard, lists + KDL_HARD_NN + parity, &s_base);
}

__global__ void __launch_bounds__(KD_THREADS)
kd_nn_verify_kernel(KdIndex ix, const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev, int64_t q_begin,
                    int64_t q_stride, const float* __restrict__ T, const int* __restrict__ done, const int* __restrict__ match,
                    const float4* __restrict__ nn_state, int* __restrict__ hard, uint32_t* lists, int parity) {
    kd_nn_verify_body(ix, queries, nq_dev, q_begin, q_stride, T, done, match, nn_state, hard, lists, parity, blockIdx.x);
}

// Each kernel of an ICP iteration below is one __device__ body, called by two entry points: the kernel of one sequence,
// which passes blockIdx.x / gridDim.x and its arguments, and the *_batch_kernel of pls_process_frames, whose
// blockIdx.y picks a sequence's descriptor and which passes that sequence's own block count.  A body reads no
// blockIdx.x or gridDim.x itself, so a sequence's striding, block partials and solve ticket are those of its single path.

// 1-NN, full search: a warp per query over the cell pyramid (warp_nearest).  hard == nullptr: every query of this
// rank's shard (a frame's first iteration); else the queued ones, seeded with their previous match.  The first warp to
// match a map point whose normal is not cached claims it (CAS on the state word) and queues it; claims are made by all
// lanes at once after 32 queries.  Each query's position and runner-up bound are kept for the later iterations' checks.
// Which warp searches which query does not change its result, so any block count gives the same bits.
// GATE: warp_nearest<true>; an outlier's match is -1, so it claims no normal.
template <bool GATE = false>
__device__ __forceinline__ void kd_nn_warp_body(const KdIndex& ix, const float4* __restrict__ queries,
                                                const uint32_t* __restrict__ nq_dev, int64_t q_begin, int64_t q_stride,
                                                const int* __restrict__ hard, uint32_t* lists, int parity,
                                                const float* __restrict__ T, const int* __restrict__ done,
                                                int* __restrict__ match, float4* __restrict__ nn_state, int want_normals,
                                                int* __restrict__ pending, unsigned long long* __restrict__ counters,
                                                unsigned block, unsigned grid, KdGate gate = KdGate{}) {
    if (done && *done) return;
    int n;
    if (hard) {
        n = (int)lists[KDL_HARD_NN + parity];
    } else {
        const int64_t nq = (int64_t)*nq_dev;
        n = nq > q_begin ? (int)((nq - q_begin + q_stride - 1) / q_stride) : 0;
        if (block == 0 && threadIdx.x == 0)  // first kernel of the iteration: recycle the other parity's lists
            for (int l = 0; l < KDL_WORDS; l += 2) lists[l + (parity ^ 1)] = 0;
    }
    const int lane = threadIdx.x & 31;
    const int warp_global = block * KD_WARPS + (threadIdx.x >> 5);
    const int total_warps = grid * KD_WARPS;
    if (warp_global >= n) return;
    float t[12];
#pragma unroll
    for (int a = 0; a < 12; ++a) t[a] = T[a];
    const KdGridLocal g = kd_load_grid(ix);
    uint32_t* pending_count = lists + KDL_PENDING + parity;
    int my_pos = -1, held = 0, cand = 0;
    auto flush_claims = [&]() {
        const bool mine = want_normals && my_pos >= 0 && claim_normal(ix, my_pos);
        const unsigned m = __ballot_sync(FULL, mine);
        if (m) {
            int base = 0;
            if (lane == 0) base = (int)atomicAdd(pending_count, (uint32_t)__popc(m));
            base = __shfl_sync(FULL, base, 0);
            if (mine) pending[base + __popc(m & ((1u << lane) - 1u))] = my_pos;
        }
        my_pos = -1;
        held = 0;
    };
    // the next query's data is fetched while this one is searched
    int s = warp_global;
    int64_t qi = hard ? (int64_t)hard[s] : q_begin + (int64_t)s * q_stride;
    float4 p0 = queries[qi];
    int hint = hard ? match[qi] : -1;
    while (true) {
        const int sn = s + total_warps;
        int64_t qn = qi;
        float4 pn = p0;
        int hn = -1;
        if (sn < n) {
            qn = hard ? (int64_t)hard[sn] : q_begin + (int64_t)sn * q_stride;
            pn = queries[qn];
            if (hard) hn = match[qn];
        }
        float p[3];
        transform_point(t, p0, p);
        float second;
        const int pos = warp_nearest<GATE>(ix, g, p[0], p[1], p[2], hint, lane, &cand, &second, gate);
        if (lane == 0) {
            match[qi] = pos;
            if (nn_state) nn_state[qi] = make_float4(p[0], p[1], p[2], second);
        }
        if (lane == held) my_pos = pos;
        if (++held == 32) flush_claims();
        if (sn >= n) break;
        s = sn;
        qi = qn;
        p0 = pn;
        hint = hn;
    }
    flush_claims();
    if (counters && lane == 0 && cand) atomicAdd(counters + KDC_NN_CAND, (unsigned long long)cand);
}

__global__ void __launch_bounds__(KD_THREADS)
kd_nn_warp_kernel(KdIndex ix, const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev, int64_t q_begin,
                  int64_t q_stride, const int* __restrict__ hard, uint32_t* lists, int parity, const float* __restrict__ T,
                  const int* __restrict__ done, int* __restrict__ match, float4* __restrict__ nn_state, int want_normals,
                  int* __restrict__ pending, unsigned long long* __restrict__ counters) {
    pls_grid_dependency_wait();
    kd_nn_warp_body(ix, queries, nq_dev, q_begin, q_stride, hard, lists, parity, T, done, match, nn_state, want_normals,
                    pending, counters, blockIdx.x, gridDim.x);
}

// Normals: a warp per queued map point, exact (k+1)-NN over the cell pyramid (warp_knn, or warp_knn_wide<R> for R > 1),
// second moments; the eigen-solves are deferred and run lane-parallel (each lane one point) so that no warp idles behind
// a serial solve.
template <int R = 1>
__device__ __forceinline__ void kd_normals_warp_body(const KdIndex& ix, int k_normals, const int* __restrict__ worklist,
                                                     const uint32_t* __restrict__ wl_count, const int* __restrict__ done,
                                                     unsigned long long* __restrict__ counters, unsigned block, unsigned grid) {
    if (done && *done) return;
    __shared__ unsigned long long s_stage[KD_WARPS][KNN_STAGE];
    const int n = (int)*wl_count;
    const int lane = threadIdx.x & 31;
    const int warp_global = block * KD_WARPS + (threadIdx.x >> 5);
    const int total_warps = grid * KD_WARPS;
    if (warp_global >= n) return;
    unsigned long long* stage = s_stage[threadIdx.x >> 5];
    const KdGridLocal g = kd_load_grid(ix);
    const uint32_t valid = kd_normal_valid(ix.gen);
    float mycov[6];
    int mypos = -1, held = 0, cand = 0, done_here = 0;
    int e = warp_global;
    int pos = worklist[e];
    float4 c = __ldg(ix.sorted + pos);
    while (true) {
        // the next point is fetched while this one is searched
        const int en = e + total_warps;
        int posn = 0;
        float4 cn = c;
        if (en < n) {
            posn = worklist[en];
            cn = __ldg(ix.sorted + posn);
        }
        float cov[6];
        warp_normal_moments<R>(ix, g, c, k_normals, lane, &cand, stage, cov);
        if (lane == held) {
#pragma unroll
            for (int a = 0; a < 6; ++a) mycov[a] = cov[a];
            mypos = pos;
        }
        ++done_here;
        if (++held == 32) {  // 32 moments collected: every lane solves its own
            store_normal(ix, mypos, mycov, valid);
            held = 0;
            mypos = -1;
        }
        if (en >= n) break;
        e = en;
        pos = posn;
        c = cn;
    }
    if (mypos >= 0) store_normal(ix, mypos, mycov, valid);
    if (counters && lane == 0) {
        atomicAdd(counters + KDC_KNN_CAND, (unsigned long long)cand);
        atomicAdd(counters + KDC_NORMALS, (unsigned long long)done_here);
    }
#ifdef PLS_KD_SPLIT
    if (lane == 0) atomicMax(&g_kd_split_normals_end, split_now((double)done_here));
#endif
}

__global__ void __launch_bounds__(KD_THREADS)
kd_normals_warp_kernel(KdIndex ix, int k_normals, const int* __restrict__ worklist, const uint32_t* __restrict__ wl_count,
                       const int* __restrict__ done, unsigned long long* __restrict__ counters) {
    pls_grid_dependency_wait();
    kd_normals_warp_body(ix, k_normals, worklist, wl_count, done, counters, blockIdx.x, gridDim.x);
}

// The same for a wide k: k + 1 in 33 ... 32 R.  Launched with KD_THREADS threads.  Left to its default, ptxas gives this
// kernel 80 registers and spills the list across the division slow paths' calls; 128 (two blocks per SM) it fits in.
template <int R>
__global__ void __maxnreg__(128)
kd_normals_wide_kernel(KdIndex ix, int k_normals, const int* __restrict__ worklist, const uint32_t* __restrict__ wl_count,
                       const int* __restrict__ done, unsigned long long* __restrict__ counters) {
    pls_grid_dependency_wait();
    kd_normals_warp_body<R>(ix, k_normals, worklist, wl_count, done, counters, blockIdx.x, gridDim.x);
}

// A thread per query: accumulate_match -> block partials; the last block sums them in fixed order and runs the solve,
// stop test and pose update.
// EVAL (pls_kdmap_evaluate_poses, launched with fuse_threshold < 0: no solve): only the matches with
// match_d2_f64 <= max_d2 are accumulated, their d^2 summed in acc[NACC], and every query is counted in acc[NACC + 1];
// the block partial rows are PLS_EVAL_STATS wide.  The ICP instantiation (EVAL = false) is the same code as before.
// GATE without EVAL (a gated registration): the same distance test on NACC-wide rows with the fused solve, so the
// count accumulator (29) counts the inliers.
// DEGEN (pls_register_scans_degeneracy): the fused solve is the eigenvalue-thresholded one of block_partial_and_finish.
// kd_residual_body's pose.  Owned by this function rather than by the template, so that the module's shared variables
// keep the order they had before kd_residual_body took EVAL: the ICP kernels keep their shared-memory layout and SASS
// (profiles/sass_evaluate_poses_census.log).
__device__ __forceinline__ float* kd_residual_pose() {
    __shared__ float sT[12];
    return sT;
}

template <bool EVAL = false, bool GATE = EVAL, bool DEGEN = false>
__device__ __forceinline__ void kd_residual_body(const KdIndex& ix, const float4* __restrict__ queries,
                                                 const uint32_t* __restrict__ nq_dev, int64_t q_begin, int64_t q_stride,
                                                 FrameResult* fr, int scheme, float sigma, const int* __restrict__ match,
                                                 double* __restrict__ partials, float fuse_threshold, unsigned block,
                                                 unsigned grid, double max_d2 KD_SPLIT_ARG, IcpDegen dg = IcpDegen{}) {
    static_assert(PLS_EVAL_STATS == NACC + 2, "evaluation rows: the 30 accumulators, sum d^2, |P|");
    constexpr int W = EVAL ? PLS_EVAL_STATS : NACC;
    if (fr->done) return;
    float* sT = kd_residual_pose();
    if (threadIdx.x < 12) sT[threadIdx.x] = fr->T[threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) PLS_SPLIT(1);
    const int64_t nq = (int64_t)*nq_dev;
    double acc[W];
#pragma unroll
    for (int a = 0; a < W; ++a) acc[a] = 0.0;
    for (int64_t s = (int64_t)block * blockDim.x + threadIdx.x;; s += (int64_t)grid * blockDim.x) {
        const int64_t qi = q_begin + s * q_stride;
        if (qi >= nq) break;
        float p[3];
        transform_point(sT, queries[qi], p);
        const int pos = match[qi];
        if constexpr (EVAL) acc[NACC + 1] += 1.0;
        if (pos < 0) continue;
        if constexpr (GATE) {
            const double d2 = match_d2_f64(p, __ldg(ix.sorted + pos));
            if (!(d2 <= max_d2)) continue;
            if constexpr (EVAL) acc[NACC] += d2;
        }
        accumulate_match(acc, ix, p, pos, scheme, sigma KD_SPLIT_PASS);
    }
    block_partial_and_finish<KD_THREADS, W, DEGEN>(acc, fr, partials, fuse_threshold, block, grid KD_SPLIT_PASS, dg);
}

__global__ void __launch_bounds__(KD_THREADS)
kd_residual_kernel(KdIndex ix, const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev, int64_t q_begin,
                   int64_t q_stride, FrameResult* fr, int scheme, float sigma,
                   const int* __restrict__ match, double* __restrict__ partials, float fuse_threshold, int64_t bound,
                   const uint32_t* __restrict__ bound_dev) {
    pls_grid_dependency_wait();
    const unsigned grid = kd_logical_blocks(bound, bound_dev);
    if (blockIdx.x >= grid) return;
    KD_SPLIT_BEGIN()
    kd_residual_body(ix, queries, nq_dev, q_begin, q_stride, fr, scheme, sigma, match, partials, fuse_threshold, blockIdx.x,
                     grid, 0.0 KD_SPLIT_PASS);
}

// ICP iterations after a frame's first, in ONE launch.  Each block takes the queries kd_residual_kernel would give it
// (same grid, same striding, so the block partials are the same bits):
//   1. per round of KD_THREADS of them, a thread per query keeps its previous match if match_proven;
//   2. the block's warps re-search the round's unproven queries (warp_nearest, seeded with the previous match) and
//      compute the normal of every new match that has none cached.  Another block may compute the same normal at the
//      same time: the computation is deterministic, so both store the same bits, and no block ever waits for another;
//   3. once every round is searched, a thread per query: accumulate_match, then the block partial and, fused, the
//      solve in the last block.  The accumulators are not live during the searches.
// A block has KD_REFINE_THREADS threads: the first KD_THREADS own the queries (steps 1 and 3, the block partial of
// kd_residual_kernel's geometry), all of its warps share the searches of step 2.  A cfg2 block re-searches 13 queries
// and computes 4 normals in the median, 30 and 13 at most (profiles/h100_kd_residual_split_after.log): with 8 warps
// the slowest block's searches took 35 us, a chain of up to four searches per warp.
// GATE: match_proven<true>, warp_nearest<true> (an outlier computes no normal) and the residual's distance test.
// DEGEN: the eigenvalue-thresholded solve (block_partial_and_finish).
constexpr int KD_REFINE_THREADS = 512;
constexpr int KD_REFINE_WARPS = KD_REFINE_THREADS / 32;
// kd_icp_refine_body's shared state, owned by this function rather than by the template for the reason kd_residual_pose
// gives: the ungated kernels keep their shared-memory layout and SASS.
struct KdRefineShared {
    float* sT;
    int* s_hard;
    int* s_nh;
    unsigned long long (*s_stage)[KNN_STAGE];
};
__device__ __forceinline__ KdRefineShared kd_refine_shared() {
    __shared__ float sT[12];
    __shared__ int s_hard[KD_THREADS];
    __shared__ int s_nh;
    __shared__ unsigned long long s_stage[KD_REFINE_WARPS][KNN_STAGE];
    return KdRefineShared{sT, s_hard, &s_nh, s_stage};
}

template <bool GATE = false, bool DEGEN = false>
__device__ __forceinline__ void kd_icp_refine_body(const KdIndex& ix, const float4* __restrict__ queries,
                                                   const uint32_t* __restrict__ nq_dev, int64_t q_begin, int64_t q_stride,
                                                   FrameResult* fr, int scheme, float sigma, int k_normals,
                                                   int* __restrict__ match, float4* __restrict__ nn_state,
                                                   double* __restrict__ partials, float fuse_threshold,
                                                   unsigned long long* __restrict__ counters, unsigned block,
                                                   unsigned grid KD_SPLIT_ARG, KdGate gate = KdGate{},
                                                   IcpDegen dg = IcpDegen{}) {
    if (fr->done) return;
    const KdRefineShared sh = kd_refine_shared();
    float* sT = sh.sT;
    int* s_hard = sh.s_hard;
    int& s_nh = *sh.s_nh;
    unsigned long long(*s_stage)[KNN_STAGE] = sh.s_stage;
    if (threadIdx.x < 12) sT[threadIdx.x] = fr->T[threadIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool owner = threadIdx.x < KD_THREADS;  // warp-uniform: this thread has a query slot
    const int64_t nq = (int64_t)*nq_dev;
    const uint32_t valid = kd_normal_valid(ix.gen);
    int cand_nn = 0, cand_knn = 0, normals_here = 0;
    for (int64_t round = (int64_t)block * KD_THREADS;; round += (int64_t)grid * KD_THREADS) {
        if (q_begin + round * q_stride >= nq) break;  // block-uniform
        if (threadIdx.x == 0) s_nh = 0;
        __syncthreads();
        const int64_t qi = q_begin + (round + threadIdx.x) * q_stride;
        if (owner && qi < nq) {
            float p[3];
            transform_point(sT, queries[qi], p);
            if (!match_proven<GATE>(ix, p, match[qi], nn_state[qi], gate.dmax)) s_hard[atomicAdd(&s_nh, 1)] = threadIdx.x;
        }
        __syncthreads();
        const int nh = s_nh;
#ifdef PLS_KD_SPLIT
        if (threadIdx.x == 0 && split) split[9] += (unsigned long long)nh;  // not a time: the block's re-searches
#endif
        if (warp < nh) {
            const KdGridLocal g = kd_load_grid(ix);
            for (int e = warp; e < nh; e += KD_REFINE_WARPS) {
                const int64_t q = q_begin + (round + s_hard[e]) * q_stride;
                float p[3];
                transform_point(sT, queries[q], p);
                float second;
                const int pos = warp_nearest<GATE>(ix, g, p[0], p[1], p[2], match[q], lane, &cand_nn, &second, gate);
                if (lane == 0) {
                    match[q] = pos;
                    nn_state[q] = make_float4(p[0], p[1], p[2], second);
                }
                if (pos < 0) continue;
                const uint32_t state = __shfl_sync(FULL, __ldcg(reinterpret_cast<const uint32_t*>(&ix.normals[pos].w)), 0);
                if (state == valid) continue;
                float cov[6];
                warp_normal_moments(ix, g, __ldg(ix.sorted + pos), k_normals, lane, &cand_knn, s_stage[warp], cov);
                if (lane == 0) store_normal(ix, pos, cov, valid);
                ++normals_here;
            }
        }
        __syncthreads();  // s_hard / s_nh are reused by the next round
    }
    if (counters && lane == 0) {
        if (cand_nn) atomicAdd(counters + KDC_NN_CAND, (unsigned long long)cand_nn);
        if (cand_knn) atomicAdd(counters + KDC_KNN_CAND, (unsigned long long)cand_knn);
        if (normals_here) atomicAdd(counters + KDC_NORMALS, (unsigned long long)normals_here);
    }
#ifdef PLS_KD_SPLIT
    if (lane == 0 && split && normals_here) atomicAdd(split + 10, (unsigned long long)normals_here);  // normals computed
#endif
    // every match and normal of this block's queries is in place (the last round ended on a barrier)
    if (threadIdx.x == 0) PLS_SPLIT(1);
    double acc[NACC];
#pragma unroll
    for (int a = 0; a < NACC; ++a) acc[a] = 0.0;
    for (int64_t s = (int64_t)block * KD_THREADS + threadIdx.x; owner; s += (int64_t)grid * KD_THREADS) {
        const int64_t qi = q_begin + s * q_stride;
        if (qi >= nq) break;
        const int pos = match[qi];
        if (pos < 0) continue;
        float p[3];
        transform_point(sT, queries[qi], p);
        if constexpr (GATE)
            if (!(match_d2_f64(p, __ldg(ix.sorted + pos)) <= gate.max_d2)) continue;
        accumulate_match(acc, ix, p, pos, scheme, sigma KD_SPLIT_PASS);
    }
    block_partial_and_finish<KD_REFINE_THREADS, NACC, DEGEN>(acc, fr, partials, fuse_threshold, block,
                                                            grid KD_SPLIT_PASS, dg);
}

__global__ void __launch_bounds__(KD_REFINE_THREADS)
kd_icp_refine_kernel(KdIndex ix, const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev, int64_t q_begin,
                     int64_t q_stride, FrameResult* fr, int scheme, float sigma, int k_normals, int* __restrict__ match,
                     float4* __restrict__ nn_state, double* __restrict__ partials, float fuse_threshold,
                     unsigned long long* __restrict__ counters, int64_t bound, const uint32_t* __restrict__ bound_dev) {
    pls_grid_dependency_wait();
    const unsigned grid = kd_logical_blocks(bound, bound_dev);
    if (blockIdx.x >= grid) return;
    KD_SPLIT_BEGIN()
    kd_icp_refine_body(ix, queries, nq_dev, q_begin, q_stride, fr, scheme, sigma, k_normals, match, nn_state, partials,
                       fuse_threshold, counters, blockIdx.x, grid KD_SPLIT_PASS);
}

// ---- several sequences per launch (pls_process_frames) --------------------------------------------------------------
// What the kernels of one ICP iteration need of one sequence: the arguments its single path passes (every query is
// the sequence's own: q_begin 0, stride 1), and its share of each launch.  Built on the host by kdmap_batch_begin and
// uploaded once per call.
struct KdSeq {
    KdIndex ix;
    const float4* queries;
    const uint32_t* nq_dev;     // query count (FrameResult counts[1])
    FrameResult* fr;            // pose, done flag, solve ticket
    int* match;
    float4* nn_state;
    int* pending;               // normals work list
    int* hard;                  // queries the verify kernel could not prove (maps of KD_COLD_MAP_POINTS or more)
    uint32_t* lists;            // work-list words (SC_KD_LISTS)
    double* partials;
    unsigned long long* counters;
    int scheme;
    float sigma;
    int k_normals;
    float fuse_threshold;
    int max_iters;              // max_num_alignments: launches of later iterations leave the sequence alone
    int blocks;                 // grid_for(query bound): the residual kernel's geometry on the single path
    int refine_blocks;          // blocks, or 0 where later iterations take the four launches (kd_later_four_launch)
    int verify_blocks;          // kd_nn_verify_kernel's grid on the single path: a thread per query
    int nn_blocks, kn_blocks;   // its share of the resident wave of the 1-NN / normals kernels
};
static_assert(sizeof(KdSeq) % sizeof(int) == 0, "KdSeq is copied in 4-byte words");

// Sequence blockIdx.y's descriptor into shared memory, for every thread of the block.
__device__ __forceinline__ void load_seq(const KdSeq* __restrict__ seqs, KdSeq& s) {
    const int* src = reinterpret_cast<const int*>(seqs + blockIdx.y);
    int* dst = reinterpret_cast<int*>(&s);
    for (int i = threadIdx.x; i < (int)(sizeof(KdSeq) / sizeof(int)); i += blockDim.x) dst[i] = __ldg(src + i);
    __syncthreads();
}

// The batched entry points do not stamp in -DPLS_KD_SPLIT builds.
#ifdef PLS_KD_SPLIT
#define KD_SPLIT_NONE()                     \
    unsigned long long* split = nullptr;    \
    __shared__ unsigned long long s_split[2];
#else
#define KD_SPLIT_NONE()
#endif

// Does iteration `it` of the sequence run through the four launches below?  Its first iteration always does; a later one
// on a map of KD_COLD_MAP_POINTS or more, while the sequence has not reached its max_iters.
__device__ __forceinline__ bool four_launch_step(const KdSeq& s, int it) {
    return it == 0 || (s.refine_blocks == 0 && it < s.max_iters);
}

// Iteration `it` >= 1 of the sequences on maps of KD_COLD_MAP_POINTS or more: kd_nn_verify_kernel of each.
__global__ void __launch_bounds__(KD_THREADS) kd_nn_verify_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.verify_blocks || !four_launch_step(s, it)) return;
    kd_nn_verify_body(s.ix, s.queries, s.nq_dev, 0, 1, s.fr->T, &s.fr->done, s.match, s.nn_state, s.hard, s.lists, it & 1,
                      blockIdx.x);
}

// Iteration 0: every query of every sequence.  Iteration `it` >= 1: the queued queries of the four-launch sequences.
__global__ void __launch_bounds__(KD_THREADS) kd_nn_warp_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.nn_blocks || !four_launch_step(s, it)) return;
    kd_nn_warp_body(s.ix, s.queries, s.nq_dev, 0, 1, it == 0 ? nullptr : s.hard, s.lists, it & 1, s.fr->T, &s.fr->done,
                    s.match, s.nn_state, 1, s.pending, s.counters, blockIdx.x, s.nn_blocks);
}

// The normals of the sequences whose k is at most 31; kd_normals_wide_batch_kernel<R> takes the others.
__global__ void __launch_bounds__(KD_THREADS) kd_normals_warp_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.kn_blocks || !four_launch_step(s, it) || kd_wide_k(s.k_normals)) return;
    kd_normals_warp_body(s.ix, s.k_normals, s.pending, s.lists + KDL_PENDING + (it & 1), &s.fr->done, s.counters,
                         blockIdx.x, s.kn_blocks);
}

// The normals of the sequences with a wide k, k + 1 <= 32 R.  Which warp computes a normal does not change its bits, so
// the sequences share the block counts of the narrow kernel.
template <int R>
__global__ void __launch_bounds__(KD_THREADS) kd_normals_wide_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.kn_blocks || !four_launch_step(s, it) || !kd_wide_k(s.k_normals)) return;
    kd_normals_warp_body<R>(s.ix, s.k_normals, s.pending, s.lists + KDL_PENDING + (it & 1), &s.fr->done, s.counters,
                            blockIdx.x, s.kn_blocks);
}

__global__ void __launch_bounds__(KD_THREADS) kd_residual_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.blocks || !four_launch_step(s, it)) return;
    KD_SPLIT_NONE()
    kd_residual_body(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.match, s.partials, s.fuse_threshold,
                     blockIdx.x, s.blocks, 0.0 KD_SPLIT_PASS);
}

// pls_kdmap_evaluate_poses: iteration 0's residual pass of every registration at its FrameResult's pose, gated by
// max_d2, with no solve (kd_residual_body<true>).
__global__ void __launch_bounds__(KD_THREADS) kd_evaluate_batch_kernel(const KdSeq* __restrict__ seqs, double max_d2) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.blocks) return;
    KD_SPLIT_NONE()
    kd_residual_body<true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.match, s.partials, -1.f, blockIdx.x,
                           s.blocks, max_d2 KD_SPLIT_PASS);
}

// Registration blockIdx.x's row: its block partials summed in the fixed order of icp_finish_in_last_block, into
// out[PLS_EVAL_STATS * blockIdx.x], and entries 0..29 into its FrameResult's last_sums.
__global__ void __launch_bounds__(256) kd_evaluate_finish_kernel(const KdSeq* __restrict__ seqs, double* __restrict__ out) {
    __shared__ double sums[PLS_EVAL_STATS];
    const KdSeq* s = seqs + blockIdx.x;
    sum_partials_256<256, PLS_EVAL_STATS>(s->partials, s->blocks, sums);
    __syncthreads();
    if (threadIdx.x < PLS_EVAL_STATS) out[(size_t)PLS_EVAL_STATS * blockIdx.x + threadIdx.x] = sums[threadIdx.x];
    if (threadIdx.x < NACC) s->fr->last_sums[threadIdx.x] = sums[threadIdx.x];
}

// Iteration `it` (>= 1) of every sequence that has not reached its max_iters and whose later iterations take one launch.
__global__ void __launch_bounds__(KD_REFINE_THREADS) kd_icp_refine_batch_kernel(const KdSeq* __restrict__ seqs, int it) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.refine_blocks || it >= s.max_iters) return;
    KD_SPLIT_NONE()
    kd_icp_refine_body(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.k_normals, s.match, s.nn_state,
                       s.partials, s.fuse_threshold, s.counters, blockIdx.x, s.refine_blocks KD_SPLIT_PASS);
}

// The gated twins of the four-launch and refine batch kernels (pls_register_scans_gated): the same bodies with GATE,
// the registrations' gate a launch argument.  It is not a KdSeq field: a wider descriptor would change the copy and the
// stride of every batch kernel above.
__global__ void __launch_bounds__(KD_THREADS) kd_nn_verify_gated_batch_kernel(const KdSeq* __restrict__ seqs, int it,
                                                                              KdGate gate) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.verify_blocks || !four_launch_step(s, it)) return;
    kd_nn_verify_body<true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr->T, &s.fr->done, s.match, s.nn_state, s.hard, s.lists,
                            it & 1, blockIdx.x, gate.dmax);
}

__global__ void __launch_bounds__(KD_THREADS) kd_nn_warp_gated_batch_kernel(const KdSeq* __restrict__ seqs, int it,
                                                                            KdGate gate) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.nn_blocks || !four_launch_step(s, it)) return;
    kd_nn_warp_body<true>(s.ix, s.queries, s.nq_dev, 0, 1, it == 0 ? nullptr : s.hard, s.lists, it & 1, s.fr->T,
                          &s.fr->done, s.match, s.nn_state, 1, s.pending, s.counters, blockIdx.x, s.nn_blocks, gate);
}

__global__ void __launch_bounds__(KD_THREADS) kd_residual_gated_batch_kernel(const KdSeq* __restrict__ seqs, int it,
                                                                             double max_d2) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.blocks || !four_launch_step(s, it)) return;
    KD_SPLIT_NONE()
    kd_residual_body<false, true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.match, s.partials,
                                  s.fuse_threshold, blockIdx.x, s.blocks, max_d2 KD_SPLIT_PASS);
}

__global__ void __launch_bounds__(KD_REFINE_THREADS) kd_icp_refine_gated_batch_kernel(const KdSeq* __restrict__ seqs,
                                                                                      int it, KdGate gate) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.refine_blocks || it >= s.max_iters) return;
    KD_SPLIT_NONE()
    kd_icp_refine_body<true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.k_normals, s.match, s.nn_state,
                             s.partials, s.fuse_threshold, s.counters, blockIdx.x, s.refine_blocks KD_SPLIT_PASS, gate);
}

// The twins of the gated residual and refine batch kernels with the eigenvalue-thresholded solve
// (pls_register_scans_degeneracy; an ungated one runs them with an infinite gate, which matches as the ungated search
// does).  min_eigenvalue and the output rows, registration blockIdx.y's at degen + ICP_DEGEN_STRIDE * blockIdx.y, are
// launch arguments for the reason the gate is one.
__global__ void __launch_bounds__(KD_THREADS) kd_residual_gated_degen_batch_kernel(const KdSeq* __restrict__ seqs, int it,
                                                                                   double max_d2, double min_eigenvalue,
                                                                                   double* __restrict__ degen) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.blocks || !four_launch_step(s, it)) return;
    KD_SPLIT_NONE()
    const IcpDegen dg{min_eigenvalue, degen + (size_t)ICP_DEGEN_STRIDE * blockIdx.y, nullptr};
    kd_residual_body<false, true, true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.match, s.partials,
                                        s.fuse_threshold, blockIdx.x, s.blocks, max_d2 KD_SPLIT_PASS, dg);
}

__global__ void __launch_bounds__(KD_REFINE_THREADS)
kd_icp_refine_gated_degen_batch_kernel(const KdSeq* __restrict__ seqs, int it, KdGate gate, double min_eigenvalue,
                                       double* __restrict__ degen) {
    __shared__ KdSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.refine_blocks || it >= s.max_iters) return;
    KD_SPLIT_NONE()
    const IcpDegen dg{min_eigenvalue, degen + (size_t)ICP_DEGEN_STRIDE * blockIdx.y, nullptr};
    kd_icp_refine_body<true, true>(s.ix, s.queries, s.nq_dev, 0, 1, s.fr, s.scheme, s.sigma, s.k_normals, s.match,
                                   s.nn_state, s.partials, s.fuse_threshold, s.counters, blockIdx.x,
                                   s.refine_blocks KD_SPLIT_PASS, gate, dg);
}

// The done flags of every sequence, for the host's extra-round check.
__global__ void kd_batch_done_kernel(const KdSeq* __restrict__ seqs, int num, int* __restrict__ out) {
    for (int i = threadIdx.x; i < num; i += blockDim.x) out[i] = seqs[i].fr->done;
}

// Fine-grained API: [n,3] rows -> float4 queries (no row is dropped: outputs stay aligned with the inputs)
__global__ void kd_rows_to_float4_kernel(const float* __restrict__ rows, int64_t n, float4* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = make_float4(rows[3 * i], rows[3 * i + 1], rows[3 * i + 2], 0.f);
}

__global__ void kd_search_export_kernel(KdIndex ix, const int* __restrict__ match, int64_t n, float* __restrict__ out_nb,
                                        float* __restrict__ out_nrm, long long* __restrict__ out_idx) {
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int pos = match[i];
        float4 q = make_float4(nan, nan, nan, 0.f), nv = make_float4(nan, nan, nan, 0.f);
        long long idx = -1;
        if (pos >= 0) {
            q = __ldg(ix.sorted + pos);
            idx = (long long)__float_as_uint(q.w);
            if (out_nrm) nv = __ldcg(ix.normals + pos);
        }
        out_nb[3 * i] = q.x; out_nb[3 * i + 1] = q.y; out_nb[3 * i + 2] = q.z;
        if (out_idx) out_idx[i] = idx;
        if (out_nrm) { out_nrm[3 * i] = nv.x; out_nrm[3 * i + 1] = nv.y; out_nrm[3 * i + 2] = nv.z; }
    }
}

// pls_kdmap_knn: the (K)-NN list warp_knn gives each of n query rows [n,3], a warp per query.  Row r of the outputs,
// entry j < K: insertion index (.w of `sorted`) or -1, the float32 squared distance of the key, the sorted position.
__global__ void __launch_bounds__(KD_THREADS)
kd_knn_export_kernel(KdIndex ix, const float* __restrict__ rows, int64_t n, int K, long long* __restrict__ out_idx,
                     float* __restrict__ out_d2, int* __restrict__ out_pos) {
    __shared__ unsigned long long s_stage[KD_WARPS][KNN_STAGE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const KdGridLocal g = kd_load_grid(ix);
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t q = (int64_t)blockIdx.x * KD_WARPS + warp; q < n; q += (int64_t)gridDim.x * KD_WARPS) {
        const float x = rows[3 * q], y = rows[3 * q + 1], z = rows[3 * q + 2];
        int pos;
        warp_knn(ix, g, x, y, z, K, lane, pos, nullptr, s_stage[warp]);
        if (lane < K) {
            long long idx = -1;
            float d2 = nan;
            if (pos >= 0) {
                const float4 s = __ldg(ix.sorted + pos);
                idx = (long long)__float_as_uint(s.w);
                d2 = dist2_point(x, y, z, s);
            }
            out_idx[q * K + lane] = idx;
            out_d2[q * K + lane] = d2;
            if (out_pos) out_pos[q * K + lane] = pos;
        }
    }
}

// The same for 32 < K <= 32 R (warp_knn_wide): lane l writes entries l, l + 32, ... of the row.  KD_THREADS threads;
// the register cap is kd_normals_wide_kernel's.
template <int R>
__global__ void __maxnreg__(128)
kd_knn_wide_export_kernel(KdIndex ix, const float* __restrict__ rows, int64_t n, int K, long long* __restrict__ out_idx,
                          float* __restrict__ out_d2, int* __restrict__ out_pos) {
    __shared__ unsigned long long s_stage[KD_WARPS][KNN_STAGE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const KdGridLocal g = kd_load_grid(ix);
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t q = (int64_t)blockIdx.x * KD_WARPS + warp; q < n; q += (int64_t)gridDim.x * KD_WARPS) {
        const float x = rows[3 * q], y = rows[3 * q + 1], z = rows[3 * q + 2];
        unsigned long long kept[R];
        warp_knn_wide<R>(ix, g, x, y, z, K, lane, kept, nullptr, s_stage[warp]);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int j = r * 32 + lane;
            if (j >= K) break;
            const int pos = kept[r] != KNN_NONE ? (int)(unsigned)kept[r] : -1;
            long long idx = -1;
            float d2 = nan;
            if (pos >= 0) {
                const float4 s = __ldg(ix.sorted + pos);
                idx = (long long)__float_as_uint(s.w);
                d2 = dist2_point(x, y, z, s);
            }
            out_idx[q * K + j] = idx;
            out_d2[q * K + j] = d2;
            if (out_pos) out_pos[q * K + j] = pos;
        }
    }
}

size_t cell_table_bytes(int64_t M, uint32_t* masks, size_t* offsets) {
    size_t off = 0;
    for (int l = 0; l < KD_MAX_LEVELS; ++l) {
        uint64_t want = (uint64_t)(1.5 * (double)M) >> l;
        uint32_t sz = 64;
        while (sz < want) sz <<= 1;
        if (masks) masks[l] = sz - 1;
        if (offsets) offsets[l] = off;
        off += (size_t)sz * sizeof(uint4);
    }
    return off;
}

// Sizes every per-point array of the map at once.  The map grows frame by frame until local_map_size frames are
// held, then oscillates around that size: reserving the steady state (local_map_size + 1 frames of the largest
// frame seen, 30 % head-room) on the first insertion means NO further allocation -- and none of the stream
// synchronisations an allocation implies -- while the map fills up, i.e. inside any timed region that starts after
// the first frame.  `need` beyond the plan (a denser frame later on) re-plans with 25 % head-room.
// Tables and normal states are generation-stamped and never cleared per build, so fresh memory is zeroed here once
// (generation 0 is never used).
void kd_reserve_capacity(pls_context* ctx, int64_t need) {
    KdMap& kd = ctx->kd;
    if (need <= kd.cap_points) return;
    cudaStream_t st = ctx->stream;
    int64_t steady = (int64_t)(1.3 * (double)kd.max_frame * (double)(ctx->cfg.local_map_size + 1));
    if (steady > need + (8ll << 20)) steady = need + (8ll << 20);  // a multi-million-point insertion plans 8 M ahead at most
    int64_t cap = need + need / 4 + 64;
    if (cap < steady) cap = steady;
    const size_t C = (size_t)cap;
    kd.store[kd.cur].reserve_exact(C * sizeof(float4), st, true);  // the live points survive
    kd.store[kd.cur ^ 1].reserve_exact(C * sizeof(float4), st);
    kd.morton.reserve_exact(C * sizeof(uint64_t), st);
    kd.order.reserve_exact(C * sizeof(uint32_t), st);
    kd.sorted.reserve_exact(C * sizeof(float4), st);
    kd.normals.reserve_exact(C * sizeof(float4), st);
    const size_t table_bytes = cell_table_bytes(cap, nullptr, nullptr);
    kd.cells.reserve_exact(table_bytes, st);
    PLS_CUDA(cudaMemsetAsync(kd.normals.p, 0, C * sizeof(float4), st));
    PLS_CUDA(cudaMemsetAsync(kd.cells.p, 0, table_bytes, st));
    kd.cap_points = cap;
}

KdIndex make_index(pls_context* ctx) {
    KdIndex ix;
    ix.sorted = ctx->kd.sorted.as<float4>();
    ix.normals = ctx->kd.normals.as<float4>();
    ix.M = (int)ctx->kd.indexed;
    ix.gen = ctx->kd.gen;
    ix.grid = ctx->kd.grid_hdr.as<KdGridHeader>();
    for (int l = 0; l < KD_MAX_LEVELS; ++l) {
        ix.table[l] = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(ctx->kd.cells.p) + ctx->kd.table_offset[l]);
        ix.mask[l] = ctx->kd.table_mask[l];
    }
    ix.stats = ctx->kd.stats.p ? ctx->kd.stats.as<unsigned long long>() : nullptr;
    return ix;
}

// The per-frame index build (stands in for the KDTree rebuild of local_map.py:365-369): header, cell keys, four
// radix passes, one finishing pass.  Nothing is cleared: tables and normal states carry the build's generation.
// upd (nullable): kd.count is a bound of the point count, which the device holds in upd->total (the launches are sized
// for the bound and read the count; the caller settles kd.indexed / kd.valid and the profile credit once it is known).
void build_index(pls_context* ctx, const KdUpdateWords* upd) {
    KdMap& kd = ctx->kd;
    cudaStream_t st = ctx->stream;
    const int64_t M = kd.count;
    kd.indexed = M;
    kd.valid = M > 0;
    if (M <= 0) return;
    ProfileScope ps(ctx, 3, (double)M * 32.0, upd == nullptr);
    const uint32_t* n_dev = upd ? &upd->total : nullptr;
    PLS_REQUIRE(M < (1ll << 30), "kd map: too many points");
    kd_reserve_capacity(ctx, M);
    kd.gen += 1;
    if (kd.gen >= 0x7ffffff0u) {  // state words are 2 gen (+1): restart the generations on clean memory
        PLS_CUDA(cudaMemsetAsync(kd.normals.p, 0, kd.normals.cap, st));
        PLS_CUDA(cudaMemsetAsync(kd.cells.p, 0, kd.cells.cap, st));
        kd.gen = 1;
    }
    const float4* pts = kd.store[kd.cur].as<float4>();
    kd.grid_hdr.reserve(sizeof(KdGridHeader), st);
    static const float cell_target = getenv("PLS_KD_CELL") ? (float)atof(getenv("PLS_KD_CELL")) : KD_CELL_TARGET;
    kd_grid_header_kernel<<<1, 32, 0, st>>>(kd.bbox.as<int>(), kd.grid_hdr.as<KdGridHeader>(), cell_target,
                                            upd ? &upd->gate : nullptr);
    PLS_CHECK_LAUNCH();
    kd.bbox_clean = true;
    launch_dependent(kd_cell_key_kernel, grid_for(M, 256, 8 * kNumSMs), 256, st, pts, M, kd.grid_hdr.as<KdGridHeader>(),
                     kd.morton.as<uint64_t>(), kd.order.as<uint32_t>(), n_dev);
    uint64_t* sk;
    uint32_t* sv;
    radix_sort_pairs(ctx, kd.morton.as<uint64_t>(), kd.order.as<uint32_t>(), M, 4, &sk, &sv, kd.cap_points, n_dev);
    // table geometry follows the capacity, not M: it only changes when the buffers are re-planned
    cell_table_bytes(kd.cap_points, kd.table_mask, kd.table_offset);
    CellTables T;
    for (int l = 0; l < KD_MAX_LEVELS; ++l) {
        T.table[l] = reinterpret_cast<uint4*>(reinterpret_cast<char*>(kd.cells.p) + kd.table_offset[l]);
        T.mask[l] = kd.table_mask[l];
    }
    launch_dependent(kd_finalize_kernel, grid_for(M, 256, 8 * kNumSMs), 256, st, pts, sk, sv, M, T, kd.grid_hdr.as<KdGridHeader>(),
                     kd.gen, kd.sorted.as<float4>(), n_dev);
}

}  // namespace

void kdmap_reset(pls_context* ctx) {
    if (getenv("PLS_KD_STATS") && !ctx->kd.stats.p) {
        ctx->kd.stats.reserve(16 * sizeof(unsigned long long), ctx->stream);
        cudaMemsetAsync(ctx->kd.stats.p, 0, 16 * sizeof(unsigned long long), ctx->stream);
    }
    ctx->kd.count = 0;
    ctx->kd.cur = 0;
    ctx->kd.frame_counts.clear();
    ctx->kd.indexed = 0;
    ctx->kd.valid = false;
    ctx->kd.bbox_clean = false;
    ctx->kd.max_frame = 0;   // the buffers (cap_points) and the generation counter are kept: a re-initialised
                             // sequence reuses them
    ctx->kd.searched = false;
}

template <typename T>
static void pack_valid_rows_impl(pls_context* ctx, const T* pts_dev, int64_t n, float4* out, uint32_t* count_dev) {
    cudaStream_t st = ctx->stream;
    if (n <= 0) {
        PLS_CUDA(cudaMemsetAsync(count_dev, 0, sizeof(uint32_t), st));
        return;
    }
    ctx->tmp[1].reserve((size_t)n, st);
    ctx->tmp[2].reserve((size_t)n * sizeof(uint32_t), st);
    const int g = grid_for(n, 256, 8 * kNumSMs);
    kd_valid_rows_kernel<T><<<g, 256, 0, st>>>(pts_dev, n, ctx->tmp[1].as<uint8_t>());
    PLS_CHECK_LAUNCH();
    exclusive_scan_flags(ctx, ctx->tmp[1].as<uint8_t>(), n, ctx->tmp[2].as<uint32_t>(), count_dev);
    kd_pack_rows_kernel<T><<<g, 256, 0, st>>>(pts_dev, n, ctx->tmp[1].as<uint8_t>(), ctx->tmp[2].as<uint32_t>(), out);
    PLS_CHECK_LAUNCH();
}

void pack_valid_rows(pls_context* ctx, const float* pts_dev, int64_t n, float4* out, uint32_t* count_dev) {
    pack_valid_rows_impl<float>(ctx, pts_dev, n, out, count_dev);
}
void pack_valid_rows_f64(pls_context* ctx, const double* pts_dev, int64_t n, float4* out, uint32_t* count_dev) {
    pack_valid_rows_impl<double>(ctx, pts_dev, n, out, count_dev);
}

void pack_valid_scans(pls_context* ctx, const std::vector<KdScanRows>& scans) {
    cudaStream_t st = ctx->stream;
    const size_t bytes = scans.size() * sizeof(KdScanRows);
    ctx->stage_in[2].reserve(bytes, st);
    PLS_CUDA(cudaMemcpyAsync(ctx->stage_in[2].p, scans.data(), bytes, cudaMemcpyHostToDevice, st));
    kd_pack_scans_kernel<<<(unsigned)scans.size(), KD_PACK_THREADS, 0, st>>>(ctx->stage_in[2].as<KdScanRows>());
    PLS_CHECK_LAUNCH();
}

void pack_valid_pixels(pls_context* ctx, const float* vmap_dev, int64_t hw, float min_norm, float4* out,
                       uint32_t* count_dev) {
    cudaStream_t st = ctx->stream;
    ctx->tmp[1].reserve((size_t)hw, st);
    ctx->tmp[2].reserve((size_t)hw * sizeof(uint32_t), st);
    const int g = grid_for(hw, 256, 8 * kNumSMs);
    kd_valid_pixels_kernel<<<g, 256, 0, st>>>(vmap_dev, hw, min_norm, ctx->tmp[1].as<uint8_t>());
    PLS_CHECK_LAUNCH();
    exclusive_scan_flags(ctx, ctx->tmp[1].as<uint8_t>(), hw, ctx->tmp[2].as<uint32_t>(), count_dev);
    kd_pack_pixels_kernel<<<g, 256, 0, st>>>(vmap_dev, hw, ctx->tmp[1].as<uint8_t>(), ctx->tmp[2].as<uint32_t>(), out);
    PLS_CHECK_LAUNCH();
}

namespace {

// The device side of a map update: move + append + evict into the other store, then the index rebuild.  total is the
// new point count, or with upd a bound of it (see build_index).
void move_and_rebuild(pls_context* ctx, int64_t skip, int64_t kept, const Rigid& X, const float4* fresh_dev,
                      int64_t num_new, int64_t total, const KdUpdateWords* upd) {
    KdMap& kd = ctx->kd;
    cudaStream_t st = ctx->stream;
    kd_reserve_capacity(ctx, total > 0 ? total : 1);
    const int dst = kd.cur ^ 1;
    kd.bbox.reserve(8 * sizeof(int), st);
    if (!kd.bbox_clean) {
        kd_bbox_init_kernel<<<1, 32, 0, st>>>(kd.bbox.as<int>());
        PLS_CHECK_LAUNCH();
    }
    kd.bbox_clean = false;
    if (total > 0) {
        kd_move_append_kernel<<<grid_for(total, 256, 8 * kNumSMs), 256, 0, st>>>(
            kd.store[kd.cur].as<float4>(), skip, kept, X, fresh_dev, nullptr, num_new, kd.store[dst].as<float4>(),
            kd.bbox.as<int>(), upd);
        PLS_CHECK_LAUNCH();
    }
    kd.cur = dst;
    kd.count = total;
    // a device-decided update leaves the searched generation's sorted points in sorted_prev (its caller swapped)
    kd.prev_gen = upd ? kd.gen : 0;
    build_index(ctx, upd);
}

}  // namespace

// Move the map by inverse(rel_pose), append `num_new` packed points, evict, rebuild the index
// (local_map.py:330-369).
void kdmap_update_packed(pls_context* ctx, const float* rel_pose_host, const float4* fresh_dev, int64_t num_new,
                         bool has_new) {
    KdMap& kd = ctx->kd;
    Rigid X;
    int64_t skip = 0;
    const bool first = kd.frame_counts.empty() && kd.count == 0;
    if (first) {
        for (int i = 0; i < 9; ++i) X.R[i] = (i % 4 == 0) ? 1.f : 0.f;
        X.t[0] = X.t[1] = X.t[2] = 0.f;
        kd.frame_counts.push_back(num_new);
    } else {
        float inv[16];
        rigid_inverse(rel_pose_host, inv);
        X.R[0] = inv[0]; X.R[1] = inv[1]; X.R[2] = inv[2];
        X.R[3] = inv[4]; X.R[4] = inv[5]; X.R[5] = inv[6];
        X.R[6] = inv[8]; X.R[7] = inv[9]; X.R[8] = inv[10];
        X.t[0] = inv[3]; X.t[1] = inv[7]; X.t[2] = inv[11];
        if (has_new) {
            kd.frame_counts.push_back(num_new);
            if ((int)kd.frame_counts.size() > ctx->cfg.local_map_size) {
                skip = kd.frame_counts.front();
                kd.frame_counts.pop_front();
            }
        }
    }
    if (!has_new) num_new = 0;
    const int64_t kept = kd.count - skip;
    const int64_t total = kept + num_new;
    if (num_new > kd.max_frame) kd.max_frame = num_new;
    move_and_rebuild(ctx, skip, kept, X, fresh_dev, num_new, total, nullptr);
}

int64_t kdmap_device_update_bound(const pls_context* ctx, int64_t new_bound) {
    const KdMap& kd = ctx->kd;
    if (kd.frame_counts.empty() || kd.gen + 1 >= 0x7ffffff0u) return 0;
    int64_t bound = kd.count + new_bound;
    if (bound > kd.cap_points) bound = kd.cap_points;
    if (bound > (1ll << 30) - 1) bound = (1ll << 30) - 1;
    return bound;
}

void kdmap_update_on_device(pls_context* ctx, const float4* fresh_dev, int64_t bound, const KdUpdateWords* upd) {
    KdMap& kd = ctx->kd;
    PLS_REQUIRE(bound > 0 && bound >= kd.count && bound <= kd.cap_points,
                "kd map: a device-decided update needs a bound within the planned capacity");
    // the host enqueues this before it has seen the frame's result, whose last correspondences
    // (pls_kdmap_last_correspondences) read the sorted points of the index the frame searched: the build writes the
    // other buffer
    std::swap(kd.sorted, kd.sorted_prev);
    kd.sorted.reserve_exact((size_t)kd.cap_points * sizeof(float4), ctx->stream);
    move_and_rebuild(ctx, 0, bound, Rigid{}, fresh_dev, bound - kd.count, bound, upd);
}

void kdmap_settle_device_update(pls_context* ctx, const KdUpdateWords& w, int local_map_size) {
    KdMap& kd = ctx->kd;
    if (w.insert) {
        kd.frame_counts.push_back((int64_t)w.num_new);
        if ((int)kd.frame_counts.size() > local_map_size) kd.frame_counts.pop_front();
        if ((int64_t)w.num_new > kd.max_frame) kd.max_frame = (int64_t)w.num_new;
    }
    kd.count = (int64_t)w.total;
    kd.indexed = kd.count;
    kd.valid = kd.count > 0;
    if (kd.count > 0) profile_credit(ctx, 3, 1, (double)kd.count * 32.0);
}

void kdmap_update(pls_context* ctx, const float* rel_pose_host, const float* pts_dev, int64_t n,
                  const float* vmap_dev, int H, int W, int64_t known_count) {
    cudaStream_t st = ctx->stream;
    const bool has_new = (pts_dev != nullptr) || (vmap_dev != nullptr);
    const int64_t cap_new = pts_dev ? n : (vmap_dev ? (int64_t)H * W : 0);
    int64_t num_new = 0;
    if (has_new && cap_new > 0) {
        ctx->tmp[4].reserve((size_t)cap_new * sizeof(float4), st);
        uint32_t* cnt = scalar_u32(ctx, SC_INSERT_COUNT);
        if (pts_dev) {
            pack_valid_rows(ctx, pts_dev, cap_new, ctx->tmp[4].as<float4>(), cnt);
        } else {
            pack_valid_pixels(ctx, vmap_dev, cap_new, 0.01f, ctx->tmp[4].as<float4>(), cnt);  // local_map.py:320-328
        }
        if (known_count >= 0) {
            num_new = known_count;
        } else {
            uint32_t c = 0;
            PLS_CUDA(cudaMemcpyAsync(&c, cnt, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
            PLS_CUDA(cudaStreamSynchronize(st));
            num_new = c;
        }
    }
    kdmap_update_packed(ctx, rel_pose_host, ctx->tmp[4].as<float4>(), num_new, has_new);
}

// Launch geometry of the search kernels: about ONE resident wave of warps (a second, partial wave would wait for the
// first to drain), each warp looping over its share.
static int resident_blocks(const void* kernel) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, KD_THREADS, 0) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 2;
    }
    return per_sm * kNumSMs;
}

static unsigned long long* kd_counters(pls_context* ctx) {
    return reinterpret_cast<unsigned long long*>(scalar_u32(ctx, SC_KD_COUNTERS));
}

// What the last search was, for pls_kdmap_last_correspondences.  n: the query count of a fine-grained search (that of an
// ICP iteration is in the FrameResult).
static void record_search(KdMap& kd, bool icp, bool sharded, bool normals, int64_t n) {
    kd.searched = true;
    kd.searched_icp = icp;
    kd.searched_sharded = sharded;
    kd.searched_normals = normals;
    kd.searched_gen = kd.gen;
    kd.searched_n = n;
}

// One sequence's kd search and ICP iteration over `query_bound` queries split over `num_ranks` shards: this shard's query
// bound, its work-list slots and its block counts.
struct KdPlan {
    int64_t mine;  // queries of this shard
    size_t slots;  // work-list slots of this shard
    int blocks;    // residual and refine kernels
    int wblocks;   // warp kernels (1-NN, normals), before the cap at a resident wave
};

// Reserves, on ctx->stream, what the plan's iterations use: nn_prev and kd_nn_state are indexed by query (not by shard
// slot), kd_worklist holds two lists of the shard's slots, partials one row per residual block.
static KdPlan plan_kd_iteration(pls_context* ctx, int64_t query_bound, int num_ranks) {
    cudaStream_t st = ctx->stream;
    KdPlan p;
    p.mine = (query_bound + num_ranks - 1) / num_ranks;
    p.slots = (size_t)p.mine + 64;
    p.blocks = grid_for(p.mine, KD_THREADS, 8 * kNumSMs);
    p.wblocks = (int)((p.mine + KD_WARPS - 1) / KD_WARPS);
    ctx->nn_prev.reserve((size_t)query_bound * sizeof(int), st);  // previous matches: ignored by iteration 0
    ctx->partials.reserve((size_t)p.blocks * NACC * sizeof(double), st);
    ctx->kd_worklist.reserve(2 * p.slots * sizeof(int), st);
    ctx->kd_nn_state.reserve(p.slots * (size_t)num_ranks * sizeof(float4), st);
    return p;
}

// kd_normals_wide_kernel<R> over the queued map points, at most one resident wave.
template <int R>
static void launch_normals_wide(pls_context* ctx, int wblocks, const KdIndex& ix, const int* pending, const uint32_t* count,
                                const int* done, unsigned long long* counters) {
    static const int resident = resident_blocks((const void*)kd_normals_wide_kernel<R>);
    launch_dependent(kd_normals_wide_kernel<R>, wblocks < resident ? wblocks : resident, KD_THREADS, ctx->stream, ix,
                     ctx->cfg.num_neighbors_normals, pending, count, done, counters);
}

// The search of one ICP iteration (or of one fine-grained API call).  first: every query is searched; later iterations
// first verify the previous matches and search only the unproven ones.
static void launch_search(pls_context* ctx, const KdPlan& plan, const KdIndex& ix, const float4* queries, const uint32_t* nq_dev,
                          int rank, int num_ranks, const float* T, const int* done, int* match, bool first, bool normals,
                          int parity) {
    cudaStream_t st = ctx->stream;
    int* pending = ctx->kd_worklist.as<int>();
    int* hard_nn = pending + plan.slots;
    float4* nn_state = ctx->kd_nn_state.as<float4>();
    uint32_t* lists = scalar_u32(ctx, SC_KD_LISTS);
    unsigned long long* counters = kd_counters(ctx);
    const int tblocks = (int)((plan.mine + KD_THREADS - 1) / KD_THREADS);
    static const int resident_nn = resident_blocks((const void*)kd_nn_warp_kernel);
    static const int resident_kn = resident_blocks((const void*)kd_normals_warp_kernel);
    const int wblocks = plan.wblocks;
    if (!first) {
        ProfileScope p6(ctx, 6, 0.0);
        kd_nn_verify_kernel<<<tblocks, KD_THREADS, 0, st>>>(ix, queries, nq_dev, (int64_t)rank, (int64_t)num_ranks, T, done, match,
                                                            nn_state, hard_nn, lists, parity);
        PLS_CHECK_LAUNCH();
    }
    {
        ProfileScope p7(ctx, 7, 0.0);
        launch_dependent(kd_nn_warp_kernel, wblocks < resident_nn ? wblocks : resident_nn, KD_THREADS, st, ix, queries, nq_dev,
                         (int64_t)rank, (int64_t)num_ranks, first ? nullptr : hard_nn, lists, parity, T, done, match, nn_state,
                         normals ? 1 : 0, pending, counters);
    }
    if (!normals) return;
    ProfileScope p9(ctx, 9, 0.0);
    const int k = ctx->cfg.num_neighbors_normals;
    if (!kd_wide_k(k)) {
        launch_dependent(kd_normals_warp_kernel, wblocks < resident_kn ? wblocks : resident_kn, KD_THREADS, st, ix, k, pending,
                         lists + KDL_PENDING + parity, done, counters);
        return;
    }
    switch (kd_wide_regs(k + 1)) {
        case 2: launch_normals_wide<2>(ctx, wblocks, ix, pending, lists + KDL_PENDING + parity, done, counters); break;
        case 4: launch_normals_wide<4>(ctx, wblocks, ix, pending, lists + KDL_PENDING + parity, done, counters); break;
        default: launch_normals_wide<8>(ctx, wblocks, ix, pending, lists + KDL_PENDING + parity, done, counters); break;
    }
}

// Later ICP iterations run as one kd_icp_refine_kernel, except on maps of this many points or more.  On the 5 M-point
// map of BASELINE config 4 the single kernel was slower on H100 (1.10-1.22 ms per registration against 0.91-0.92 with
// the four launches; the same with the kernel at 120 registers and no spills), on the 0.65 M-point cfg2 map faster.
// The cut-off between the two is not tuned: no map size in between has been measured.
constexpr int64_t KD_COLD_MAP_POINTS = 2000000;

// Do an ICP's later iterations on a map of `indexed` points with k normal neighbours take the four launches (verify /
// 1-NN / normals / residual) rather than kd_icp_refine_kernel?  On large maps (above), and for a wide k: the refine
// kernel computes normals inline with the one-key-per-lane warp_knn only, so its registers stay those of k <= 31.
static bool kd_later_four_launch(int64_t indexed, int k) { return indexed >= KD_COLD_MAP_POINTS || kd_wide_k(k); }

// One ICP iteration over the device-resident queries (float4 in ctx->query_ptr, count in the FrameResult); writes
// block partials to ctx->partials and returns the block count.
int kdmap_icp_iteration(pls_context* ctx, int64_t query_bound, const uint32_t* bound_dev, int rank, int num_ranks, int it,
                        float fuse_threshold, bool* solved) {
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    PLS_REQUIRE(!bound_dev || num_ranks == 1, "kd ICP: a device-side query bound needs an unsharded frame");
    cudaStream_t st = ctx->stream;
    FrameResult* fr = frame_result_dev(ctx);
    const uint32_t* nq_dev = reinterpret_cast<const uint32_t*>(&fr->counts[1]);
    // credited per executed iteration by the caller (the launch is a no-op once ICP converged)
    ProfileScope ps(ctx, 0, 0.0, false);
    const KdIndex ix = make_index(ctx);
    const KdPlan plan = plan_kd_iteration(ctx, query_bound, num_ranks);
    const int blocks = plan.blocks;
    record_search(ctx->kd, true, num_ranks > 1, true, 0);
    if (it == 0 || kd_later_four_launch(ctx->kd.indexed, ctx->cfg.num_neighbors_normals)) {
        launch_search(ctx, plan, ix, ctx->query_ptr, nq_dev, rank, num_ranks, fr->T, &fr->done, ctx->nn_prev.as<int>(), it == 0,
                      true, it & 1);
        ProfileScope p10(ctx, 10, 0.0);
        launch_dependent(kd_residual_kernel, blocks, KD_THREADS, st, ix, ctx->query_ptr, nq_dev, (int64_t)rank, (int64_t)num_ranks,
                         fr, ctx->cfg.scheme, ctx->cfg.sigma, ctx->nn_prev.as<int>(), ctx->partials.as<double>(), fuse_threshold,
                         plan.mine, bound_dev);
    } else {
        ProfileScope p11(ctx, 11, 0.0);
        launch_dependent(kd_icp_refine_kernel, blocks, KD_REFINE_THREADS, st, ix, ctx->query_ptr, nq_dev, (int64_t)rank,
                         (int64_t)num_ranks, fr, ctx->cfg.scheme, ctx->cfg.sigma, ctx->cfg.num_neighbors_normals,
                         ctx->nn_prev.as<int>(), ctx->kd_nn_state.as<float4>(), ctx->partials.as<double>(), fuse_threshold,
                         kd_counters(ctx), plan.mine, bound_dev);
    }
    *solved = fuse_threshold >= 0.f;
    return blocks;
}

// The descriptor of one sequence's (or one registration's) ICP on ctx's map, with its per-query and per-block state at
// the given addresses; fr is its FrameResult, queries and nq_dev its queries and their count.
static KdSeq make_seq(pls_context* ctx, const KdPlan& plan, const float4* queries, FrameResult* fr, const uint32_t* nq_dev,
                      int* match, float4* nn_state, int* worklist, uint32_t* words, double* partials, int share_nn,
                      int share_kn) {
    KdSeq s;
    s.ix = make_index(ctx);
    s.queries = queries;
    s.nq_dev = nq_dev;
    s.fr = fr;
    s.match = match;
    s.nn_state = nn_state;
    s.pending = worklist;
    s.hard = worklist + plan.slots;
    s.lists = words + (SC_KD_LISTS - SC_KD_COUNTERS);
    s.partials = partials;
    s.counters = reinterpret_cast<unsigned long long*>(words);
    s.scheme = ctx->cfg.scheme;
    s.sigma = ctx->cfg.sigma;
    s.k_normals = ctx->cfg.num_neighbors_normals;
    s.fuse_threshold = ctx->cfg.threshold_delta_pose;
    s.max_iters = ctx->cfg.max_num_alignments;
    s.blocks = plan.blocks;
    s.refine_blocks = kd_later_four_launch(ctx->kd.indexed, ctx->cfg.num_neighbors_normals) ? 0 : plan.blocks;
    s.verify_blocks = (int)((plan.mine + KD_THREADS - 1) / KD_THREADS);
    s.nn_blocks = plan.wblocks < share_nn ? plan.wblocks : share_nn;
    s.kn_blocks = plan.wblocks < share_kn ? plan.wblocks : share_kn;
    return s;
}

// The launch widths of kdmap_batch_iterations for these descriptors (see kdmap_batch_begin), and their upload into
// lead->batch_buf on st.
static void upload_seqs(pls_context* lead, const std::vector<KdSeq>& seqs, cudaStream_t st, int* grid) {
    grid[0] = grid[1] = grid[2] = 1;
    grid[3] = grid[4] = grid[5] = 0;
    for (const KdSeq& s : seqs) {
        grid[0] = grid[0] > s.blocks ? grid[0] : s.blocks;
        grid[1] = grid[1] > s.nn_blocks ? grid[1] : s.nn_blocks;
        grid[2] = grid[2] > s.kn_blocks ? grid[2] : s.kn_blocks;
        if (s.refine_blocks == 0) grid[3] = grid[3] > s.verify_blocks ? grid[3] : s.verify_blocks;
        else grid[4] = 1;
        if (kd_wide_k(s.k_normals)) {
            const int r = kd_wide_regs(s.k_normals + 1);
            grid[5] = grid[5] > r ? grid[5] : r;
        }
    }
    const size_t bytes = seqs.size() * sizeof(KdSeq);
    lead->batch_buf.reserve(bytes + PLS_MAX_SEQUENCES * sizeof(int), st);
    PLS_CUDA(cudaMemcpyAsync(lead->batch_buf.p, seqs.data(), bytes, cudaMemcpyHostToDevice, st));
}

// pls_process_frames: the descriptors of the sequences whose ICP runs in this call, into lead->batch_buf (uploaded on
// st), and every buffer their iterations use reserved as their single path reserves it.
// grid[KD_BATCH_GRID]: the launch widths, the largest residual / 1-NN / normals block count of a sequence, the largest
// verify block count of a sequence whose later iterations take the four launches (0: none does), 1 if any sequence's
// take kd_icp_refine_kernel, and the keys per lane R of the widest k above 31 (0: every k is at most 31).
void kdmap_batch_begin(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                       int* grid) {
    static const int resident_nn = resident_blocks((const void*)kd_nn_warp_batch_kernel);
    static const int resident_kn = resident_blocks((const void*)kd_normals_warp_batch_kernel);
    const int share_nn = (resident_nn + num - 1) / num, share_kn = (resident_kn + num - 1) / num;
    std::vector<KdSeq> seqs;
    for (int i = 0; i < num; ++i) {
        pls_context* ctx = ctxs[i];
        PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
        const KdPlan plan = plan_kd_iteration(ctx, query_bounds[i], 1);
        ctx->last_sharded = false;
        record_search(ctx->kd, true, false, true, 0);
        FrameResult* fr = frame_result_dev(ctx);
        seqs.push_back(make_seq(ctx, plan, ctx->query_ptr, fr, reinterpret_cast<const uint32_t*>(&fr->counts[1]), ctx->nn_prev.as<int>(),
                                ctx->kd_nn_state.as<float4>(), ctx->kd_worklist.as<int>(), scalar_u32(ctx, SC_KD_COUNTERS),
                                ctx->partials.as<double>(), share_nn, share_kn));
    }
    upload_seqs(lead, seqs, st, grid);
}

// ICP iterations [first, last) of the sequences kdmap_batch_begin (or kdmap_hypotheses_begin) described, on st: one
// launch per kernel for all of them.  A later iteration is kd_icp_refine_batch_kernel for the sequences whose later
// iterations take one launch and the four launches verify / 1-NN / normals / residual for the others; the normals of a
// wide k are one more launch, made only if some sequence has one.  No launch grows with num.
// The 1-NN and normals launches of iteration `it` of the four-launch path for the sequences described in seqs; gate
// (nullable): the gated registrations' gate.
static void batch_search(const KdSeq* seqs, int num, cudaStream_t st, const int* grid, int it,
                         const KdGate* gate = nullptr) {
    if (gate) kd_nn_warp_gated_batch_kernel<<<dim3(grid[1], num), KD_THREADS, 0, st>>>(seqs, it, *gate);
    else kd_nn_warp_batch_kernel<<<dim3(grid[1], num), KD_THREADS, 0, st>>>(seqs, it);
    PLS_CHECK_LAUNCH();
    kd_normals_warp_batch_kernel<<<dim3(grid[2], num), KD_THREADS, 0, st>>>(seqs, it);
    PLS_CHECK_LAUNCH();
    if (grid[5]) {
        const dim3 g(grid[2], num);
        if (grid[5] == 2) kd_normals_wide_batch_kernel<2><<<g, KD_THREADS, 0, st>>>(seqs, it);
        else if (grid[5] == 4) kd_normals_wide_batch_kernel<4><<<g, KD_THREADS, 0, st>>>(seqs, it);
        else kd_normals_wide_batch_kernel<8><<<g, KD_THREADS, 0, st>>>(seqs, it);
        PLS_CHECK_LAUNCH();
    }
}

// The gate of a finite max_distance >= 0 (KdGate, kdmap_device.cuh): max_d2 = max_distance^2 in float64, and the
// float32 bounds rounded up.
static KdGate kd_gate_of(double max_distance) {
    auto up = [](double v) {  // the least float32 >= v (+inf above FLT_MAX)
        if (!(v <= (double)FLT_MAX)) return INFINITY;
        float f = (float)v;
        return (double)f < v ? nextafterf(f, INFINITY) : f;
    };
    KdGate g;
    g.max_d2 = max_distance * max_distance;
    g.g2 = up(g.max_d2 * (1.0 + 0x1p-20) + 0x1p-126);
    g.dmax = up(max_distance);
    return g;
}

void kdmap_batch_iterations(pls_context* lead, int num, cudaStream_t st, const int* grid, int first, int last,
                            double max_distance, double min_eigenvalue, double* degen) {
    const KdSeq* seqs = lead->batch_buf.as<KdSeq>();
    // the thresholded solve runs in the gated kernels; at max_distance = +inf their gate (kd_gate_of: every bound +inf)
    // keeps every match, and matches exactly as the ungated search
    const bool thresholded = min_eigenvalue > 0.0;
    const KdGate g = kd_gate_of(isinf(max_distance) && !thresholded ? 0.0 : max_distance);
    const KdGate* gate = isinf(max_distance) && !thresholded ? nullptr : &g;
    for (int it = first; it < last; ++it) {
        if (it > 0 && grid[4]) {
            if (thresholded)
                kd_icp_refine_gated_degen_batch_kernel<<<dim3(grid[0], num), KD_REFINE_THREADS, 0, st>>>(
                    seqs, it, *gate, min_eigenvalue, degen);
            else if (gate) kd_icp_refine_gated_batch_kernel<<<dim3(grid[0], num), KD_REFINE_THREADS, 0, st>>>(seqs, it, *gate);
            else kd_icp_refine_batch_kernel<<<dim3(grid[0], num), KD_REFINE_THREADS, 0, st>>>(seqs, it);
            PLS_CHECK_LAUNCH();
        }
        if (it > 0 && !grid[3]) continue;
        if (it > 0) {
            if (gate) kd_nn_verify_gated_batch_kernel<<<dim3(grid[3], num), KD_THREADS, 0, st>>>(seqs, it, *gate);
            else kd_nn_verify_batch_kernel<<<dim3(grid[3], num), KD_THREADS, 0, st>>>(seqs, it);
            PLS_CHECK_LAUNCH();
        }
        batch_search(seqs, num, st, grid, it, gate);
        if (thresholded)
            kd_residual_gated_degen_batch_kernel<<<dim3(grid[0], num), KD_THREADS, 0, st>>>(seqs, it, gate->max_d2,
                                                                                          min_eigenvalue, degen);
        else if (gate) kd_residual_gated_batch_kernel<<<dim3(grid[0], num), KD_THREADS, 0, st>>>(seqs, it, gate->max_d2);
        else kd_residual_batch_kernel<<<dim3(grid[0], num), KD_THREADS, 0, st>>>(seqs, it);
        PLS_CHECK_LAUNCH();
    }
}

// pls_kdmap_evaluate_poses: iteration 0's search of the registrations kdmap_hypotheses_begin described (started at
// their poses), then their gated residual pass and their rows into out [num, PLS_EVAL_STATS] (device), on st.
void kdmap_evaluate_batch(pls_context* ctx, int num, cudaStream_t st, const int* grid, double max_d2, double* out) {
    const KdSeq* seqs = ctx->batch_buf.as<KdSeq>();
    batch_search(seqs, num, st, grid, 0);
    kd_evaluate_batch_kernel<<<dim3(grid[0], num), KD_THREADS, 0, st>>>(seqs, max_d2);
    PLS_CHECK_LAUNCH();
    kd_evaluate_finish_kernel<<<num, 256, 0, st>>>(seqs, out);
    PLS_CHECK_LAUNCH();
}

// pls_register_hypotheses / pls_register_scans: the ICP state of `num` registrations on ctx's map, registration h of
// scans[h], each a slice of ctx->hyp_buf laid out as pls_register_frame's own buffers for that scan's query bound; their
// descriptors into ctx->batch_buf.  Returns the registrations' FrameResults (contiguous) and their 16 counter and
// work-list words each, for the caller to initialise before the first iteration; grid as kdmap_batch_begin.
void kdmap_hypotheses_begin(pls_context* ctx, const KdScan* scans, int num, cudaStream_t st, int* grid, FrameResult** frs,
                            uint32_t** words) {
    PLS_REQUIRE(ctx->kd.valid, "kd map: search before any update");
    static const int resident_nn = resident_blocks((const void*)kd_nn_warp_batch_kernel);
    static const int resident_kn = resident_blocks((const void*)kd_normals_warp_batch_kernel);
    ctx->last_sharded = false;
    record_search(ctx->kd, true, false, true, 0);
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t fr_bytes = up((size_t)num * sizeof(FrameResult)), word_bytes = up((size_t)num * 16 * sizeof(uint32_t));
    // each plan also reserves ctx's own buffers for its bound: the last registration is copied there
    std::vector<KdPlan> plans;
    std::vector<size_t> offs;
    size_t total = fr_bytes + word_bytes;
    for (int h = 0; h < num; ++h) {
        plans.push_back(plan_kd_iteration(ctx, scans[h].bound, 1));
        const KdPlan& p = plans.back();
        offs.push_back(total);
        // partial rows wide enough for pls_kdmap_evaluate_poses's (PLS_EVAL_STATS >= NACC)
        total += up((size_t)scans[h].bound * sizeof(int)) + up(p.slots * sizeof(float4)) + up(2 * p.slots * sizeof(int)) +
                 up((size_t)p.blocks * PLS_EVAL_STATS * sizeof(double));
    }
    ctx->hyp_buf.reserve(total, st);
    char* base = ctx->hyp_buf.as<char>();
    *frs = reinterpret_cast<FrameResult*>(base);
    *words = reinterpret_cast<uint32_t*>(base + fr_bytes);
    const int share_nn = (resident_nn + num - 1) / num, share_kn = (resident_kn + num - 1) / num;
    std::vector<KdSeq> seqs;
    for (int h = 0; h < num; ++h) {
        const KdPlan& p = plans[(size_t)h];
        char* match = base + offs[(size_t)h];
        char* state = match + up((size_t)scans[h].bound * sizeof(int));
        char* list = state + up(p.slots * sizeof(float4));
        char* part = list + up(2 * p.slots * sizeof(int));
        seqs.push_back(make_seq(ctx, p, scans[h].queries, *frs + h, scans[h].nq_dev, reinterpret_cast<int*>(match),
                                reinterpret_cast<float4*>(state), reinterpret_cast<int*>(list), *words + 16 * h,
                                reinterpret_cast<double*>(part), share_nn, share_kn));
    }
    upload_seqs(ctx, seqs, st, grid);
}

// Registration h's matches, search states and FrameResult (all but the counts) into ctx's own, and its scan's query
// count and queries: pls_kdmap_last_correspondences and pls_last_icp_sums then read that registration as the last search.
void kdmap_hypothesis_adopt(pls_context* ctx, const KdScan& scan, int h, cudaStream_t st) {
    KdSeq s;
    PLS_CUDA(cudaMemcpyAsync(&s, ctx->batch_buf.as<KdSeq>() + h, sizeof(KdSeq), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_CUDA(cudaMemcpyAsync(ctx->nn_prev.p, s.match, (size_t)scan.bound * sizeof(int), cudaMemcpyDeviceToDevice, st));
    PLS_CUDA(cudaMemcpyAsync(ctx->kd_nn_state.p, s.nn_state, (size_t)scan.bound * sizeof(float4), cudaMemcpyDeviceToDevice,
                             st));
    FrameResult* fr = frame_result_dev(ctx);
    PLS_CUDA(cudaMemcpyAsync(fr, s.fr, offsetof(FrameResult, counts), cudaMemcpyDeviceToDevice, st));
    uint32_t* nq = reinterpret_cast<uint32_t*>(&fr->counts[1]);
    if (scan.nq_dev != nq) PLS_CUDA(cudaMemcpyAsync(nq, scan.nq_dev, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    ctx->query_ptr = scan.queries;
}

// The done flag of every sequence of the batch: one gather launch, one copy, one synchronisation.
void kdmap_batch_done(pls_context* lead, int num, cudaStream_t st, int* out) {
    int* dev = reinterpret_cast<int*>(lead->batch_buf.as<char>() + (size_t)num * sizeof(KdSeq));
    kd_batch_done_kernel<<<1, 64, 0, st>>>(lead->batch_buf.as<KdSeq>(), num, dev);
    PLS_CHECK_LAUNCH();
    PLS_CUDA(cudaMemcpyAsync(out, dev, (size_t)num * sizeof(int), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));
}

}  // namespace pls

using namespace pls;

extern "C" {

int pls_kdmap_update_points(pls_context* ctx, const float* rel_pose, const float* points, int64_t n) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(rel_pose, "pls_kdmap_update_points: rel_pose required");
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, "context holds a projective map");
    float rel[16];
    if (is_device_ptr(rel_pose)) PLS_CUDA(cudaMemcpy(rel, rel_pose, sizeof(rel), cudaMemcpyDeviceToHost));
    else memcpy(rel, rel_pose, sizeof(rel));
    const float* d = (points && n > 0) ? (const float*)to_device(ctx, points, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]) : nullptr;
    kdmap_update(ctx, rel, d, d ? n : 0, nullptr, 0, 0, -1);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_kdmap_set_points(pls_context* ctx, const void* xyz, int is_f64, int64_t n) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, "context holds a projective map");
    PLS_REQUIRE(n >= 0 && (xyz || n == 0), "pls_kdmap_set_points: points must be [n,3] with n >= 0");
    PLS_REQUIRE(n < (1ll << 30), "kd map: too many points");
    sync_all(ctx);
    cudaStream_t st = ctx->stream;
    const size_t elem = is_f64 ? sizeof(double) : sizeof(float);
    const void* d = n > 0 ? to_device(ctx, xyz, (size_t)n * 3 * elem, ctx->stage_in[0]) : nullptr;
    if (n > 0) {  // every row must be searchable: checked before the map changes
        uint32_t* bad = scalar_u32(ctx, SC_SPARE0);
        PLS_CUDA(cudaMemsetAsync(bad, 0, sizeof(uint32_t), st));
        const int g = grid_for(n, 256, 8 * kNumSMs);
        if (is_f64) kd_nonfinite_rows_kernel<double><<<g, 256, 0, st>>>((const double*)d, n, bad);
        else kd_nonfinite_rows_kernel<float><<<g, 256, 0, st>>>((const float*)d, n, bad);
        PLS_CHECK_LAUNCH();
        uint32_t nbad = 0;
        PLS_CUDA(cudaMemcpyAsync(&nbad, bad, sizeof(nbad), cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        PLS_REQUIRE(nbad == 0, "pls_kdmap_set_points: the cloud has rows with a NaN or infinite coordinate, which the "
                               "kd map cannot search");
    }
    kdmap_reset(ctx);
    if (n > 0) {
        // no row is dropped (all are finite): the packers give the rows in order, as float4
        ctx->tmp[4].reserve((size_t)n * sizeof(float4), st);
        if (is_f64) pack_valid_rows_f64(ctx, (const double*)d, n, ctx->tmp[4].as<float4>(), scalar_u32(ctx, SC_INSERT_COUNT));
        else pack_valid_rows(ctx, (const float*)d, n, ctx->tmp[4].as<float4>(), scalar_u32(ctx, SC_INSERT_COUNT));
    }
    // the map's first insertion (identity, nothing to move or evict) ...
    kdmap_update_packed(ctx, nullptr, ctx->tmp[4].as<float4>(), n, true);
    // ... held as no frame: the frames inserted later count from the first update on, and the steady-state capacity
    // plan follows them, not the cloud
    ctx->kd.frame_counts.clear();
    ctx->kd.max_frame = 0;
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_API_END(ctx)
}

int pls_kdmap_frames(pls_context* ctx, int64_t* out_counts, int* out_num) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(out_num, "pls_kdmap_frames: null output");
    const std::deque<int64_t>& fc = ctx->kd.frame_counts;
    *out_num = (int)fc.size();
    if (out_counts)
        for (size_t i = 0; i < fc.size(); ++i) out_counts[i] = fc[i];
    PLS_API_END(ctx)
}

int pls_kdmap_update_vertex_map(pls_context* ctx, const float* rel_pose, const float* vertex_map, int height, int width) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(rel_pose && vertex_map && height > 0 && width > 0, "pls_kdmap_update_vertex_map: bad arguments");
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_KDTREE, "context holds a projective map");
    float rel[16];
    if (is_device_ptr(rel_pose)) PLS_CUDA(cudaMemcpy(rel, rel_pose, sizeof(rel), cudaMemcpyDeviceToHost));
    else memcpy(rel, rel_pose, sizeof(rel));
    const float* d = (const float*)to_device(ctx, vertex_map, (size_t)3 * height * width * sizeof(float), ctx->stage_in[0]);
    kdmap_update(ctx, rel, nullptr, 0, d, height, width, -1);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_kdmap_stats(pls_context* ctx, unsigned long long* out16) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(out16, "pls_kdmap_stats: null output");
    memset(out16, 0, 16 * sizeof(unsigned long long));
    if (ctx->kd.stats.p) {
        PLS_CUDA(cudaMemcpyAsync(out16, ctx->kd.stats.p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
        PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    PLS_API_END(ctx)
}

int pls_kdmap_size(pls_context* ctx, int64_t* num_points) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(num_points, "pls_kdmap_size: null output");
    *num_points = ctx->kd.count;
    PLS_API_END(ctx)
}

int pls_kdmap_points(pls_context* ctx, float* out) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(out, "pls_kdmap_points: null output");
    const int64_t M = ctx->kd.count;
    if (M > 0) {
        OutArg o = out_arg(ctx, out, (size_t)M * 3 * sizeof(float), ctx->stage_out[0]);
        kd_export_kernel<<<grid_for(M, 256, 8 * kNumSMs), 256, 0, ctx->stream>>>(ctx->kd.store[ctx->kd.cur].as<float4>(), M,
                                                                                 (float*)o.dev);
        PLS_CHECK_LAUNCH();
        finish_out(ctx, o);
        PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    PLS_API_END(ctx)
}

int pls_kdmap_nn_search(pls_context* ctx, const float* queries, int64_t n, float* out_neighbors, float* out_normals,
                        int64_t* out_idx) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(queries && out_neighbors && n > 0, "pls_kdmap_nn_search: bad arguments");
    if (!ctx->kd.valid) throw pls::Error{PLS_E_STATE, "pls_kdmap_nn_search: the map is empty"};
    const float* d = (const float*)to_device(ctx, queries, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    OutArg onb = out_arg(ctx, out_neighbors, (size_t)n * 3 * sizeof(float), ctx->stage_out[0]);
    OutArg onr = out_arg(ctx, out_normals, (size_t)n * 3 * sizeof(float), ctx->stage_out[1]);
    OutArg oix = out_arg(ctx, out_idx, (size_t)n * sizeof(int64_t), ctx->stage_out[2]);
    // the same warp-cooperative kernels as the ICP loop, with an identity transform and no previous matches
    cudaStream_t st = ctx->stream;
    ctx->queries.reserve((size_t)n * sizeof(float4), st);
    ctx->tmp[6].reserve(16 * sizeof(float) + 16, st);
    static const float eye12[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    PLS_CUDA(cudaMemcpyAsync(ctx->tmp[6].p, eye12, sizeof(eye12), cudaMemcpyHostToDevice, st));
    uint32_t* nq = scalar_u32(ctx, SC_QUERY_COUNT);
    const uint32_t nq_host[3] = {(uint32_t)n, 0u, 0u};
    PLS_CUDA(cudaMemcpyAsync(nq, nq_host, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    PLS_CUDA(cudaMemsetAsync(scalar_u32(ctx, SC_KD_LISTS), 0, 8 * sizeof(uint32_t), st));
    kd_rows_to_float4_kernel<<<grid_for(n, 256, 8 * kNumSMs), 256, 0, st>>>(d, n, ctx->queries.as<float4>());
    PLS_CHECK_LAUNCH();
    const KdIndex ix = make_index(ctx);
    const KdPlan plan = plan_kd_iteration(ctx, n, 1);
    launch_search(ctx, plan, ix, ctx->queries.as<float4>(), nq, 0, 1, ctx->tmp[6].as<float>(), nullptr, ctx->nn_prev.as<int>(),
                  true, out_normals != nullptr, 0);
    record_search(ctx->kd, false, false, out_normals != nullptr, n);
    kd_search_export_kernel<<<grid_for(n, 256, 8 * kNumSMs), 256, 0, st>>>(ix, ctx->nn_prev.as<int>(), n, (float*)onb.dev,
                                                                            (float*)onr.dev, (long long*)oix.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, onb);
    finish_out(ctx, onr);
    finish_out(ctx, oix);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_kdmap_knn(pls_context* ctx, const float* queries, int64_t n, int k, int64_t* out_idx, float* out_d2,
                  int32_t* out_pos) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(queries && out_idx && out_d2 && n > 0, "pls_kdmap_knn: bad arguments");
    PLS_REQUIRE(k >= 0 && k + 1 <= KD_KMAX_WIDE, "pls_kdmap_knn: k must be in [0, 255]");
    if (!ctx->kd.valid) throw pls::Error{PLS_E_STATE, "pls_kdmap_knn: the map is empty"};
    const int K = k + 1;
    const size_t entries = (size_t)n * K;
    const float* d = (const float*)to_device(ctx, queries, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    OutArg oix = out_arg(ctx, out_idx, entries * sizeof(int64_t), ctx->stage_out[0]);
    OutArg od2 = out_arg(ctx, out_d2, entries * sizeof(float), ctx->stage_out[1]);
    OutArg ops = out_arg(ctx, out_pos, entries * sizeof(int32_t), ctx->stage_out[2]);
    const int blocks = grid_for(n, KD_THREADS / 32, 8 * kNumSMs);
    const KdIndex ix = make_index(ctx);
    long long* pi = (long long*)oix.dev;
    float* pd = (float*)od2.dev;
    int* pp = (int*)ops.dev;
    cudaStream_t st = ctx->stream;
    if (K <= KD_KMAX) kd_knn_export_kernel<<<blocks, KD_THREADS, 0, st>>>(ix, d, n, K, pi, pd, pp);
    else if (kd_wide_regs(K) == 2) kd_knn_wide_export_kernel<2><<<blocks, KD_THREADS, 0, st>>>(ix, d, n, K, pi, pd, pp);
    else if (kd_wide_regs(K) == 4) kd_knn_wide_export_kernel<4><<<blocks, KD_THREADS, 0, st>>>(ix, d, n, K, pi, pd, pp);
    else kd_knn_wide_export_kernel<8><<<blocks, KD_THREADS, 0, st>>>(ix, d, n, K, pi, pd, pp);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, oix);
    finish_out(ctx, od2);
    finish_out(ctx, ops);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

// A read-only look at the last search.  PLS_API_BEGIN_FRAME: a pending map update stays pending -- flushing it would
// rebuild the index the stored positions refer to.
int pls_kdmap_last_correspondences(pls_context* ctx, int64_t n, int64_t* out_idx, float* out_neighbors, float* out_normals,
                                   float* out_search_state, double* out_sums) {
    PLS_API_BEGIN_FRAME(ctx)
    const KdMap& kd = ctx->kd;
    if (!kd.searched) throw pls::Error{PLS_E_STATE, "pls_kdmap_last_correspondences: no kd search has run"};
    // the search ran on the current index, or on the one the frame's own device-decided update has since replaced
    // (its sorted points are kept in sorted_prev; the normals are only rewritten by the next search)
    const bool current = kd.valid && kd.searched_gen == kd.gen;
    const bool replaced = kd.prev_gen != 0 && kd.searched_gen == kd.prev_gen;
    if (!current && !replaced)
        throw pls::Error{PLS_E_STATE, "pls_kdmap_last_correspondences: the map was rebuilt since the last search"};
    if (kd.searched_sharded)
        throw pls::Error{PLS_E_STATE, "pls_kdmap_last_correspondences: the last ICP split its queries over the ranks"};
    cudaStream_t st = ctx->stream;
    int64_t count = kd.searched_n;
    if (kd.searched_icp) {
        long long c = 0;
        PLS_CUDA(cudaMemcpyAsync(&c, &frame_result_dev(ctx)->counts[1], sizeof(c), cudaMemcpyDeviceToHost, st));
        PLS_CUDA(cudaStreamSynchronize(st));
        count = (int64_t)c;
    }
    PLS_REQUIRE(n == count, "pls_kdmap_last_correspondences: n must be the query count of the last search");
    if (n > 0 && (out_idx || out_neighbors || out_normals)) {
        OutArg onb = out_arg(ctx, out_neighbors, (size_t)n * 3 * sizeof(float), ctx->stage_out[0]);
        OutArg onr = out_arg(ctx, out_normals, (size_t)n * 3 * sizeof(float), ctx->stage_out[1]);
        OutArg oix = out_arg(ctx, out_idx, (size_t)n * sizeof(int64_t), ctx->stage_out[2]);
        float* nb = (float*)onb.dev;
        if (!nb) {  // the export always writes the neighbours
            ctx->stage_out[3].reserve((size_t)n * 3 * sizeof(float), st);
            nb = ctx->stage_out[3].as<float>();
        }
        KdIndex ix = make_index(ctx);
        if (!current) ix.sorted = kd.sorted_prev.as<float4>();
        kd_search_export_kernel<<<grid_for(n, 256, 8 * kNumSMs), 256, 0, st>>>(
            ix, ctx->nn_prev.as<int>(), n, nb, kd.searched_normals ? (float*)onr.dev : nullptr,
            (long long*)oix.dev);
        PLS_CHECK_LAUNCH();
        if (onr.dev && !kd.searched_normals)  // the search computed no normals: NaN
            PLS_CUDA(cudaMemsetAsync(onr.dev, 0xff, onr.bytes, st));
        finish_out(ctx, onb);
        finish_out(ctx, onr);
        finish_out(ctx, oix);
    }
    if (n > 0 && out_search_state)
        PLS_CUDA(cudaMemcpyAsync(out_search_state, ctx->kd_nn_state.p, (size_t)n * sizeof(float4), cudaMemcpyDefault, st));
    if (out_sums) {
        if (kd.searched_icp) {
            PLS_CUDA(cudaMemcpyAsync(out_sums, frame_result_dev(ctx)->last_sums, NACC * sizeof(double), cudaMemcpyDefault, st));
        } else {
            PLS_CUDA(cudaStreamSynchronize(st));
            if (is_device_ptr(out_sums)) PLS_CUDA(cudaMemsetAsync(out_sums, 0xff, NACC * sizeof(double), st));
            else memset(out_sums, 0xff, NACC * sizeof(double));
        }
    }
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_API_END(ctx)
}

#ifdef PLS_KD_SPLIT
// Development builds only: copies the stamp records (KD_SPLIT_WORDS words, then the normals kernel's end) to `out`
// and clears them.  `words` must be KD_SPLIT_WORDS + 1.
PLS_API int pls_debug_kd_split(pls_context* ctx, unsigned long long* out, int64_t words) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(out && words == (int64_t)KD_SPLIT_WORDS + 1, "pls_debug_kd_split: bad arguments");
    sync_all(ctx);
    PLS_CUDA(cudaMemcpyFromSymbol(out, g_kd_split, KD_SPLIT_WORDS * sizeof(unsigned long long)));
    PLS_CUDA(cudaMemcpyFromSymbol(out + KD_SPLIT_WORDS, g_kd_split_normals_end, sizeof(unsigned long long)));
    static const unsigned long long zero = 0;
    void* p = nullptr;
    PLS_CUDA(cudaGetSymbolAddress(&p, g_kd_split));
    PLS_CUDA(cudaMemset(p, 0, KD_SPLIT_WORDS * sizeof(unsigned long long)));
    PLS_CUDA(cudaMemcpyToSymbol(g_kd_split_normals_end, &zero, sizeof(zero)));
    PLS_API_END(ctx)
}
#endif

}  // extern "C"
