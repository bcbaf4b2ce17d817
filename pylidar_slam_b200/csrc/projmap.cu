// K3/K4 -- the projective local map (replaces ProjectiveLocalMap, slam/odometry/local_map.py:91-240,
// compute_normal_map and compute_neighbors, slam/common/geometry.py:240-295,397-439).
//
//   normal_map_kernel       5x5 (k x k) zero-padded box sums of v and v v^T from a shared-memory
//                           tile, n ~ (sum v v^T)^-1 sum v through the cofactor matrix, float32
//   model_zbuf_kernel       build_model (local_map.py:177-202): every stored frame k is re-expressed
//   model_resolve_kernel    in the newest frame (p' = R_k v + t_k, n' = R_k n, masked) and re-projected
//                           with its own closest-wins z-buffer into _model_vmap / _model_nmap [K,3,H,W]
//   query_zbuf_kernel       nearest_neighbor_search (local_map.py:205-235): the transformed queries
//                           are z-buffered into the target vertex map (one survivor per pixel)
//   proj_icp_iter_kernel    per pixel: argmin_k |p - v_k| over the K model maps (first minimum wins,
//                           null candidates skipped), gather the winner's point and normal, point-to-
//                           plane residual / Jacobian / weight and the block-reduced normal equations.
//                           Streams HW*12*(K+1) bytes per launch: the HBM-bound correspondence kernel.
//   proj_pairs_kernel       the same association materialised per pixel for the fine-grained API
#include <stdlib.h>

#include "gn_device.cuh"
#include "icp_device.cuh"
#include "internal.cuh"
#include "pose_device.cuh"
#include "projection_device.cuh"

namespace pls {

namespace {

inline int grid_for(int64_t n, int threads, int cap_blocks = 16 * kNumSMs) {
    int64_t b = (n + threads - 1) / threads;
    return (int)(b < 1 ? 1 : (b > cap_blocks ? cap_blocks : b));
}

// ------------------------------------------------------------------------------------------ K3
constexpr int NM_TX = 32, NM_TY = 8, NM_MAXR = 4;  // kernel sizes up to 9

__global__ void __launch_bounds__(NM_TX* NM_TY)
normal_map_kernel(const float* __restrict__ vmap, int batch, int H, int W, int ksize, float* __restrict__ out) {
    __shared__ float tile[3][NM_TY + 2 * NM_MAXR][NM_TX + 2 * NM_MAXR + 1];
    const int r = ksize / 2;
    const int b = blockIdx.z;
    const int x0 = blockIdx.x * NM_TX, y0 = blockIdx.y * NM_TY;
    const int64_t hw = (int64_t)H * W;
    const float* v = vmap + (size_t)b * 3 * hw;
    const int tw = NM_TX + 2 * r, th = NM_TY + 2 * r;
    for (int i = threadIdx.y * NM_TX + threadIdx.x; i < tw * th; i += NM_TX * NM_TY) {
        int ty = i / tw, tx = i - ty * tw;
        int gx = x0 + tx - r, gy = y0 + ty - r;
        bool in = gx >= 0 && gx < W && gy >= 0 && gy < H;
        int64_t g = (int64_t)gy * W + gx;
        tile[0][ty][tx] = in ? v[g] : 0.f;
        tile[1][ty][tx] = in ? v[hw + g] : 0.f;
        tile[2][ty][tx] = in ? v[2 * hw + g] : 0.f;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= W || y >= H) return;
    // Operation order and rounding follow the reference exactly (its normals are dominated by float32
    // rounding: it inverts the UNCENTRED second-moment matrix, cond ~ r^2/sigma^2 >> 1/eps, so only a
    // bit-faithful evaluation reproduces them):
    //  * box sums = sequential float32 adds over the window, rows outer / columns inner, of separately
    //    rounded products (conv2d with a ones kernel over `v` and `v v^T`, geometry.py:258-268)
    float sx = 0.f, sy = 0.f, sz = 0.f, sxx = 0.f, sxy = 0.f, sxz = 0.f, syy = 0.f, syz = 0.f, szz = 0.f;
    for (int dy = 0; dy < ksize; ++dy)
        for (int dx = 0; dx < ksize; ++dx) {
            const float px = tile[0][threadIdx.y + dy][threadIdx.x + dx];
            const float py = tile[1][threadIdx.y + dy][threadIdx.x + dx];
            const float pz = tile[2][threadIdx.y + dy][threadIdx.x + dx];
            sx = __fadd_rn(sx, px); sy = __fadd_rn(sy, py); sz = __fadd_rn(sz, pz);
            sxx = __fadd_rn(sxx, __fmul_rn(px, px)); sxy = __fadd_rn(sxy, __fmul_rn(px, py));
            sxz = __fadd_rn(sxz, __fmul_rn(px, pz)); syy = __fadd_rn(syy, __fmul_rn(py, py));
            syz = __fadd_rn(syz, __fmul_rn(py, pz)); szz = __fadd_rn(szz, __fmul_rn(pz, pz));
        }
    //  * cofactor rows c_i = A[i-2] x A[i-1], each component fma(a1, b2, -(a2 * b1))  (geometry.py:65-76)
    const float A0[3] = {sxx, sxy, sxz}, A1[3] = {sxy, syy, syz}, A2[3] = {sxz, syz, szz};
    auto cross = [](const float* a, const float* b, float* c) {
        c[0] = __fmaf_rn(a[1], b[2], -__fmul_rn(a[2], b[1]));
        c[1] = __fmaf_rn(a[2], b[0], -__fmul_rn(a[0], b[2]));
        c[2] = __fmaf_rn(a[0], b[1], -__fmul_rn(a[1], b[0]));
    };
    auto dot3 = [](float a0, float b0, float a1, float b1, float a2, float b2) {
        return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
    };
    float c0[3], c1[3], c2[3];
    cross(A1, A2, c0);
    cross(A2, A0, c1);
    cross(A0, A1, c2);
    //  * det = mean of the three row expansions, ((d0 + d1) + d2) / 3  (geometry.py:87)
    const float d0 = dot3(c0[0], A0[0], c0[1], A0[1], c0[2], A0[2]);
    const float d1 = dot3(c1[0], A1[0], c1[1], A1[1], c1[2], A1[2]);
    const float d2 = dot3(c2[0], A2[0], c2[1], A2[1], c2[2], A2[2]);
    const float det = __fdiv_rn(__fadd_rn(__fadd_rn(d0, d1), d2), 3.0f);
    float n[3] = {0.f, 0.f, 0.f};
    if (fabsf(det) > 1e-6f) {
        //  * n = (cof / det)^T b : n_i = sum_j (cof[j][i] / det) b_j  (geometry.py:89-114,273)
        n[0] = dot3(__fdiv_rn(c0[0], det), sx, __fdiv_rn(c1[0], det), sy, __fdiv_rn(c2[0], det), sz);
        n[1] = dot3(__fdiv_rn(c0[1], det), sx, __fdiv_rn(c1[1], det), sy, __fdiv_rn(c2[1], det), sz);
        n[2] = dot3(__fdiv_rn(c0[2], det), sx, __fdiv_rn(c1[2], det), sy, __fdiv_rn(c2[2], det), sz);
        //  * norm = sqrt(fma(n2, n2, fma(n1, n1, n0 * n0)))  (torch.norm's vectorised kernel)
        float nn = __fsqrt_rn(__fmaf_rn(n[2], n[2], __fmaf_rn(n[1], n[1], __fmul_rn(n[0], n[0]))));
        if (nn == 0.f) nn = 1.f;
        n[0] = __fdiv_rn(n[0], nn); n[1] = __fdiv_rn(n[1], nn); n[2] = __fdiv_rn(n[2], nn);
    }
    const float cx = tile[0][threadIdx.y + r][threadIdx.x + r], cy = tile[1][threadIdx.y + r][threadIdx.x + r],
                cz = tile[2][threadIdx.y + r][threadIdx.x + r];
    if (cx == 0.f && cy == 0.f && cz == 0.f) n[0] = n[1] = n[2] = 0.f;  // torch.norm(vertex) == 0
    float* o = out + (size_t)b * 3 * hw + (int64_t)y * W + x;
    o[0] = n[0];
    o[hw] = n[1];
    o[2 * hw] = n[2];
}

// ------------------------------------------------------------------------------------------ model layout
// The re-projected model maps are stored TILE-INTERLEAVED in HBM: [tile = pix / 128][row = k * 3 + c][pix % 128]
// with a fixed tile stride of Kcap * 3 * 128 floats (Kcap = local_map_size).  All candidates of a 128-pixel
// tile are then ONE contiguous block (K * 3 * 512 bytes): a single TMA bulk copy per tile and a purely
// sequential HBM stream for the correspondence kernel.  The reference's planar [K,3,H,W] view exists only
// at the API boundary (pls_projmap_model converts).
constexpr int PT_TILE = 128;
__device__ __host__ __forceinline__ size_t model_off(int64_t pix, int row, int kcap) {
    return (size_t)(pix / PT_TILE) * ((size_t)kcap * 3 * PT_TILE) + (size_t)row * PT_TILE + (size_t)(pix % PT_TILE);
}
// The model NORMALS are only ever gathered for the winning candidate of a pixel, so they are stored as one
// float4 per (tile, k, pixel): the gather is a single 16-byte access (one 32-byte sector) instead of three.
__device__ __host__ __forceinline__ size_t normal_off(int64_t pix, int k, int kcap) {
    return ((size_t)(pix / PT_TILE) * kcap + (size_t)k) * PT_TILE + (size_t)(pix % PT_TILE);  // float4 units
}

// ------------------------------------------------------------------------------------------ model rebuild
struct PoseSet {
    const float* poses;  // [K][16] device
};

__device__ __forceinline__ bool model_point(const float* __restrict__ vmaps, const float* __restrict__ P, int64_t hw,
                                            int64_t src, float* p) {
    const float x = vmaps[src], y = vmaps[hw + src], z = vmaps[2 * hw + src];
    // mask_not_null (geometry.py:157-177): any channel non-zero
    if (fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f) {
        transform_point(P, make_float4(x, y, z, 0.f), p);
        return true;
    }
    return false;
}

// (a rank of a sharded job keeps only the pixels [pix_lo, pix_hi) of its own tiles)
__global__ void model_zbuf_kernel(const float* __restrict__ vmaps, const float* __restrict__ poses, int K, int head,
                                  int slots, ProjConst pc, int pix_lo, int pix_hi, unsigned long long* __restrict__ zbuf) {
    const int64_t hw = (int64_t)pc.H * pc.W;
    const int64_t total = (int64_t)K * hw;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = g / hw, src = g - k * hw;
        float p[3];
        if (!model_point(vmaps + (size_t)((head + k) % slots) * 3 * hw, poses + 16 * k, hw, src, p)) continue;
        int pix;
        float r;
        if (project_to_pixel(p[0], p[1], p[2], pc, pix, r, RangeOrder::kYFirst) && pix >= pix_lo && pix < pix_hi) {
            unsigned long long key = ((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)src;
            atomicMin(&zbuf[k * hw + pix], key);
        }
    }
}

__global__ void model_resolve_kernel(const float* __restrict__ vmaps, const float* __restrict__ nmaps,
                                     const float* __restrict__ poses, int K, int head, int slots, int kcap, int64_t hw,
                                     int64_t pix_lo, int64_t pix_hi, const unsigned long long* __restrict__ zbuf,
                                     float* __restrict__ model_v, float4* __restrict__ model_n) {
    const int64_t span = pix_hi - pix_lo, total = (int64_t)K * span;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = g / span, pix = pix_lo + (g - k * span);
        const unsigned long long key = zbuf[k * hw + pix];
        float p[3] = {0.f, 0.f, 0.f}, n[3] = {0.f, 0.f, 0.f};
        if (key != ~0ull) {
            const int64_t src = (int64_t)(uint32_t)(key & 0xffffffffull);
            const float* P = poses + 16 * k;
            const size_t slot = (size_t)((head + k) % slots);
            model_point(vmaps + slot * 3 * hw, P, hw, src, p);
            const float* nm = nmaps + slot * 3 * hw;
            const float nx = nm[src], ny = nm[hw + src], nz = nm[2 * hw + src];
            n[0] = P[0] * nx + P[1] * ny + P[2] * nz;
            n[1] = P[4] * nx + P[5] * ny + P[6] * nz;
            n[2] = P[8] * nx + P[9] * ny + P[10] * nz;
        }
        const size_t o = model_off(pix, (int)k * 3, kcap);
        model_v[o] = p[0]; model_v[o + PT_TILE] = p[1]; model_v[o + 2 * PT_TILE] = p[2];
        model_n[normal_off(pix, (int)k, kcap)] = make_float4(n[0], n[1], n[2], 0.f);
    }
}

// ------------------------------------------------------------------------------------------ search
__device__ __forceinline__ void load_T(const float* __restrict__ T, float* sT) {
    if (threadIdx.x < 12) sT[threadIdx.x] = T[threadIdx.x];
    __syncthreads();
}

// Query i, moved by the pose T (null: where it stands), into the closest-wins z-buffer of the pixels [pix_lo, pix_hi).
// Every query z-buffer (single, batched and per hypothesis) is built here, so they all get the same winners.
__device__ __forceinline__ void query_zbuf_insert(const float4& p0, int64_t i, const float* T, const ProjConst& pc, int pix_lo,
                                                  int pix_hi, unsigned long long* __restrict__ zbuf) {
    float p[3] = {p0.x, p0.y, p0.z};
    if (T) transform_point(T, p0, p);
    int pix;
    float r;
    // x first, unlike the other z-buffers: the order these z-buffers have always been built with
    if (project_to_pixel(p[0], p[1], p[2], pc, pix, r, RangeOrder::kXFirst) && pix >= pix_lo && pix < pix_hi) {
        unsigned long long key = ((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)i;
        atomicMin(&zbuf[pix], key);
    }
}

// The kernels of an ICP iteration below are __device__ bodies with two entry points each: the kernel of one sequence,
// which passes blockIdx.x / gridDim.x and its arguments, and the *_batch_kernel of pls_process_frames, whose blockIdx.y
// picks a sequence's descriptor (ProjSeq) and which passes that sequence's own block count.  A body reads no blockIdx.x
// or gridDim.x itself, so a sequence's striding, tile assignment and partial rows are those of its single path.
__device__ __forceinline__ void query_zbuf_body(const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev,
                                                int64_t nq_host, const float* __restrict__ T, const int* __restrict__ done,
                                                ProjConst pc, int pix_lo, int pix_hi, unsigned long long* __restrict__ zbuf,
                                                unsigned block, unsigned grid) {
    if (done && *done) return;
    __shared__ float sT[12];
    if (T) load_T(T, sT);
    const int64_t nq = nq_dev ? (int64_t)*nq_dev : nq_host;
    for (int64_t i = (int64_t)block * blockDim.x + threadIdx.x; i < nq; i += (int64_t)grid * blockDim.x)
        query_zbuf_insert(queries[i], i, T ? sT : nullptr, pc, pix_lo, pix_hi, zbuf);
}

__global__ void query_zbuf_kernel(const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev, int64_t nq_host,
                                  const float* __restrict__ T, const int* __restrict__ done, ProjConst pc, int pix_lo,
                                  int pix_hi, unsigned long long* __restrict__ zbuf) {
    query_zbuf_body(queries, nq_dev, nq_host, T, done, pc, pix_lo, pix_hi, zbuf, blockIdx.x, gridDim.x);
}

// z-buffer winners -> the target vertex map of this iteration, float4 (p transformed, valid flag) per pixel
__device__ __forceinline__ void query_resolve_body(unsigned long long* __restrict__ zbuf, const float4* __restrict__ queries,
                                                   const float* __restrict__ T, const int* __restrict__ done, int64_t pix_lo,
                                                   int64_t pix_hi, float4* __restrict__ tgt, unsigned block, unsigned grid) {
    if (done && *done) return;
    __shared__ float sT[12];
    load_T(T, sT);
    for (int64_t pix = pix_lo + (int64_t)block * blockDim.x + threadIdx.x; pix < pix_hi; pix += (int64_t)grid * blockDim.x) {
        const unsigned long long key = zbuf[pix];
        zbuf[pix] = ~0ull;  // leave the z-buffer cleared for the next iteration (no separate memset)
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        if (key != ~0ull) {
            float p[3];
            transform_point(sT, queries[(uint32_t)(key & 0xffffffffull)], p);
            o = make_float4(p[0], p[1], p[2], 1.f);
        }
        tgt[pix] = o;
    }
}

__global__ void query_resolve_kernel(unsigned long long* __restrict__ zbuf, const float4* __restrict__ queries,
                                     const float* __restrict__ T, const int* __restrict__ done, int64_t pix_lo,
                                     int64_t pix_hi, float4* __restrict__ tgt) {
    query_resolve_body(zbuf, queries, T, done, pix_lo, pix_hi, tgt, blockIdx.x, gridDim.x);
}

// Arg-min over distances WITHOUT the square roots in the common case.  The reference takes the arg-min over
// torch.norm (then torch.min keeps the first minimum: geometry.py:424-428), and two different squared distances can share
// one correctly rounded root -- but only if they lie within 2^-22 of each other (the pre-image of a float under sqrt is at
// most that wide, relatively).  The tile loop therefore compares squares against best2 * (1 - 2^-21), records whether any
// comparison fell inside that band, and redoes such a pixel (about one in 50 000) with the roots.

// acc += [ (wJ)(wJ)^T upper, (wJ)(wr), (wr)^2, r^2, 1 ] in float32: a thread of the tile-streaming kernel meets a
// handful of pixels only (tiles / CTAs), their sum goes to float64 before the block reduction -- each partial sum
// carries ~1e-7 relative rounding, the half-million-term totals stay far more accurate than the reference's float32
// sgemm while the accumulators cost 30 registers instead of 60
__device__ __forceinline__ void accumulate_normal_equations_f32(float* acc, const float* J, float w, float wr, float r) {
    float wj[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) wj[a] = J[a] * w;
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) acc[k++] += wj[a] * wj[b];
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += wj[a] * wr;
    acc[27] += wr * wr;
    acc[28] += r * r;
    acc[29] += 1.0f;
}

// argmin over the K candidates at one pixel; returns false if none is valid
__device__ __forceinline__ bool pixel_argmin(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K,
                                             int kcap, int64_t pix, const float* p, float* q, float* n) {
    float best = __int_as_float(0x7f800000);
    int kbest = -1;
    float bq[3] = {0.f, 0.f, 0.f};
    const float* mvb = model_v + model_off(pix, 0, kcap);
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
        const float* mv = mvb + (size_t)k * 3 * PT_TILE;
        const float x = mv[0], y = mv[PT_TILE], z = mv[2 * PT_TILE];
        if (fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f) {
            const float dx = p[0] - x, dy = p[1] - y, dz = p[2] - z;
            const float d = sqrtf(dx * dx + dy * dy + dz * dz);
            if (d < best) {  // torch.min keeps the first minimum
                best = d;
                kbest = k;
                bq[0] = x; bq[1] = y; bq[2] = z;
            }
        }
    }
    if (kbest < 0) return false;
    q[0] = bq[0]; q[1] = bq[1]; q[2] = bq[2];
    const float4 mn = model_n[normal_off(pix, kbest, kcap)];
    n[0] = mn.x; n[1] = mn.y; n[2] = mn.z;
    return true;
}

constexpr int PJ_THREADS = 256;

__global__ void __launch_bounds__(PJ_THREADS)
proj_icp_iter_kernel(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K, int kcap,
                     const unsigned long long* __restrict__ zbuf, const float4* __restrict__ queries,
                     const FrameResult* __restrict__ fr, int64_t pix_begin, int64_t pix_end, int scheme, float sigma,
                     double* __restrict__ partials) {
    if (fr->done) return;
    __shared__ float sT[12];
    load_T(fr->T, sT);
    double acc[NACC];
#pragma unroll
    for (int a = 0; a < NACC; ++a) acc[a] = 0.0;
    for (int64_t pix = pix_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < pix_end;
         pix += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = zbuf[pix];
        if (key == ~0ull) continue;
        float p[3], q[3], n[3];
        transform_point(sT, queries[(uint32_t)(key & 0xffffffffull)], p);
        if (!pixel_argmin(model_v, model_n, K, kcap, pix, p, q, n)) continue;
        float J[6];
        const float r = p2plane_residual_jacobian_identity(p, q, n, J);
        const float w = ls_weight<float>(scheme, sigma, r, p, q);
        accumulate_normal_equations<float>(acc, J, w, r * w, r);
    }
    block_reduce_store<PJ_THREADS>(acc, partials + (size_t)blockIdx.x * NACC);
}

// ---- TMA-staged variant ---------------------------------------------------------------------------
// Persistent CTAs (2 per SM); each loops over 128-pixel tiles.  For a tile, ONE thread issues K*3 bulk
// async copies (cp.async.bulk, the TMA engine; 512 contiguous bytes per candidate plane) that land in a
// [K*3][128] shared-memory stage and complete on that stage's mbarrier; 3 stages keep two tiles (up to
// 60 KB per CTA) in flight while the third is consumed, with no registers tied up by outstanding loads.
// The consumers (one thread per pixel) read conflict-free from shared memory.
constexpr int PT_STAGES = 3;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// L2 eviction-priority policies (the fixed encodings of createpolicy.fractional.L2::evict_last / evict_first, fraction 1)
constexpr unsigned long long L2_EVICT_LAST = 0x14F0000000000000ull, L2_EVICT_FIRST = 0x12F0000000000000ull;
__device__ __forceinline__ void bulk_copy_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, unsigned long long policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ float ldg_f32_hint(const float* p, unsigned long long policy) {
    float v;
    asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(policy));
    return v;
}
__device__ __forceinline__ float4 ldg_f4_hint(const float4* p, unsigned long long policy) {
    float4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(policy));
    return v;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}

__device__ __forceinline__ void
proj_icp_tma_body(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K, int kcap,
                  const float4* __restrict__ tgt, const FrameResult* __restrict__ fr, int64_t tile_begin, int64_t tile_end, int scheme, float sigma,
                  int stages, int ktma, int64_t resident_end, unsigned long long policy_resident,
                  unsigned long long policy_stream, double* __restrict__ partials, unsigned block, unsigned grid) {
    if (fr->done) return;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[PT_STAGES];
    float* stage_base = reinterpret_cast<float*>(smem_raw);
    // candidates [0, ktma) are staged through shared memory by the TMA engine; candidates [ktma, K) are read by
    // the consumers themselves with coalesced loads (the tile-interleaved rows are 512 contiguous bytes), issued
    // BEFORE the mbarrier wait: the LSU path and the TMA path pull from HBM concurrently
    const int rows = ktma * 3;
    const uint32_t model_bytes = (uint32_t)rows * PT_TILE * sizeof(float);
    const uint32_t stage_floats = (uint32_t)(rows + 4) * PT_TILE;  // + the tile of the target vertex map (float4 per pixel)
    const uint32_t stage_bytes = stage_floats * sizeof(float);
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) mbar_init(&full_bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int64_t first_tile = tile_begin + block;
    const int64_t stride = grid;
    auto issue = [&](int64_t tile, int s) {  // thread 0 only
        mbar_arrive_expect_tx(&full_bar[s], stage_bytes);
        // the tile's K*3 candidate rows are contiguous in the tile-interleaved layout: one bulk copy; a second
        // one brings the tile of the (z-buffered, already transformed) target vertex map
        // the same model is streamed once per ICP iteration: the tiles below `resident_end` ask L2 to keep them
        // (evict-last) and are served from L2 from the second iteration on; the rest passes through (evict-first)
        // without pushing them out
        float* dst = stage_base + (size_t)s * stage_floats;
        bulk_copy_g2s_hint(dst, model_v + (size_t)tile * ((size_t)kcap * 3 * PT_TILE), model_bytes, &full_bar[s],
                           tile < resident_end ? policy_resident : policy_stream);
        bulk_copy_g2s(dst + (size_t)rows * PT_TILE, tgt + tile * PT_TILE, PT_TILE * sizeof(float4), &full_bar[s]);
    };
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) {
            const int64_t t = first_tile + (int64_t)s * stride;
            if (t < tile_end) issue(t, s);
        }
    }
    float acc[NACC];
#pragma unroll
    for (int a = 0; a < NACC; ++a) acc[a] = 0.f;
    bool pend = false;
    float pp[3] = {0.f, 0.f, 0.f}, pq[3] = {0.f, 0.f, 0.f}, pn[3] = {0.f, 0.f, 0.f};
    int it = 0;
    for (int64_t tile = first_tile; tile < tile_end; tile += stride, ++it) {
        const int s = it % stages;
        const uint32_t parity = (uint32_t)((it / stages) & 1);
        const int64_t pix = tile * PT_TILE + threadIdx.x;
        constexpr int KDIRECT_MAX = 10;
        float dv[3 * KDIRECT_MAX];
        {
            const float* g = model_v + (size_t)tile * ((size_t)kcap * 3 * PT_TILE) + (size_t)ktma * 3 * PT_TILE + threadIdx.x;
            const unsigned long long policy = tile < resident_end ? policy_resident : policy_stream;
#pragma unroll
            for (int j = 0; j < 3 * KDIRECT_MAX; ++j)
                dv[j] = (j < (K - ktma) * 3) ? ldg_f32_hint(g + (size_t)j * PT_TILE, policy) : 0.f;
        }
        mbar_wait(&full_bar[s], parity);
        bool matched = false;
        float q[3] = {0.f, 0.f, 0.f};
        int kbest = -1;
        const float4 tp = reinterpret_cast<const float4*>(stage_base + (size_t)s * stage_floats + (size_t)rows * PT_TILE)[threadIdx.x];
        const float p[3] = {tp.x, tp.y, tp.z};
        const bool has = tp.w != 0.f;
        if (has) {
            const float* st = stage_base + (size_t)s * stage_floats + threadIdx.x;
            // Branch-free arg-min on squared distances.  `band` records whether any comparison fell inside the
            // 2^-22 band where the squares cannot decide (see above): the pixel is then redone with the roots.
            float best2 = __int_as_float(0x7f800000);  // squared distance of the best candidate so far
            bool band = false;
#pragma unroll 4
            for (int k = 0; k < ktma; ++k) {
                const float x = st[(3 * k) * PT_TILE], y = st[(3 * k + 1) * PT_TILE], z = st[(3 * k + 2) * PT_TILE];
                const float dx = p[0] - x, dy = p[1] - y, dz = p[2] - z;
                const float d2 = dx * dx + dy * dy + dz * dz;
                // torch.min keeps the first minimum; null candidates (all channels 0) do not compete
                const bool live = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f;
                const bool lt = live && d2 < best2 * 0.99999952f;
                band |= live && !lt && d2 < best2;
                best2 = lt ? d2 : best2;
                kbest = lt ? k : kbest;
                q[0] = lt ? x : q[0]; q[1] = lt ? y : q[1]; q[2] = lt ? z : q[2];
            }
#pragma unroll
            for (int j = 0; j < KDIRECT_MAX; ++j) {
                if (j < K - ktma) {
                    const float x = dv[3 * j], y = dv[3 * j + 1], z = dv[3 * j + 2];
                    const float dx = p[0] - x, dy = p[1] - y, dz = p[2] - z;
                    const float d2 = dx * dx + dy * dy + dz * dz;
                    const bool live = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f;
                    const bool lt = live && d2 < best2 * 0.99999952f;
                    band |= live && !lt && d2 < best2;
                    best2 = lt ? d2 : best2;
                    kbest = lt ? ktma + j : kbest;
                    q[0] = lt ? x : q[0]; q[1] = lt ? y : q[1]; q[2] = lt ? z : q[2];
                }
            }
            if (band) {  // about one pixel in 50 000: the reference's arg-min over the roots, first minimum wins
                float best = __int_as_float(0x7f800000);
                kbest = -1;
                for (int k = 0; k < K; ++k) {
                    float x, y, z;
                    if (k < ktma) {
                        x = st[(3 * k) * PT_TILE]; y = st[(3 * k + 1) * PT_TILE]; z = st[(3 * k + 2) * PT_TILE];
                    } else {
                        const float* gk = model_v + (size_t)tile * ((size_t)kcap * 3 * PT_TILE) + (size_t)k * 3 * PT_TILE + threadIdx.x;
                        x = __ldg(gk); y = __ldg(gk + PT_TILE); z = __ldg(gk + 2 * PT_TILE);
                    }
                    if (fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f) {
                        const float dx = p[0] - x, dy = p[1] - y, dz = p[2] - z;
                        const float d = sqrtf(dx * dx + dy * dy + dz * dz);
                        if (d < best) {
                            best = d;
                            kbest = k;
                            q[0] = x; q[1] = y; q[2] = z;
                        }
                    }
                }
            }
            matched = kbest >= 0;
        }
        __syncthreads();  // every consumer is done with stage s before the async proxy refills it
        if (threadIdx.x == 0) {
            const int64_t nt = tile + (int64_t)stages * stride;
            if (nt < tile_end) issue(nt, s);
        }
        // software pipeline: first consume the PREVIOUS tile's correspondence (its normal gather was issued
        // one iteration ago and has had this tile's wait + arg-min to land) ...
        if (pend) {
            float J[6];
            const float r = p2plane_residual_jacobian_identity(pp, pq, pn, J);
            const float w = ls_weight<float>(scheme, sigma, r, pp, pq);
            accumulate_normal_equations_f32(acc, J, w, r * w, r);
        }
        // ... then issue THIS tile's winner-normal gather straight into the pending registers (no copy that
        // would force the load to complete here)
        pend = matched;
        if (matched) {
            const float4 mn = ldg_f4_hint(model_n + normal_off(pix, kbest, kcap), policy_stream);  // one 16-byte gather, no reuse
            pn[0] = mn.x; pn[1] = mn.y; pn[2] = mn.z;
#pragma unroll
            for (int c = 0; c < 3; ++c) { pp[c] = p[c]; pq[c] = q[c]; }
        }
    }
    if (pend) {
        float J[6];
        const float r = p2plane_residual_jacobian_identity(pp, pq, pn, J);
        const float w = ls_weight<float>(scheme, sigma, r, pp, pq);
        accumulate_normal_equations_f32(acc, J, w, r * w, r);
    }
    double acc64[NACC];
#pragma unroll
    for (int a = 0; a < NACC; ++a) acc64[a] = (double)acc[a];
    block_reduce_store<PT_TILE>(acc64, partials + (size_t)block * NACC);
    // (the solve stays in icp_step_kernel: finishing the iteration in the CTA that arrives last, as kd_residual_kernel
    // does, was slower here)
}

__global__ void __launch_bounds__(PT_TILE)
proj_icp_tma_kernel(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K, int kcap,
                    const float4* __restrict__ tgt, const FrameResult* __restrict__ fr, int64_t tile_begin, int64_t tile_end, int scheme, float sigma,
                    int stages, int ktma, int64_t resident_end, unsigned long long policy_resident,
                    unsigned long long policy_stream, double* __restrict__ partials) {
    proj_icp_tma_body(model_v, model_n, K, kcap, tgt, fr, tile_begin, tile_end, scheme, sigma, stages, ktma, resident_end,
                      policy_resident, policy_stream, partials, blockIdx.x, gridDim.x);
}

// ---- many pose hypotheses of one scan (pls_register_hypotheses) -----------------------------------------------------
// Hypothesis h of a chunk owns FrameResult frs[h], the h-th hw-pixel slice of the query z-buffers `zbufs` and of the
// target maps `tgts`, and the h-th `part_rows`-double range of the partial rows; the scan's queries and the model are
// shared.  Every hypothesis's arithmetic is its single call's (projmap_icp_iteration), so it gets that call's bits.

// Each query is loaded once and z-buffered into the z-buffer of every live hypothesis, transformed by that hypothesis's
// pose.  The 64-bit atomic-min keys make every z-buffer the one its single call builds, whatever the order.
__global__ void __launch_bounds__(256)
query_zbuf_hyp_kernel(const float4* __restrict__ queries, const uint32_t* __restrict__ nq_dev,
                      const FrameResult* __restrict__ frs, int num, ProjConst pc, int64_t hw,
                      unsigned long long* __restrict__ zbufs) {
    __shared__ float sT[PLS_MAX_SEQUENCES][12];
    __shared__ int live[PLS_MAX_SEQUENCES];
    __shared__ int s_live;
    if (threadIdx.x == 0) {
        int c = 0;
        for (int h = 0; h < num; ++h)
            if (!frs[h].done) live[c++] = h;
        s_live = c;
    }
    __syncthreads();
    const int nl = s_live;
    if (nl == 0) return;
    for (int i = threadIdx.x; i < nl * 12; i += blockDim.x) sT[i / 12][i % 12] = frs[live[i / 12]].T[i % 12];
    __syncthreads();
    const int64_t nq = (int64_t)*nq_dev;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 p0 = queries[i];
        for (int j = 0; j < nl; ++j) query_zbuf_insert(p0, i, sT[j], pc, 0, (int)hw, zbufs + (size_t)live[j] * hw);
    }
}

// blockIdx.y = hypothesis: its z-buffer winners into its target map, leaving its z-buffer cleared.
__global__ void query_resolve_hyp_kernel(unsigned long long* __restrict__ zbufs, const float4* __restrict__ queries,
                                         const FrameResult* __restrict__ frs, int64_t hw, float4* __restrict__ tgts) {
    const int h = blockIdx.y;
    query_resolve_body(zbufs + (size_t)h * hw, queries, frs[h].T, &frs[h].done, 0, hw, tgts + (size_t)h * hw, blockIdx.x,
                       gridDim.x);
}

// The TMA kernel of every live hypothesis: proj_icp_tma_body on hypothesis h's target map, FrameResult and partial rows,
// as CTA `cta` of the single call's `blocks` (same tiles in the same order, same pixel per thread, same partial row), so
// each hypothesis's rows are its single call's by construction.  blockIdx.x = cta * num + h: the CTAs of all hypotheses
// that read one tile range are neighbours in the launch order, so they run in one wave and can share the model tiles
// through L2.  A done hypothesis's CTAs return at once (the body's own test), before any copy.
__global__ void __launch_bounds__(PT_TILE)
proj_icp_tma_hyp_kernel(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K, int kcap,
                        const float4* __restrict__ tgts, int64_t hw, const FrameResult* __restrict__ frs, int num,
                        int blocks, int64_t tiles, int scheme, float sigma, int stages, int ktma, int64_t resident_end,
                        double* __restrict__ partials, int64_t part_rows) {
    const int cta = (int)blockIdx.x / num, h = (int)blockIdx.x % num;
    proj_icp_tma_body(model_v, model_n, K, kcap, tgts + (size_t)h * hw, frs + h, 0, tiles, scheme, sigma, stages, ktma,
                      resident_end, L2_EVICT_LAST, L2_EVICT_FIRST, partials + (size_t)h * part_rows, cta, blocks);
}

// ---- several sequences per launch (pls_process_frames) --------------------------------------------------------------
// What the kernels of one ICP iteration need of one sequence: the arguments its single path passes (one rank: every
// tile and every pixel), and its share of each launch.  Built on the host by projmap_batch_begin and uploaded once per
// call.  A sequence that cannot take the TMA path has no blocks in the first three kernels: its correspondences run
// through its own launches (proj_icp_iter_kernel), and only the step kernel is shared.
struct ProjSeq {
    const float* model_v;
    const float4* model_n;
    const float4* queries;
    const uint32_t* nq_dev;     // query count (FrameResult counts[1])
    FrameResult* fr;            // pose, done flag
    unsigned long long* zbuf;   // the query z-buffer (tmp[3]), all-empty between iterations
    float4* tgt;                // the target vertex map of the iteration (tmp[7])
    double* partials;           // step_blocks rows
    ProjConst pc;
    int K, kcap, ktma, stages;
    int scheme;
    float sigma;
    float threshold_delta;
    int64_t tiles;              // hw / 128: the tile range [0, tiles)
    int64_t resident_end;       // tiles below it are read evict-last
    int zbuf_blocks, resolve_blocks, tma_blocks;  // the single path's geometry of each kernel (0: not launched)
    int step_blocks;            // partial rows the step sums: the TMA kernel's or proj_icp_iter_kernel's blocks
    int max_iters;              // max_num_alignments: launches of later iterations leave the sequence alone
};
static_assert(sizeof(ProjSeq) % sizeof(int) == 0, "ProjSeq is copied in 4-byte words");

// Sequence blockIdx.y's descriptor into shared memory, for every thread of the block.
__device__ __forceinline__ void load_seq(const ProjSeq* __restrict__ seqs, ProjSeq& s) {
    const int* src = reinterpret_cast<const int*>(seqs + blockIdx.y);
    int* dst = reinterpret_cast<int*>(&s);
    for (int i = threadIdx.x; i < (int)(sizeof(ProjSeq) / sizeof(int)); i += blockDim.x) dst[i] = __ldg(src + i);
    __syncthreads();
}

__global__ void query_zbuf_batch_kernel(const ProjSeq* __restrict__ seqs, int it) {
    __shared__ ProjSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.zbuf_blocks || it >= s.max_iters) return;
    query_zbuf_body(s.queries, s.nq_dev, 0, s.fr->T, &s.fr->done, s.pc, 0, (int)(s.tiles * PT_TILE), s.zbuf, blockIdx.x,
                    s.zbuf_blocks);
}

__global__ void query_resolve_batch_kernel(const ProjSeq* __restrict__ seqs, int it) {
    __shared__ ProjSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.resolve_blocks || it >= s.max_iters) return;
    query_resolve_body(s.zbuf, s.queries, s.fr->T, &s.fr->done, 0, s.tiles * PT_TILE, s.tgt, blockIdx.x, s.resolve_blocks);
}

__global__ void __launch_bounds__(PT_TILE) proj_icp_tma_batch_kernel(const ProjSeq* __restrict__ seqs, int it) {
    __shared__ ProjSeq s;
    load_seq(seqs, s);
    if ((int)blockIdx.x >= s.tma_blocks || it >= s.max_iters) return;
    proj_icp_tma_body(s.model_v, s.model_n, s.K, s.kcap, s.tgt, s.fr, 0, s.tiles, s.scheme, s.sigma, s.stages, s.ktma,
                      s.resident_end, L2_EVICT_LAST, L2_EVICT_FIRST, s.partials, blockIdx.x, s.tma_blocks);
}

// One block per sequence: the fixed-order sum of its own partial rows, the guards, the solve and the done latch.
__global__ void __launch_bounds__(256) icp_step_batch_kernel(const ProjSeq* __restrict__ seqs, int it) {
    __shared__ ProjSeq s;
    load_seq(seqs, s);
    if (it >= s.max_iters) return;
    icp_step_body(s.fr, s.partials, s.step_blocks, nullptr, s.threshold_delta);
}

// The done flags of every sequence, for the host's extra-round check.
__global__ void proj_batch_done_kernel(const ProjSeq* __restrict__ seqs, int num, int* __restrict__ out) {
    for (int i = threadIdx.x; i < num; i += blockDim.x) out[i] = seqs[i].fr->done;
}

// per-pixel association for the fine-grained API: flag + (q, n, p)
__global__ void proj_pairs_kernel(const float* __restrict__ model_v, const float4* __restrict__ model_n, int K, int kcap,
                                  int64_t hw, const unsigned long long* __restrict__ zbuf, const float4* __restrict__ queries,
                                  uint8_t* __restrict__ flags, float* __restrict__ pairs /* [hw][9] */) {
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < hw; pix += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = zbuf[pix];
        uint8_t ok = 0;
        if (key != ~0ull) {
            const float4 p0 = queries[(uint32_t)(key & 0xffffffffull)];
            float p[3] = {p0.x, p0.y, p0.z}, q[3], n[3];
            if (pixel_argmin(model_v, model_n, K, kcap, pix, p, q, n)) {
                ok = 1;
                float* o = pairs + 9 * pix;
                o[0] = q[0]; o[1] = q[1]; o[2] = q[2];
                o[3] = n[0]; o[4] = n[1]; o[5] = n[2];
                o[6] = p[0]; o[7] = p[1]; o[8] = p[2];
            }
        }
        flags[pix] = ok;
    }
}

__global__ void proj_compact_kernel(const uint8_t* __restrict__ flags, const uint32_t* __restrict__ pos,
                                    const float* __restrict__ pairs, int64_t hw, float* __restrict__ out_q,
                                    float* __restrict__ out_n, float* __restrict__ out_p) {
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < hw; pix += (int64_t)gridDim.x * blockDim.x) {
        if (!flags[pix]) continue;
        const uint32_t d = pos[pix];
        const float* s = pairs + 9 * pix;
        for (int c = 0; c < 3; ++c) {
            out_q[3 * (size_t)d + c] = s[c];
            if (out_n) out_n[3 * (size_t)d + c] = s[3 + c];
            if (out_p) out_p[3 * (size_t)d + c] = s[6 + c];
        }
    }
}

// stateless compute_neighbors (geometry.py:397-439)
__global__ void compute_neighbors_kernel(const float* __restrict__ tgt, const float* __restrict__ ref,
                                         const float* __restrict__ fields, int K, int C, int64_t hw,
                                         float* __restrict__ out_nb, float* __restrict__ out_f) {
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < hw; pix += (int64_t)gridDim.x * blockDim.x) {
        const float p[3] = {tgt[pix], tgt[hw + pix], tgt[2 * hw + pix]};
        const bool tgt_ok = fmaxf(fmaxf(fabsf(p[0]), fabsf(p[1])), fabsf(p[2])) > 0.f;
        float best = __int_as_float(0x7f800000);
        int kbest = 0;  // torch.min over all-inf returns index 0
        if (tgt_ok) {
            for (int k = 0; k < K; ++k) {
                const float* mv = ref + (size_t)k * 3 * hw + pix;
                const float x = mv[0], y = mv[hw], z = mv[2 * hw];
                if (fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z)) > 0.f) {
                    const float dx = p[0] - x, dy = p[1] - y, dz = p[2] - z;
                    const float d = sqrtf(dx * dx + dy * dy + dz * dz);
                    if (d < best) { best = d; kbest = k; }
                }
            }
        }
        const float* mv = ref + (size_t)kbest * 3 * hw + pix;
        out_nb[pix] = tgt_ok ? mv[0] : 0.f;
        out_nb[hw + pix] = tgt_ok ? mv[hw] : 0.f;
        out_nb[2 * hw + pix] = tgt_ok ? mv[2 * hw] : 0.f;
        if (fields)
            for (int c = 0; c < C; ++c) out_f[(size_t)c * hw + pix] = fields[((size_t)kbest * C + c) * hw + pix];
    }
}

// tile-interleaved -> the reference's planar [K,3,H,W]
__global__ void model_export_kernel(const float* __restrict__ tiled, int K, int kcap, int64_t hw, float* __restrict__ planar) {
    const int64_t total = (int64_t)K * 3 * hw;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = g / hw, pix = g - row * hw;
        planar[g] = tiled[model_off(pix, (int)row, kcap)];
    }
}

__global__ void normal_export_kernel(const float4* __restrict__ tiled, int K, int kcap, int64_t hw, float* __restrict__ planar) {
    const int64_t total = (int64_t)K * hw;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = g / hw, pix = g - k * hw;
        const float4 n = tiled[normal_off(pix, (int)k, kcap)];
        planar[(k * 3 + 0) * hw + pix] = n.x;
        planar[(k * 3 + 1) * hw + pix] = n.y;
        planar[(k * 3 + 2) * hw + pix] = n.z;
    }
}

// The pixel range of the model this rank needs: all of it, or -- when the ICP iterations of this job are split across
// ranks (icp_shards) and the TMA path applies -- the tiles the rank reduces (projmap_icp_iteration takes the same split).
void model_range(pls_context* ctx, bool full, int64_t* lo, int64_t* hi) {
    const int64_t hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
    *lo = 0;
    *hi = hw;
    if (full || hw % PT_TILE != 0 || !icp_shards(ctx, hw)) return;
    const int64_t tiles = hw / PT_TILE;
    const int rank = comm_rank(ctx), size = comm_size(ctx);
    *lo = (tiles * rank / size) * PT_TILE;
    *hi = (tiles * (rank + 1) / size) * PT_TILE;
}

void rebuild_model(pls_context* ctx, bool full = false) {
    ProjMap& pm = ctx->pm;
    cudaStream_t st = ctx->stream;
    const int H = ctx->cfg.height, W = ctx->cfg.width;
    const int64_t hw = (int64_t)H * W;
    const int K = pm.K;
    if (K == 0) return;
    int64_t lo, hi;
    model_range(ctx, full, &lo, &hi);
    ProfileScope ps(ctx, 2, (double)K * (hw * 24.0 + (hi - lo) * (24.0 + 16.0)));
    pm.poses.reserve((size_t)ctx->cfg.local_map_size * 16 * sizeof(float) + 64, st);
    PLS_CUDA(cudaMemcpyAsync(pm.poses.p, pm.host_poses.data(), (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
    pm.zbuf.reserve((size_t)(K > 1 ? K : 1) * hw * sizeof(unsigned long long), st);
    const int kcap = ctx->cfg.local_map_size;
    const size_t model_floats = (size_t)((hw + PT_TILE - 1) / PT_TILE) * kcap * 3 * PT_TILE;
    pm.model_v.reserve(model_floats * sizeof(float), st);
    pm.model_n.reserve((size_t)((hw + PT_TILE - 1) / PT_TILE) * kcap * PT_TILE * sizeof(float4), st);
    if (lo == 0 && hi == hw)
        PLS_CUDA(cudaMemsetAsync(pm.zbuf.p, 0xff, (size_t)K * hw * sizeof(unsigned long long), st));
    else  // only the rank's own pixel columns of each of the K z-buffers
        PLS_CUDA(cudaMemset2DAsync(pm.zbuf.as<unsigned long long>() + lo, (size_t)hw * sizeof(unsigned long long), 0xff,
                                   (size_t)(hi - lo) * sizeof(unsigned long long), (size_t)K, st));
    ProjConst pc = make_proj_const(H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
    const int slots = ctx->cfg.local_map_size + 1;
    model_zbuf_kernel<<<grid_for(K * hw, 256), 256, 0, st>>>(pm.vmaps.as<float>(), pm.poses.as<float>(), K, pm.head, slots,
                                                             pc, (int)lo, (int)hi, pm.zbuf.as<unsigned long long>());
    PLS_CHECK_LAUNCH();
    model_resolve_kernel<<<grid_for(K * (hi - lo), 256), 256, 0, st>>>(pm.vmaps.as<float>(), pm.nmaps.as<float>(),
                                                                       pm.poses.as<float>(), K, pm.head, slots, kcap, hw, lo, hi,
                                                                       pm.zbuf.as<unsigned long long>(),
                                                                       pm.model_v.as<float>(), pm.model_n.as<float4>());
    PLS_CHECK_LAUNCH();
    pm.valid = true;
    pm.built_lo = lo;
    pm.built_hi = hi;
}

// Callers that read the whole model (export, the stand-alone search) on a rank that built only its share.
void ensure_full_model(pls_context* ctx) {
    const int64_t hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
    if (ctx->pm.valid && (ctx->pm.built_lo != 0 || ctx->pm.built_hi != hw)) rebuild_model(ctx, true);
}

}  // namespace

void launch_normal_map(pls_context* ctx, const float* vmap, int batch, int H, int W, int ksize, float* out) {
    PLS_REQUIRE(ksize >= 1 && ksize <= 2 * NM_MAXR + 1 && (ksize & 1), "normal map: odd kernel size 1..9");
    dim3 grid((W + NM_TX - 1) / NM_TX, (H + NM_TY - 1) / NM_TY, batch), block(NM_TX, NM_TY);
    normal_map_kernel<<<grid, block, 0, ctx->stream>>>(vmap, batch, H, W, ksize, out);
    PLS_CHECK_LAUNCH();
}

void projmap_reset(pls_context* ctx) {
    ctx->pm.K = 0;
    ctx->pm.head = 0;
    ctx->pm.valid = false;
    ctx->pm.host_poses.clear();
}

// ProjectiveLocalMap.update (local_map.py:126-174): poses_k <- rel^-1 poses_k, append, evict, rebuild.
void projmap_update(pls_context* ctx, const float* rel_pose_host, const float* vmap_dev) {
    ProjMap& pm = ctx->pm;
    cudaStream_t st = ctx->stream;
    const int H = ctx->cfg.height, W = ctx->cfg.width;
    const int64_t hw = (int64_t)H * W;
    const int cap = ctx->cfg.local_map_size;
    const size_t frame_bytes = (size_t)3 * hw * sizeof(float);
    pm.vmaps.reserve((size_t)(cap + 1) * frame_bytes, st, true);
    pm.nmaps.reserve((size_t)(cap + 1) * frame_bytes, st, true);
    if (pm.K == 0) {
        PLS_REQUIRE(vmap_dev != nullptr, "projective map: the first update needs a vertex map");
        pm.host_poses.assign(rel_pose_host, rel_pose_host + 16);
        PLS_CUDA(cudaMemcpyAsync(pm.vmaps.p, vmap_dev, frame_bytes, cudaMemcpyDeviceToDevice, st));
        launch_normal_map(ctx, vmap_dev, 1, H, W, ctx->cfg.normals_kernel_size, pm.nmaps.as<float>());
        pm.K = 1;
    } else {
        float inv[16], tmp[16];
        rigid_inverse(rel_pose_host, inv);
        for (int k = 0; k < pm.K; ++k) {
            mat4_mul(inv, &pm.host_poses[16 * k], tmp);
            memcpy(&pm.host_poses[16 * k], tmp, sizeof(tmp));
        }
        const int slots = cap + 1;
        if (vmap_dev) {
            float eye[16];
            for (int i = 0; i < 16; ++i) eye[i] = (i % 5 == 0) ? 1.f : 0.f;
            pm.host_poses.insert(pm.host_poses.end(), eye, eye + 16);
            const size_t slot = (size_t)((pm.head + pm.K) % slots);  // ring of cap+1 frame slots
            char* vdst = reinterpret_cast<char*>(pm.vmaps.p) + slot * frame_bytes;
            char* ndst = reinterpret_cast<char*>(pm.nmaps.p) + slot * frame_bytes;
            PLS_CUDA(cudaMemcpyAsync(vdst, vmap_dev, frame_bytes, cudaMemcpyDeviceToDevice, st));
            launch_normal_map(ctx, vmap_dev, 1, H, W, ctx->cfg.normals_kernel_size, reinterpret_cast<float*>(ndst));
            pm.K += 1;
        }
        if (pm.K > cap) {  // drop the oldest frame: advance the ring head
            pm.head = (pm.head + 1) % slots;
            pm.host_poses.erase(pm.host_poses.begin(), pm.host_poses.begin() + 16);
            pm.K -= 1;
        }
    }
    rebuild_model(ctx);
}

namespace {

// The launch geometry of one ICP iteration of ctx on rank `rank` of `num_ranks`, shared by projmap_icp_iteration and
// projmap_batch_begin.
struct ProjPlan {
    bool use_tma;
    int ktma, stages;
    size_t smem;                  // the TMA kernel's dynamic shared memory
    int64_t tile_begin, tile_end; // the rank's tiles (TMA path)
    int64_t need_lo, need_hi;     // the pixels the rank reduces
    int blocks;                   // partial rows: the TMA kernel's CTAs, or proj_icp_iter_kernel's blocks
};

// PLS_PROJ_RESIDENT_MB into *mb if it is set; returns whether it is.
bool resident_mb_env(int* mb) {
    static const char* e = getenv("PLS_PROJ_RESIDENT_MB");
    static const int v = e ? atoi(e) : 0;
    if (e) *mb = v;
    return e != nullptr;
}

ProjPlan plan_proj_iteration(const pls_context* ctx, int rank, int num_ranks) {
    const int64_t hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
    const int K = ctx->pm.K;
    ProjPlan p;
    // split of the K candidates between the TMA path and the direct-load path (at most 10 direct)
    static const int kdirect_env = getenv("PLS_PROJ_KDIRECT") ? atoi(getenv("PLS_PROJ_KDIRECT")) : 4;
    int kdirect = kdirect_env < 0 ? 0 : (kdirect_env > 10 ? 10 : kdirect_env);
    if (kdirect > K - 1) kdirect = K > 1 ? K - 1 : 0;
    p.ktma = K - kdirect;
    const size_t stage_bytes = (size_t)(p.ktma * 3 + 4) * PT_TILE * sizeof(float);
    static const bool no_tma = getenv("PLS_PROJ_NO_TMA") != nullptr;
    static const int stages = getenv("PLS_PROJ_STAGES") ? atoi(getenv("PLS_PROJ_STAGES")) : 2;
    p.stages = stages;
    p.use_tma = !no_tma && hw % PT_TILE == 0 && stages >= 1 && stages <= PT_STAGES && stage_bytes * stages <= 200 * 1024;
    p.smem = stage_bytes * stages;
    // the pixels this rank reduces: whole 128-pixel tiles on the TMA path.  Only they take part in the z-buffer of the
    // transformed queries and in the target map, and only they need the model (a sharded rank builds just its share)
    const int64_t tiles = hw / PT_TILE;
    p.tile_begin = tiles * rank / num_ranks;
    p.tile_end = tiles * (rank + 1) / num_ranks;
    p.need_lo = p.use_tma ? p.tile_begin * PT_TILE : hw * rank / num_ranks;
    p.need_hi = p.use_tma ? p.tile_end * PT_TILE : hw * (rank + 1) / num_ranks;
    if (p.use_tma) {
        // TMA-staged persistent kernel over 128-pixel tiles; ranks take contiguous tile ranges
        int per_sm = (int)((220 * 1024) / (p.smem + 2048));
        per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
        // equal tile counts per CTA: ceil(tiles / ceil(tiles / max_ctas)) persistent CTAs
        const int64_t my_tiles = p.tile_end - p.tile_begin;
        const int64_t max_ctas = (int64_t)per_sm * kNumSMs;
        const int64_t per_cta = (my_tiles + max_ctas - 1) / max_ctas;
        p.blocks = (int)((my_tiles + (per_cta > 0 ? per_cta : 1) - 1) / (per_cta > 0 ? per_cta : 1));
        if (p.blocks < 1) p.blocks = 1;
    } else {
        p.blocks = grid_for(p.need_hi - p.need_lo, PJ_THREADS, 4 * kNumSMs);
    }
    return p;
}

// The end of the tiles [tile_begin, ...) read evict-last: the first `budget` bytes of the model, a tile at a time.
int64_t resident_end_tile(const pls_context* ctx, int64_t tile_begin, int64_t budget) {
    const int64_t tile_bytes = (int64_t)ctx->cfg.local_map_size * 3 * PT_TILE * sizeof(float);
    return tile_begin + budget / tile_bytes;
}

}  // namespace

// one ICP iteration on the projective map; pixels [rank*hw/R, (rank+1)*hw/R) are reduced by this rank
int projmap_icp_iteration(pls_context* ctx, int64_t query_bound, int rank, int num_ranks) {
    ProjMap& pm = ctx->pm;
    PLS_REQUIRE(pm.valid, "projective map: search before any update");
    cudaStream_t st = ctx->stream;
    const int H = ctx->cfg.height, W = ctx->cfg.width;
    const int64_t hw = (int64_t)H * W;
    FrameResult* fr = frame_result_dev(ctx);
    ctx->tmp[3].reserve((size_t)hw * sizeof(unsigned long long), st);
    unsigned long long* zbuf = ctx->tmp[3].as<unsigned long long>();
    // the TMA path's resolve kernel leaves the z-buffer cleared, so only the first iteration of a frame memsets
    if (!pm.zbuf_clean) PLS_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)hw * sizeof(unsigned long long), st));
    pm.zbuf_clean = false;
    ProjConst pc = make_proj_const(H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
    const int K = pm.K;
    const ProjPlan plan = plan_proj_iteration(ctx, rank, num_ranks);
    const bool use_tma = plan.use_tma;
    const int64_t tile_begin = plan.tile_begin, tile_end = plan.tile_end;
    const int64_t need_lo = plan.need_lo, need_hi = plan.need_hi;
    if (need_lo < pm.built_lo || need_hi > pm.built_hi) rebuild_model(ctx, true);  // (the split rule changed since the update)
    query_zbuf_kernel<<<grid_for(query_bound, 256), 256, 0, st>>>(
        ctx->query_ptr, reinterpret_cast<const uint32_t*>(&fr->counts[1]), 0, fr->T, &fr->done, pc,
        use_tma ? (int)need_lo : 0, use_tma ? (int)need_hi : (int)hw, zbuf);
    PLS_CHECK_LAUNCH();
    const int blocks = plan.blocks;
    if (use_tma) {
        static bool attr_set = false;
        if (!attr_set) {
            PLS_CUDA(cudaFuncSetAttribute(proj_icp_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            attr_set = true;
        }
        ctx->partials.reserve((size_t)blocks * NACC * sizeof(double), st);
        ctx->tmp[7].reserve((size_t)hw * sizeof(float4), st);
        query_resolve_kernel<<<grid_for(need_hi - need_lo, 256), 256, 0, st>>>(zbuf, ctx->query_ptr, fr->T, &fr->done, need_lo, need_hi,
                                                                               ctx->tmp[7].as<float4>());
        PLS_CHECK_LAUNCH();
        // how much of this rank's share of the model asks to stay in the 50 MB L2 between iterations (swept on H100:
        // 16 MB is best for cfg3 and within 2 us of no hint for cfg5; 32 MB and more lose on both, profiles/README.md)
        int resident_mb = 16;
        resident_mb_env(&resident_mb);
        const int64_t resident_end = resident_end_tile(ctx, tile_begin, (int64_t)resident_mb << 20);
        // (a persisting access-policy window on the stream -- a set-aside part of L2 -- was tried instead of the
        // per-instruction priorities and was slower)
        ProfileScope ps(ctx, 1, 0.0, false);
        proj_icp_tma_kernel<<<blocks, PT_TILE, plan.smem, st>>>(pm.model_v.as<float>(), pm.model_n.as<float4>(), K,
                                                                ctx->cfg.local_map_size, ctx->tmp[7].as<float4>(), fr, tile_begin,
                                                                tile_end, ctx->cfg.scheme, ctx->cfg.sigma, plan.stages, plan.ktma,
                                                                resident_end, L2_EVICT_LAST, L2_EVICT_FIRST,
                                                                ctx->partials.as<double>());
        PLS_CHECK_LAUNCH();
        pm.zbuf_clean = true;
        return blocks;
    }
    const int64_t pix_begin = need_lo, pix_end = need_hi;
    ctx->partials.reserve((size_t)blocks * NACC * sizeof(double), st);
    {
        ProfileScope ps(ctx, 1, 0.0, false);
        proj_icp_iter_kernel<<<blocks, PJ_THREADS, 0, st>>>(pm.model_v.as<float>(), pm.model_n.as<float4>(), pm.K,
                                                            ctx->cfg.local_map_size, zbuf,
                                                            ctx->query_ptr, fr, pix_begin, pix_end, ctx->cfg.scheme,
                                                            ctx->cfg.sigma, ctx->partials.as<double>());
        PLS_CHECK_LAUNCH();
    }
    return blocks;
}

// pls_process_frames: the descriptors of the projective sequences whose ICP runs in this call, into lead->batch_buf
// (uploaded on st) with their done flags and then the TMA sequences' partial rows behind them, one range per sequence,
// and every buffer their iterations use reserved as their single path reserves it.
// grid[4]: the launch widths (the largest query z-buffer / resolve / TMA block count of a sequence) and the TMA
// kernel's dynamic shared memory (the largest of a sequence; 0: no sequence takes the TMA path).
void projmap_batch_begin(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                         int* grid) {
    std::vector<ProjSeq> seqs((size_t)num);
    std::vector<ProjPlan> plans((size_t)num);
    int tma_seqs = 0;
    size_t rows = 0;
    for (int i = 0; i < num; ++i) {
        PLS_REQUIRE(ctxs[i]->pm.valid, "projective map: search before any update");
        plans[(size_t)i] = plan_proj_iteration(ctxs[i], 0, 1);
        if (plans[(size_t)i].use_tma) {
            tma_seqs += 1;
            rows += (size_t)plans[(size_t)i].blocks;
        }
    }
    // The L2 budget for evict-last reads: the single path's 16 MB, split evenly across the TMA sequences (measured on
    // H100 against 16 MB for each of them, DESIGN section 11).  PLS_PROJ_RESIDENT_MB is each sequence's own budget.
    int mb = 16;
    const int64_t budget = resident_mb_env(&mb) ? (int64_t)mb << 20 : ((int64_t)16 << 20) / (tma_seqs > 0 ? tma_seqs : 1);
    const size_t head = (num * sizeof(ProjSeq) + PLS_MAX_SEQUENCES * sizeof(int) + 255) / 256 * 256;
    lead->batch_buf.reserve(head + rows * NACC * sizeof(double), st);
    double* part = reinterpret_cast<double*>(lead->batch_buf.as<char>() + head);
    grid[0] = grid[1] = grid[2] = 1;
    grid[3] = 0;
    for (int i = 0; i < num; ++i) {
        pls_context* ctx = ctxs[i];
        const ProjPlan& plan = plans[(size_t)i];
        const int64_t hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
        FrameResult* fr = frame_result_dev(ctx);
        ctx->last_sharded = false;
        ctx->tmp[3].reserve((size_t)hw * sizeof(unsigned long long), st);
        ProjSeq& s = seqs[(size_t)i];
        s.model_v = ctx->pm.model_v.as<float>();
        s.model_n = ctx->pm.model_n.as<float4>();
        s.queries = ctx->query_ptr;
        s.nq_dev = reinterpret_cast<const uint32_t*>(&fr->counts[1]);
        s.fr = fr;
        s.zbuf = ctx->tmp[3].as<unsigned long long>();
        s.pc = make_proj_const(ctx->cfg.height, ctx->cfg.width, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
        s.K = ctx->pm.K;
        s.kcap = ctx->cfg.local_map_size;
        s.ktma = plan.ktma;
        s.stages = plan.stages;
        s.scheme = ctx->cfg.scheme;
        s.sigma = ctx->cfg.sigma;
        s.threshold_delta = ctx->cfg.threshold_delta_pose;
        s.tiles = hw / PT_TILE;
        s.resident_end = resident_end_tile(ctx, 0, budget);
        s.step_blocks = plan.blocks;
        s.max_iters = ctx->cfg.max_num_alignments;
        if (plan.use_tma) {
            ctx->tmp[7].reserve((size_t)hw * sizeof(float4), st);
            s.tgt = ctx->tmp[7].as<float4>();
            s.partials = part;
            part += (size_t)plan.blocks * NACC;
            s.zbuf_blocks = grid_for(query_bounds[i], 256);
            s.resolve_blocks = grid_for(hw, 256);
            s.tma_blocks = plan.blocks;
            grid[0] = grid[0] > s.zbuf_blocks ? grid[0] : s.zbuf_blocks;
            grid[1] = grid[1] > s.resolve_blocks ? grid[1] : s.resolve_blocks;
            grid[2] = grid[2] > s.tma_blocks ? grid[2] : s.tma_blocks;
            grid[3] = grid[3] > (int)plan.smem ? grid[3] : (int)plan.smem;
        } else {
            // its own launches write ctx->partials (projmap_icp_iteration reserves the same size: no reallocation)
            ctx->partials.reserve((size_t)plan.blocks * NACC * sizeof(double), st);
            s.tgt = nullptr;
            s.partials = ctx->partials.as<double>();
            s.zbuf_blocks = s.resolve_blocks = s.tma_blocks = 0;
        }
    }
    PLS_CUDA(cudaMemcpyAsync(lead->batch_buf.p, seqs.data(), seqs.size() * sizeof(ProjSeq), cudaMemcpyHostToDevice, st));
}

// ICP iterations [first, last) of the sequences projmap_batch_begin described, on st: one launch per kernel for all of
// them.  A sequence off the TMA path runs its correspondences through its own launches; the step kernel serves all.
void projmap_batch_iterations(pls_context* lead, pls_context* const* ctxs, const int64_t* query_bounds, int num, cudaStream_t st,
                              const int* grid, int first, int last) {
    const ProjSeq* seqs = lead->batch_buf.as<ProjSeq>();
    static bool attr_set = false;
    if (!attr_set) {
        PLS_CUDA(cudaFuncSetAttribute(proj_icp_tma_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set = true;
    }
    for (int it = first; it < last; ++it) {
        for (int i = 0; i < num; ++i) {
            pls_context* ctx = ctxs[i];
            if (it >= ctx->cfg.max_num_alignments) continue;
            if (plan_proj_iteration(ctx, 0, 1).use_tma) {
                // the first iteration clears the query z-buffer (the frame's own projection used it); the resolve kernel
                // leaves it clear for the next
                if (it == 0)
                    PLS_CUDA(cudaMemsetAsync(ctx->tmp[3].p, 0xff,
                                             (size_t)ctx->cfg.height * ctx->cfg.width * sizeof(unsigned long long), st));
                ctx->pm.zbuf_clean = true;
                continue;
            }
            cudaStream_t own = ctx->stream;
            ctx->stream = st;
            try {
                projmap_icp_iteration(ctx, query_bounds[i], 0, 1);
            } catch (...) {
                ctx->stream = own;
                throw;
            }
            ctx->stream = own;
        }
        if (grid[3] > 0) {
            query_zbuf_batch_kernel<<<dim3(grid[0], num), 256, 0, st>>>(seqs, it);
            PLS_CHECK_LAUNCH();
            query_resolve_batch_kernel<<<dim3(grid[1], num), 256, 0, st>>>(seqs, it);
            PLS_CHECK_LAUNCH();
            proj_icp_tma_batch_kernel<<<dim3(grid[2], num), PT_TILE, (size_t)grid[3], st>>>(seqs, it);
            PLS_CHECK_LAUNCH();
        }
        icp_step_batch_kernel<<<dim3(1, num), 256, 0, st>>>(seqs, it);
        PLS_CHECK_LAUNCH();
    }
}

// The done flag of every sequence of the batch: one gather launch, one copy, one synchronisation.
void projmap_batch_done(pls_context* lead, int num, cudaStream_t st, int* out) {
    int* dev = reinterpret_cast<int*>(lead->batch_buf.as<char>() + (size_t)num * sizeof(ProjSeq));
    proj_batch_done_kernel<<<1, 64, 0, st>>>(lead->batch_buf.as<ProjSeq>(), num, dev);
    PLS_CHECK_LAUNCH();
    PLS_CUDA(cudaMemcpyAsync(out, dev, (size_t)num * sizeof(int), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));
}

namespace {

// Where the state of `num` hypotheses lives in ctx->hyp_buf: their FrameResults, 16 begin words each (the counter words
// frame_begin_body clears), then per hypothesis a query z-buffer, a target map (TMA path) and the single call's partial
// rows.
struct HypLayout {
    ProjPlan plan;
    int64_t hw;
    size_t fr_off, words_off, zbuf_off, tgt_off, part_off, total;
};

HypLayout hyp_layout(const pls_context* ctx, int num) {
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    HypLayout L;
    L.plan = plan_proj_iteration(ctx, 0, 1);
    L.hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
    L.fr_off = 0;
    L.words_off = up((size_t)num * sizeof(FrameResult));
    L.zbuf_off = L.words_off + up((size_t)num * 16 * sizeof(uint32_t));
    L.tgt_off = L.zbuf_off + up((size_t)num * L.hw * sizeof(unsigned long long));
    L.part_off = L.tgt_off + (L.plan.use_tma ? up((size_t)num * L.hw * sizeof(float4)) : 0);
    L.total = L.part_off + (size_t)num * L.plan.blocks * NACC * sizeof(double);
    return L;
}

}  // namespace

// pls_register_hypotheses on ctx's projective map: the state of `num` hypotheses of the scan in ctx->query_ptr (count in
// ctx's FrameResult) in ctx->hyp_buf, their step descriptors (ProjSeq) and done flags in ctx->batch_buf.  Returns their
// FrameResults and 16 words each, for hypotheses_begin_kernel.
void projmap_hypotheses_begin(pls_context* ctx, int num, cudaStream_t st, FrameResult** frs, uint32_t** words) {
    PLS_REQUIRE(ctx->pm.valid, "projective map: search before any update");
    const HypLayout L = hyp_layout(ctx, num);
    ctx->last_sharded = false;
    ctx->hyp_buf.reserve(L.total, st);
    char* base = ctx->hyp_buf.as<char>();
    *frs = reinterpret_cast<FrameResult*>(base + L.fr_off);
    *words = reinterpret_cast<uint32_t*>(base + L.words_off);
    std::vector<ProjSeq> seqs((size_t)num);
    for (int h = 0; h < num; ++h) {
        ProjSeq& s = seqs[(size_t)h];
        memset(&s, 0, sizeof(s));
        s.model_v = ctx->pm.model_v.as<float>();
        s.model_n = ctx->pm.model_n.as<float4>();
        s.queries = ctx->query_ptr;
        s.fr = *frs + h;
        s.zbuf = reinterpret_cast<unsigned long long*>(base + L.zbuf_off) + (size_t)h * L.hw;
        s.tgt = L.plan.use_tma ? reinterpret_cast<float4*>(base + L.tgt_off) + (size_t)h * L.hw : nullptr;
        s.partials = reinterpret_cast<double*>(base + L.part_off) + (size_t)h * L.plan.blocks * NACC;
        s.K = ctx->pm.K;
        s.kcap = ctx->cfg.local_map_size;
        s.scheme = ctx->cfg.scheme;
        s.sigma = ctx->cfg.sigma;
        s.threshold_delta = ctx->cfg.threshold_delta_pose;
        s.step_blocks = L.plan.blocks;
        s.max_iters = ctx->cfg.max_num_alignments;
    }
    const size_t head = (num * sizeof(ProjSeq) + PLS_MAX_SEQUENCES * sizeof(int) + 255) / 256 * 256;
    ctx->batch_buf.reserve(head, st);
    PLS_CUDA(cudaMemcpyAsync(ctx->batch_buf.p, seqs.data(), seqs.size() * sizeof(ProjSeq), cudaMemcpyHostToDevice, st));
}

// ICP iterations [first, last) of the hypotheses projmap_hypotheses_begin described, on st.  TMA path: one z-buffer,
// one resolve, one proj_icp_tma_hyp_kernel and one step launch per iteration, whatever num.  Off it, each hypothesis
// runs proj_icp_iter_kernel in its own launch, as projmap_icp_iteration does; the z-buffer and step launches are shared.
void projmap_hypotheses_iterations(pls_context* ctx, int64_t query_bound, int num, cudaStream_t st, int first, int last) {
    const HypLayout L = hyp_layout(ctx, num);
    const ProjPlan& plan = L.plan;
    char* base = ctx->hyp_buf.as<char>();
    const FrameResult* frs = reinterpret_cast<const FrameResult*>(base + L.fr_off);
    unsigned long long* zbufs = reinterpret_cast<unsigned long long*>(base + L.zbuf_off);
    float4* tgts = reinterpret_cast<float4*>(base + L.tgt_off);
    double* parts = reinterpret_cast<double*>(base + L.part_off);
    const size_t part_rows = (size_t)plan.blocks * NACC;
    const ProjConst pc = make_proj_const(ctx->cfg.height, ctx->cfg.width, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
    const uint32_t* nq_dev = reinterpret_cast<const uint32_t*>(&frame_result_dev(ctx)->counts[1]);
    const int K = ctx->pm.K, kcap = ctx->cfg.local_map_size;
    int resident_mb = 16;
    resident_mb_env(&resident_mb);
    const int64_t resident_end = resident_end_tile(ctx, 0, (int64_t)resident_mb << 20);
    static bool attr_set = false;
    if (!attr_set) {
        PLS_CUDA(cudaFuncSetAttribute(proj_icp_tma_hyp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set = true;
    }
    for (int it = first; it < last; ++it) {
        // the single call clears its z-buffer before every iteration off the TMA path, before the first on it (the
        // resolve kernel leaves it clear)
        if (!plan.use_tma || it == 0)
            PLS_CUDA(cudaMemsetAsync(zbufs, 0xff, (size_t)num * L.hw * sizeof(unsigned long long), st));
        query_zbuf_hyp_kernel<<<grid_for(query_bound, 256), 256, 0, st>>>(ctx->query_ptr, nq_dev, frs, num, pc, L.hw, zbufs);
        PLS_CHECK_LAUNCH();
        if (plan.use_tma) {
            query_resolve_hyp_kernel<<<dim3(grid_for(L.hw, 256), num), 256, 0, st>>>(zbufs, ctx->query_ptr, frs, L.hw, tgts);
            PLS_CHECK_LAUNCH();
            const int64_t tiles = L.hw / PT_TILE;
            proj_icp_tma_hyp_kernel<<<(unsigned)(plan.blocks * num), PT_TILE, plan.smem, st>>>(
                ctx->pm.model_v.as<float>(), ctx->pm.model_n.as<float4>(), K, kcap, tgts, L.hw, frs, num, plan.blocks,
                tiles, ctx->cfg.scheme, ctx->cfg.sigma, plan.stages, plan.ktma, resident_end, parts, (int64_t)part_rows);
            PLS_CHECK_LAUNCH();
        } else {
            for (int h = 0; h < num; ++h) {
                proj_icp_iter_kernel<<<plan.blocks, PJ_THREADS, 0, st>>>(ctx->pm.model_v.as<float>(), ctx->pm.model_n.as<float4>(), K,
                                                                         kcap, zbufs + (size_t)h * L.hw, ctx->query_ptr, frs + h,
                                                                         0, L.hw, ctx->cfg.scheme, ctx->cfg.sigma,
                                                                         parts + (size_t)h * part_rows);
                PLS_CHECK_LAUNCH();
            }
        }
        icp_step_batch_kernel<<<dim3(1, num), 256, 0, st>>>(ctx->batch_buf.as<ProjSeq>(), it);
        PLS_CHECK_LAUNCH();
    }
}

// Hypothesis h's FrameResult (all but the counts) into ctx's own, and ctx's query z-buffer as the single call leaves it:
// pls_last_icp_sums and a following frame then see ctx as if pls_register_frame had run that hypothesis last.
void projmap_hypothesis_adopt(pls_context* ctx, int h, cudaStream_t st) {
    const HypLayout L = hyp_layout(ctx, h + 1);
    const FrameResult* fr = reinterpret_cast<const FrameResult*>(ctx->hyp_buf.as<char>() + L.fr_off) + h;
    PLS_CUDA(cudaMemcpyAsync(frame_result_dev(ctx), fr, offsetof(FrameResult, counts), cudaMemcpyDeviceToDevice, st));
    PLS_CUDA(cudaMemsetAsync(scalar_u32(ctx, SC_KD_COUNTERS), 0, 16 * sizeof(uint32_t), st));  // frame_begin clears them
    ctx->tmp[3].reserve((size_t)L.hw * sizeof(unsigned long long), st);
    if (L.plan.use_tma) PLS_CUDA(cudaMemsetAsync(ctx->tmp[3].p, 0xff, (size_t)L.hw * sizeof(unsigned long long), st));
    ctx->pm.zbuf_clean = L.plan.use_tma;
}

}  // namespace pls

using namespace pls;

extern "C" {

int pls_normal_map(pls_context* ctx, const float* vertex_map, int batch, int height, int width, int kernel_size, float* out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(vertex_map && out && batch > 0 && height > 0 && width > 0, "pls_normal_map: bad arguments");
    const size_t bytes = (size_t)batch * 3 * height * width * sizeof(float);
    const float* d = (const float*)to_device(ctx, vertex_map, bytes, ctx->stage_in[0]);
    OutArg o = out_arg(ctx, out, bytes, ctx->stage_out[0]);
    launch_normal_map(ctx, d, batch, height, width, kernel_size, (float*)o.dev);
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_compute_neighbors(pls_context* ctx, const float* tgt, const float* ref, const float* fields, int num_ref,
                          int num_field_channels, int height, int width, float* out_nb, float* out_fields) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(tgt && ref && out_nb && num_ref > 0 && height > 0 && width > 0, "pls_compute_neighbors: bad arguments");
    PLS_REQUIRE(!fields || (out_fields && num_field_channels > 0), "pls_compute_neighbors: fields need an output");
    const int64_t hw = (int64_t)height * width;
    const float* d_t = (const float*)to_device(ctx, tgt, (size_t)3 * hw * sizeof(float), ctx->stage_in[0]);
    const float* d_r = (const float*)to_device(ctx, ref, (size_t)num_ref * 3 * hw * sizeof(float), ctx->stage_in[1]);
    const float* d_f = (const float*)to_device(ctx, fields, (size_t)num_ref * num_field_channels * hw * sizeof(float), ctx->stage_in[2]);
    OutArg onb = out_arg(ctx, out_nb, (size_t)3 * hw * sizeof(float), ctx->stage_out[0]);
    OutArg of = out_arg(ctx, fields ? out_fields : nullptr, (size_t)num_field_channels * hw * sizeof(float), ctx->stage_out[1]);
    compute_neighbors_kernel<<<grid_for(hw, 256), 256, 0, ctx->stream>>>(d_t, d_r, d_f, num_ref, num_field_channels, hw,
                                                                         (float*)onb.dev, (float*)of.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, onb);
    finish_out(ctx, of);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_projmap_update(pls_context* ctx, const float* rel_pose, const float* vertex_map) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(rel_pose, "pls_projmap_update: rel_pose required");
    PLS_REQUIRE(ctx->cfg.local_map_type == PLS_MAP_PROJECTIVE, "context holds a kd map");
    float rel[16];
    if (is_device_ptr(rel_pose)) PLS_CUDA(cudaMemcpy(rel, rel_pose, sizeof(rel), cudaMemcpyDeviceToHost));
    else memcpy(rel, rel_pose, sizeof(rel));
    const size_t bytes = (size_t)3 * ctx->cfg.height * ctx->cfg.width * sizeof(float);
    const float* d = (const float*)to_device(ctx, vertex_map, bytes, ctx->stage_in[0]);
    projmap_update(ctx, rel, d);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_projmap_num_frames(pls_context* ctx, int* num_frames) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(num_frames, "pls_projmap_num_frames: null output");
    *num_frames = ctx->pm.K;
    PLS_API_END(ctx)
}

int pls_projmap_last_frame(pls_context* ctx, float* out_vmap) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(out_vmap, "pls_projmap_last_frame: null output");
    const ProjMap& pm = ctx->pm;
    if (pm.K == 0) throw pls::Error{PLS_E_STATE, "pls_projmap_last_frame: the map holds no frame"};
    const size_t frame_bytes = (size_t)3 * ctx->cfg.height * ctx->cfg.width * sizeof(float);
    const size_t slot = (size_t)((pm.head + pm.K - 1) % (ctx->cfg.local_map_size + 1));  // the ring slot of the newest
    OutArg o = out_arg(ctx, out_vmap, frame_bytes, ctx->stage_out[0]);
    PLS_CUDA(cudaMemcpyAsync(o.dev, pm.vmaps.as<char>() + slot * frame_bytes, frame_bytes, cudaMemcpyDeviceToDevice,
                             ctx->stream));
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_projmap_model(pls_context* ctx, float* out_vmap, float* out_nmap) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(ctx->pm.valid, "pls_projmap_model: empty map");
    ensure_full_model(ctx);
    const int64_t hw = (int64_t)ctx->cfg.height * ctx->cfg.width;
    const size_t bytes = (size_t)ctx->pm.K * 3 * hw * sizeof(float);
    auto put = [&](float* dst, const float* tiled, DBuf& stage) {
        if (!dst) return;
        OutArg o = out_arg(ctx, dst, bytes, stage);
        model_export_kernel<<<grid_for((int64_t)ctx->pm.K * 3 * hw, 256), 256, 0, ctx->stream>>>(tiled, ctx->pm.K, ctx->cfg.local_map_size,
                                                                                              hw, (float*)o.dev);
        PLS_CHECK_LAUNCH();
        finish_out(ctx, o);
    };
    put(out_vmap, ctx->pm.model_v.as<float>(), ctx->stage_out[0]);
    if (out_nmap) {
        OutArg o = out_arg(ctx, out_nmap, bytes, ctx->stage_out[1]);
        normal_export_kernel<<<grid_for((int64_t)ctx->pm.K * hw, 256), 256, 0, ctx->stream>>>(ctx->pm.model_n.as<float4>(), ctx->pm.K,
                                                                                           ctx->cfg.local_map_size, hw, (float*)o.dev);
        PLS_CHECK_LAUNCH();
        finish_out(ctx, o);
    }
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_projmap_nn_search(pls_context* ctx, const float* queries, int64_t n, float* out_neighbors, float* out_normals,
                          float* out_targets, int64_t* out_count) {
    PLS_API_BEGIN(ctx)
    map_stream_wait(ctx);
    PLS_REQUIRE(queries && out_neighbors && out_count && n > 0, "pls_projmap_nn_search: bad arguments");
    if (!ctx->pm.valid) throw pls::Error{PLS_E_STATE, "pls_projmap_nn_search: the map is empty"};
    cudaStream_t st = ctx->stream;
    const int H = ctx->cfg.height, W = ctx->cfg.width;
    const int64_t hw = (int64_t)H * W;
    const float* d = (const float*)to_device(ctx, queries, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    // queries as float4 (no NaN filtering here: the reference passes them through unchanged)
    ctx->queries.reserve((size_t)n * sizeof(float4), st);
    uint32_t* cnt = scalar_u32(ctx, SC_NAN_COUNT);
    pack_valid_rows(ctx, d, n, ctx->queries.as<float4>(), cnt);
    ctx->tmp[3].reserve((size_t)hw * sizeof(unsigned long long), st);
    unsigned long long* zbuf = ctx->tmp[3].as<unsigned long long>();
    PLS_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)hw * sizeof(unsigned long long), st));
    ProjConst pc = make_proj_const(H, W, ctx->cfg.up_fov_deg, ctx->cfg.down_fov_deg);
    ensure_full_model(ctx);
    query_zbuf_kernel<<<grid_for(n, 256), 256, 0, st>>>(ctx->queries.as<float4>(), cnt, 0, nullptr, nullptr, pc, 0, (int)hw, zbuf);
    PLS_CHECK_LAUNCH();
    ctx->tmp[1].reserve((size_t)hw, st);
    ctx->tmp[2].reserve((size_t)hw * sizeof(uint32_t), st);
    ctx->tmp[7].reserve((size_t)hw * 9 * sizeof(float), st);
    proj_pairs_kernel<<<grid_for(hw, 256), 256, 0, st>>>(ctx->pm.model_v.as<float>(), ctx->pm.model_n.as<float4>(), ctx->pm.K,
                                                          ctx->cfg.local_map_size, hw, zbuf, ctx->queries.as<float4>(), ctx->tmp[1].as<uint8_t>(),
                                                          ctx->tmp[7].as<float>());
    PLS_CHECK_LAUNCH();
    uint32_t* total = scalar_u32(ctx, SC_PROJ_NC);
    exclusive_scan_flags(ctx, ctx->tmp[1].as<uint8_t>(), hw, ctx->tmp[2].as<uint32_t>(), total);
    OutArg oq = out_arg(ctx, out_neighbors, (size_t)hw * 3 * sizeof(float), ctx->stage_out[0]);
    OutArg on = out_arg(ctx, out_normals, (size_t)hw * 3 * sizeof(float), ctx->stage_out[1]);
    OutArg op = out_arg(ctx, out_targets, (size_t)hw * 3 * sizeof(float), ctx->stage_out[2]);
    proj_compact_kernel<<<grid_for(hw, 256), 256, 0, st>>>(ctx->tmp[1].as<uint8_t>(), ctx->tmp[2].as<uint32_t>(),
                                                            ctx->tmp[7].as<float>(), hw, (float*)oq.dev, (float*)on.dev,
                                                            (float*)op.dev);
    PLS_CHECK_LAUNCH();
    uint32_t nc = 0;
    PLS_CUDA(cudaMemcpyAsync(&nc, total, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PLS_CUDA(cudaStreamSynchronize(st));
    *out_count = nc;
    finish_out(ctx, oq, (size_t)nc * 3 * sizeof(float));
    finish_out(ctx, on, (size_t)nc * 3 * sizeof(float));
    finish_out(ctx, op, (size_t)nc * 3 * sizeof(float));
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_API_END(ctx)
}

}  // extern "C"
