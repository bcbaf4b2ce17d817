// Unsupervised point-to-plane training loss, forward + backward in one pass -- the other caller of the projection /
// normal-map helpers of the hot path (SURVEY.md section 8f rank 3).
//
// Replaces _PointToPlaneLossModule.point_to_plane_loss (slam/training/loss_modules.py:51-104) and the autograd graph
// behind it:
//   p'      = (R p + t) * [p != 0]                         every pixel of the target vertex map, batch b
//   vm'     = build_projection_map(p')                     closest point per pixel (projection.py:331-418)
//   r       = n . (q - vm'),  a = mask |r|                 q / n = reference vertex / normal map, mask = all three non-null
//   loss    = mean_b ( sum_pix C(a)^2 / sum_pix mask )     C = the weighting scheme's cost (optimization.py:61-208)
//   dloss/d[R|t]: autograd lets values flow through the scatter `image[b,:,row,col] = values[b,order,:]`; index_put's
//   backward hands EVERY point written to a pixel that pixel's gradient (also the points a closer one overwrote), and the
//   rounded pixel coordinates carry none.  Reproduced as is.
//
//   loss_zbuf_kernel       transform + pixel math + one 64-bit atomicMin per point (range bits << 32 | index)
//   loss_accumulate_kernel per point: the pixel it landed in, that pixel's winner, the pixel's terms (training_device.cuh);
//                          the winner also books C^2 and mask; everyone books g and g p^T; float64 accumulation,
//                          warp-shuffle + shared-memory block reduction, one partial row per block (no atomics)
//   loss_finalize_kernel   fixed-order sum of the partial rows per batch element, 1/(M_b B) scaling, the chain rule
//                          through build_pose_matrix when the caller passed pose parameters
//
// HBM-bound: per point 12 B target + 8 B z-buffer (atomic) in pass 1; 12 + 8 + 12 (winner) + 24 (q, n) B in pass 2.
#include "internal.cuh"
#include "pose_device.cuh"
#include "projection_device.cuh"
#include "training_device.cuh"

namespace pls {

namespace {

constexpr int TL_THREADS = 256;
constexpr int TL_ROW = 16;  // sum C^2, sum mask, g (3), g p^T (9), landed points, pad

__device__ __forceinline__ void load_pose(const float* __restrict__ mats, int b, float* sT) {
    if (threadIdx.x < 12) sT[threadIdx.x] = mats[16 * (size_t)b + threadIdx.x];
    __syncthreads();
}

__device__ __forceinline__ bool moved_point(const float* __restrict__ vm, int64_t hw, int64_t i, const float* sT, float* p, float* pm) {
    p[0] = vm[i]; p[1] = vm[hw + i]; p[2] = vm[2 * hw + i];
    // mask_vm = (|p| != 0); the null point stays null after the transform (loss_modules.py:79-83)
    if (p[0] == 0.f && p[1] == 0.f && p[2] == 0.f) return false;
    transform_point(sT, make_float4(p[0], p[1], p[2], 0.f), pm);
    return true;
}

__global__ void __launch_bounds__(TL_THREADS)
loss_zbuf_kernel(const float* __restrict__ vm_target, const float* __restrict__ mats, int64_t hw, ProjConst pc,
                 unsigned long long* __restrict__ zbuf) {
    __shared__ float sT[12];
    const int b = blockIdx.y;
    load_pose(mats, b, sT);
    const float* vm = vm_target + 3 * hw * (size_t)b;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x) {
        float p[3], pm[3];
        if (!moved_point(vm, hw, i, sT, p, pm)) continue;
        int pix;
        float r;
        // the order loss_accumulate_kernel finds each pixel's winner with
        if (project_to_pixel(pm[0], pm[1], pm[2], pc, pix, r, RangeOrder::kYFirst))
            atomicMin(&zbuf[hw * (size_t)b + pix], ((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)i);
    }
}

__global__ void __launch_bounds__(TL_THREADS)
loss_accumulate_kernel(const float* __restrict__ vm_target, const float* __restrict__ vm_reference,
                       const float* __restrict__ nm_reference, const float* __restrict__ mats, int64_t hw, ProjConst pc,
                       const unsigned long long* __restrict__ zbuf, int scheme, float sigma, double* __restrict__ partials) {
    __shared__ float sT[12];
    const int b = blockIdx.y;
    load_pose(mats, b, sT);
    const float* vm = vm_target + 3 * hw * (size_t)b;
    const float* vr = vm_reference + 3 * hw * (size_t)b;
    const float* nr = nm_reference + 3 * hw * (size_t)b;
    double acc[TL_ROW];
#pragma unroll
    for (int a = 0; a < TL_ROW; ++a) acc[a] = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x) {
        float p[3], pm[3];
        if (!moved_point(vm, hw, i, sT, p, pm)) continue;
        int pix;
        float r;
        if (!project_to_pixel(pm[0], pm[1], pm[2], pc, pix, r, RangeOrder::kYFirst)) continue;  // loss_zbuf_kernel's order
        const uint32_t win = (uint32_t)(zbuf[hw * (size_t)b + pix] & 0xffffffffull);
        float pw[3] = {pm[0], pm[1], pm[2]};
        if (win != (uint32_t)i) {
            float pj[3];
            moved_point(vm, hw, (int64_t)win, sT, pj, pw);
        }
        const float q[3] = {vr[pix], vr[hw + pix], vr[2 * hw + pix]};
        const float n[3] = {nr[pix], nr[hw + pix], nr[2 * hw + pix]};
        double mask, c2, g[3];
        loss_pixel_terms(scheme, (double)sigma, pw, q, n, mask, c2, g);
        if (win == (uint32_t)i) {  // each pixel is booked once, by its surviving point
            acc[0] += c2;
            acc[1] += mask;
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            acc[2 + a] += g[a];
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[5 + 3 * a + c] += g[a] * (double)p[c];
        }
        acc[14] += 1.0;
    }
    __shared__ double red[TL_THREADS / 32][TL_ROW];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < TL_ROW; ++a) {
        const double v = warp_sum(acc[a]);
        if (lane == 0) red[warp][a] = v;
    }
    __syncthreads();
    if (threadIdx.x < TL_ROW) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < TL_THREADS / 32; ++w) s += red[w][threadIdx.x];
        partials[((size_t)b * gridDim.x + blockIdx.x) * TL_ROW + threadIdx.x] = s;
    }
}

// One block per call; warp w handles batch elements w, w + 8, ...: lane a < 16 sums accumulator a over the blocks in
// fixed order, lane 0 then scales and (optionally) chains to the pose parameters.
__global__ void __launch_bounds__(TL_THREADS)
loss_finalize_kernel(const double* __restrict__ partials, int blocks_per_batch, int batch, const float* __restrict__ params,
                     float* __restrict__ loss_per_batch, float* __restrict__ grad_mats, float* __restrict__ grad_params,
                     float* __restrict__ loss_out) {
    __shared__ double s_loss[64];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int b = warp; b < batch; b += TL_THREADS / 32) {
        double s = 0.0;
        if (lane < TL_ROW)
            for (int k = 0; k < blocks_per_batch; ++k) s += partials[((size_t)b * blocks_per_batch + k) * TL_ROW + lane];
        double row[TL_ROW];
#pragma unroll
        for (int a = 0; a < TL_ROW; ++a) row[a] = __shfl_sync(0xffffffffu, s, a);
        if (lane == 0) {
            const double M = row[1];
            const double lb = row[0] / M;  // loss_modules.py:102 (no guard against M == 0 in the reference either)
            if (b < 64) s_loss[b] = lb;
            if (loss_per_batch) loss_per_batch[b] = (float)lb;
            const double sc = 1.0 / (M * (double)batch);
            double G[12];  // rows of [dL/dR | dL/dt]
            for (int a = 0; a < 3; ++a) {
                for (int c = 0; c < 3; ++c) G[4 * a + c] = row[5 + 3 * a + c] * sc;
                G[4 * a + 3] = row[2 + a] * sc;
            }
            if (grad_mats) {
                for (int k = 0; k < 12; ++k) grad_mats[16 * (size_t)b + k] = (float)G[k];
                for (int k = 12; k < 16; ++k) grad_mats[16 * (size_t)b + k] = 0.f;
            }
            if (grad_params && params) {
                // chain rule through Pose.build_pose_matrix (pose.py:120-144; rotation.py:166-184)
                float dR[27];
                euler_jacobian(params + 6 * (size_t)b + 3, dR);
                for (int a = 0; a < 3; ++a) grad_params[6 * (size_t)b + a] = (float)G[4 * a + 3];
                for (int k = 0; k < 3; ++k) {
                    double s2 = 0.0;
                    for (int a = 0; a < 3; ++a)
                        for (int c = 0; c < 3; ++c) s2 += G[4 * a + c] * (double)dR[9 * k + 3 * a + c];
                    grad_params[6 * (size_t)b + 3 + k] = (float)s2;
                }
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && loss_out) {
        double s = 0.0;
        for (int b = 0; b < batch; ++b) s += s_loss[b];
        *loss_out = (float)(s / (double)batch);
    }
}

__global__ void pose_build_batch_kernel(const float* __restrict__ params, int batch, float* __restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) build_pose(params + 6 * (size_t)b, out + 16 * (size_t)b);
}

}  // namespace
}  // namespace pls

using namespace pls;

extern "C" {

int pls_p2plane_loss(pls_context* ctx, const float* vm_target, const float* vm_reference, const float* nm_reference,
                     const float* pose_mats, const float* pose_params, int batch, int height, int width, float up_fov_deg,
                     float down_fov_deg, int scheme, float sigma, float* out_loss, float* out_loss_per_batch,
                     float* out_grad_mats, float* out_grad_params) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(vm_target && vm_reference && nm_reference && (pose_mats || pose_params) && out_loss,
                "pls_p2plane_loss: vertex / normal maps, a pose and the loss pointer are required");
    PLS_REQUIRE(batch > 0 && batch <= 64 && height > 0 && width > 0, "pls_p2plane_loss: 1 <= batch <= 64, positive image size");
    PLS_REQUIRE(scheme >= 0 && scheme <= PLS_SCHEME_CAUCHY, "pls_p2plane_loss: unknown weighting scheme");
    PLS_REQUIRE(!out_grad_params || pose_params, "pls_p2plane_loss: gradients w.r.t. parameters need the parameters");
    cudaStream_t st = ctx->stream;
    const int64_t hw = (int64_t)height * width;
    const size_t map_bytes = (size_t)batch * 3 * hw * sizeof(float);
    const float* d_vt = (const float*)to_device(ctx, vm_target, map_bytes, ctx->stage_in[0]);
    const float* d_vr = (const float*)to_device(ctx, vm_reference, map_bytes, ctx->stage_in[1]);
    const float* d_nr = (const float*)to_device(ctx, nm_reference, map_bytes, ctx->stage_in[2]);
    const float* d_params = pose_params ? (const float*)to_device(ctx, pose_params, (size_t)batch * 6 * sizeof(float), ctx->stage_in[3]) : nullptr;
    const float* d_mats;
    if (pose_mats) {
        ctx->next_buf[0].reserve((size_t)batch * 16 * sizeof(float), st);
        if (is_device_ptr(pose_mats)) d_mats = pose_mats;
        else {
            PLS_CUDA(cudaMemcpyAsync(ctx->next_buf[0].p, pose_mats, (size_t)batch * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
            d_mats = ctx->next_buf[0].as<float>();
        }
    } else {
        ctx->next_buf[0].reserve((size_t)batch * 16 * sizeof(float), st);
        pose_build_batch_kernel<<<1, 64, 0, st>>>(d_params, batch, ctx->next_buf[0].as<float>());
        PLS_CHECK_LAUNCH();
        d_mats = ctx->next_buf[0].as<float>();
    }
    int64_t bpb = (hw + TL_THREADS - 1) / TL_THREADS;
    const int64_t cap = (4 * kNumSMs + batch - 1) / batch;
    if (bpb > cap) bpb = cap;
    if (bpb < 1) bpb = 1;
    const dim3 grid((unsigned)bpb, (unsigned)batch);
    ctx->next_buf[1].reserve((size_t)batch * hw * sizeof(unsigned long long), st);
    ctx->next_buf[2].reserve((size_t)batch * bpb * TL_ROW * sizeof(double), st);
    unsigned long long* zbuf = ctx->next_buf[1].as<unsigned long long>();
    PLS_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)batch * hw * sizeof(unsigned long long), st));
    const ProjConst pc = make_proj_const(height, width, up_fov_deg, down_fov_deg);
    loss_zbuf_kernel<<<grid, TL_THREADS, 0, st>>>(d_vt, d_mats, hw, pc, zbuf);
    PLS_CHECK_LAUNCH();
    loss_accumulate_kernel<<<grid, TL_THREADS, 0, st>>>(d_vt, d_vr, d_nr, d_mats, hw, pc, zbuf, scheme, sigma,
                                                        ctx->next_buf[2].as<double>());
    PLS_CHECK_LAUNCH();
    OutArg o_loss = out_arg(ctx, out_loss, sizeof(float), ctx->stage_out[0]);
    OutArg o_pb = out_arg(ctx, out_loss_per_batch, (size_t)batch * sizeof(float), ctx->stage_out[1]);
    OutArg o_gm = out_arg(ctx, out_grad_mats, (size_t)batch * 16 * sizeof(float), ctx->stage_out[2]);
    OutArg o_gp = out_arg(ctx, out_grad_params, (size_t)batch * 6 * sizeof(float), ctx->stage_out[3]);
    loss_finalize_kernel<<<1, TL_THREADS, 0, st>>>(ctx->next_buf[2].as<double>(), (int)bpb, batch, d_params, (float*)o_pb.dev,
                                                   (float*)o_gm.dev, (float*)o_gp.dev, (float*)o_loss.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, o_loss);
    finish_out(ctx, o_pb);
    finish_out(ctx, o_gm);
    finish_out(ctx, o_gp);
    PLS_CUDA(cudaStreamSynchronize(st));
    PLS_API_END(ctx)
}

}  // extern "C"
