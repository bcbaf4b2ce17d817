// K6/K7 -- point-to-plane (and, behind the same registry, point-to-point) Gauss-Newton alignment on given
// correspondences, for a batch of B >= 1 correspondence sets of N points each (B = 1: pls_align_p2plane / _p2point).
//
//   gn_accumulate_kernel : residual r = n.(R(x) p + t(x) - q), Jacobian row
//                          J = [n, (dR/de_k p).n], robust weight w, and the reduction of the
//                          30 normal-equation accumulators (21 upper JtWJ, 6 JtWr, sum (w r)^2,
//                          sum r^2, count): per-thread fp64 accumulation of fp32 (or fp64) terms,
//                          warp-shuffle then shared-memory block reduction, one partial row per
//                          block (deterministic two-stage sum, no atomics).  A flat grid: each element
//                          owns blocks_per_element consecutive blocks and strides over its points as a
//                          single alignment of N points would.
//   gn_solve_kernel      : one warp per element sums its block partials in fixed order and solves its 6x6
//                          system; the block that finishes last applies the reference's joint rules to the
//                          whole batch (gn_device.cuh: |r| < 1e-7 over all B*N residuals -> warn/stop, any
//                          |det H| < 1e-7 -> error, else x += dx and stop once |dx| over all B*6 < norm_stop).
//
// Replaces PointToPlaneCost.get_residual_fun / get_residual_jac_fun
// (slam/common/optimization.py:356-435), _WLSScheme.weights + the seven cost functions
// (:45-50,61-226), GaussNewton.compute (:296-344) and GaussNewtonPointToPlaneAlignment.align
// (slam/odometry/alignment.py:91-127).  COST_POINT swaps in PointToPointCost's closures (optimization.py:458-541)
// for GaussNewtonPointToPointAlignment.align (alignment.py:144-189); everything after the residual/Jacobian row is
// shared.
#include <climits>

#include "gn_device.cuh"
#include "internal.cuh"
#include "pose_device.cuh"

namespace pls {

namespace {

constexpr int GN_THREADS = 256;
constexpr int GN_SOLVE_THREADS = 256;
constexpr int GN_SOLVE_WARPS = GN_SOLVE_THREADS / 32;  // elements per solve block
enum { COST_PLANE = 0, COST_POINT = 1 };

template <typename T, int COST>
__global__ void __launch_bounds__(GN_THREADS)
gn_accumulate_kernel(const T* __restrict__ ref, const T* __restrict__ tgt, const T* __restrict__ nrm, int64_t n,
                     int blocks_per_element, const GnHead* __restrict__ head, const T* __restrict__ x, int scheme,
                     T sigma, T* __restrict__ loss_out, double* __restrict__ partials) {
    if (head->done) return;
    const int64_t b = blockIdx.x / blocks_per_element;
    const int block = (int)(blockIdx.x - b * blocks_per_element);
    __shared__ T sR[9], st[3], sdR[27];
    if (threadIdx.x == 0) {
        T M[16];
        build_pose(x + 6 * b, M);
        sR[0] = M[0]; sR[1] = M[1]; sR[2] = M[2];
        sR[3] = M[4]; sR[4] = M[5]; sR[5] = M[6];
        sR[6] = M[8]; sR[7] = M[9]; sR[8] = M[10];
        st[0] = M[3]; st[1] = M[7]; st[2] = M[11];
        euler_jacobian(x + 6 * b + 3, sdR);
    }
    __syncthreads();
    double acc[NACC];
#pragma unroll
    for (int a = 0; a < NACC; ++a) acc[a] = 0.0;
    for (int64_t i = (int64_t)block * blockDim.x + threadIdx.x; i < n; i += (int64_t)blocks_per_element * blockDim.x) {
        const int64_t k = b * n + i;
        T p[3] = {tgt[3 * k], tgt[3 * k + 1], tgt[3 * k + 2]};
        T q[3] = {ref[3 * k], ref[3 * k + 1], ref[3 * k + 2]};
        T J[6];
        T r;
        if constexpr (COST == COST_PLANE) {
            T nn[3] = {nrm[3 * k], nrm[3 * k + 1], nrm[3 * k + 2]};
            r = p2plane_residual_jacobian<T>(p, q, nn, sR, st, sdR, J);
        } else {
            r = p2point_residual_jacobian<T>(p, q, sR, st, sdR, J);
        }
        T w = ls_weight<T>(scheme, sigma, r, p, q);
        T wr = r * w;
        if (loss_out) loss_out[k] = wr * wr;
        accumulate_normal_equations<T>(acc, J, w, wr, r);
    }
    block_reduce_store<GN_THREADS>(acc, partials + (size_t)blockIdx.x * NACC);
}

template <typename T>
__global__ void __launch_bounds__(GN_SOLVE_THREADS)
gn_solve_kernel(GnHead* head, T* x, T* dT, GnStep* steps, const double* __restrict__ partials, int64_t batch,
                int blocks_per_element, T norm_stop) {
    if (head->done) return;
    __shared__ GnJoint red[GN_SOLVE_WARPS];
    __shared__ GnStep s_steps[GN_SOLVE_WARPS];
    __shared__ double s_sums[GN_SOLVE_WARPS][NACC];
    __shared__ int s_last, s_status;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // a batch of at most GN_SOLVE_WARPS elements is solved by one block, which keeps the steps in shared memory
    if (gridDim.x == 1) steps = s_steps;
    const int64_t first = (int64_t)blockIdx.x * GN_SOLVE_WARPS;
    const int elems = (int)(batch - first < GN_SOLVE_WARPS ? batch - first : GN_SOLVE_WARPS);
    // Each accumulator of each element: lane-strided rows, then the shuffle-down tree.  Which warp does it does not
    // change the bits, so the work is laid out for latency: with many rows per element the block's warps share the
    // (element, accumulator) pairs; with few, a warp takes one element and keeps all 30 loads of a row in flight.
    if (blocks_per_element > 32) {
        for (int p = warp; p < elems * NACC; p += GN_SOLVE_WARPS) {
            const int e = p / NACC, a = p - e * NACC;
            const double* rows = partials + (size_t)(first + e) * blocks_per_element * NACC;
            double v = 0.0;
            for (int r = lane; r < blocks_per_element; r += 32) v += rows[(size_t)r * NACC + a];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0) s_sums[e][a] = v;
        }
    } else if (warp < elems) {
        const double* rows = partials + (size_t)(first + warp) * blocks_per_element * NACC;
        double sums[NACC];
#pragma unroll
        for (int a = 0; a < NACC; ++a) sums[a] = 0.0;
        for (int r = lane; r < blocks_per_element; r += 32) {
#pragma unroll
            for (int a = 0; a < NACC; ++a) sums[a] += rows[(size_t)r * NACC + a];
        }
#pragma unroll
        for (int a = 0; a < NACC; ++a) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sums[a] += __shfl_down_sync(0xffffffffu, sums[a], o);
            if (lane == 0) s_sums[warp][a] = sums[a];
        }
    }
    __syncthreads();
    if (lane == 0 && warp < elems) {
        GnStep step;
        step.det = solve6(s_sums[warp], step.dx);
        step.r2 = s_sums[warp][28];
        steps[first + warp] = step;
    }
    if (gridDim.x > 1) {
        __threadfence();  // this block's steps are visible before its ticket
        __syncthreads();
        if (threadIdx.x == 0) s_last = atomicAdd(&head->ticket, 1u) == gridDim.x - 1;
        __syncthreads();
        if (!s_last) return;
        __threadfence();
    } else {
        __syncthreads();
    }
    // The last block: no block of this launch read steps[] before this point, so no SM holds a stale copy of it.
    // Joint sums in a fixed order: thread-strided elements, the shuffle-down tree, then the warps in order.
    GnJoint j = {0.0, 0.0, 0};
    gn_joint_reduce<T>(steps, batch, threadIdx.x, GN_SOLVE_THREADS, j);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        j.r2 += __shfl_down_sync(0xffffffffu, j.r2, o);
        j.dx2 += __shfl_down_sync(0xffffffffu, j.dx2, o);
        j.singular |= __shfl_down_sync(0xffffffffu, j.singular, o);
    }
    if (lane == 0) red[warp] = j;
    __syncthreads();
    if (threadIdx.x == 0) {
        GnJoint total = red[0];
        for (int w = 1; w < GN_SOLVE_WARPS; ++w) gn_joint_merge(total, red[w]);
        head->ticket = 0;
        s_status = gn_joint_decide<T>(head, total, norm_stop);
    }
    __syncthreads();
    gn_joint_apply<T>(steps, batch, threadIdx.x, GN_SOLVE_THREADS, s_status, x, dT);
}

// Enqueues all max_iters iterations (a launch after the batch converged exits at once), copies the results out and
// synchronises once.  Returns the status of the last executed iteration; *iters_out (if given) the iterations executed.
template <typename T, int COST>
int align_impl(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t batch, int64_t n, int scheme,
               double sigma, int max_iters, double norm_stop, const void* x0, void* out_dT, void* out_x, void* out_loss,
               int* iters_out) {
    cudaStream_t st = ctx->stream;
    const int64_t rows = batch * n;
    const size_t pts_bytes = (size_t)rows * 3 * sizeof(T);
    const T* d_ref = (const T*)to_device(ctx, ref, pts_bytes, ctx->stage_in[0]);
    const T* d_tgt = (const T*)to_device(ctx, tgt, pts_bytes, ctx->stage_in[1]);
    const T* d_nrm = COST == COST_PLANE ? (const T*)to_device(ctx, nrm, pts_bytes, ctx->stage_in[2]) : nullptr;
    OutArg o_loss = out_arg(ctx, out_loss, (size_t)rows * sizeof(T), ctx->stage_out[0]);

    int64_t bpe = (n + GN_THREADS - 1) / GN_THREADS;
    if (bpe > 2 * kNumSMs) bpe = 2 * kNumSMs;
    if (bpe < 1) bpe = 1;
    PLS_REQUIRE(batch <= INT_MAX / bpe, "pls_align: batch too large for one launch");
    const int blocks_per_element = (int)bpe;

    // x and dT live in the caller's device outputs (or their staging): the solve kernel updates them in place.
    // Scratch: GnHead | steps [B] | x / dT where the caller asked for none.
    OutArg o_dT = out_arg(ctx, out_dT, (size_t)batch * 16 * sizeof(T), ctx->stage_out[1]);
    OutArg o_x = out_arg(ctx, out_x, (size_t)batch * 6 * sizeof(T), ctx->stage_out[2]);
    const size_t steps_off = (sizeof(GnHead) + 15) & ~(size_t)15;
    size_t end = steps_off + (size_t)batch * sizeof(GnStep);
    const size_t x_off = end;
    if (!o_x.dev) end += (size_t)batch * 6 * sizeof(T);
    const size_t dT_off = end;
    if (!o_dT.dev) end += (size_t)batch * 16 * sizeof(T);
    ctx->tmp[0].reserve(end, st);
    char* base = ctx->tmp[0].as<char>();
    GnHead* d_head = reinterpret_cast<GnHead*>(base);
    GnStep* d_steps = reinterpret_cast<GnStep*>(base + steps_off);
    T* d_x = o_x.dev ? (T*)o_x.dev : reinterpret_cast<T*>(base + x_off);
    T* d_dT = o_dT.dev ? (T*)o_dT.dev : reinterpret_cast<T*>(base + dT_off);
    PLS_CUDA(cudaMemsetAsync(d_head, 0, sizeof(GnHead), st));
    if (x0) PLS_CUDA(cudaMemcpyAsync(d_x, x0, (size_t)batch * 6 * sizeof(T), cudaMemcpyDefault, st));
    else PLS_CUDA(cudaMemsetAsync(d_x, 0, (size_t)batch * 6 * sizeof(T), st));

    ctx->partials.reserve((size_t)batch * blocks_per_element * NACC * sizeof(double), st);
    const int grid = (int)(batch * blocks_per_element);
    const int solve_grid = (int)((batch + GN_SOLVE_WARPS - 1) / GN_SOLVE_WARPS);
    const int iters = max_iters < 1 ? 1 : max_iters;
    for (int it = 0; it < iters; ++it) {
        {
            ProfileScope ps(ctx, 5, (double)rows * (COST == COST_PLANE ? 9 : 6) * sizeof(T) + (double)grid * NACC * 8.0);
            gn_accumulate_kernel<T, COST><<<grid, GN_THREADS, 0, st>>>(d_ref, d_tgt, d_nrm, n, blocks_per_element, d_head,
                                                                       d_x, scheme, (T)sigma, (T*)o_loss.dev,
                                                                       ctx->partials.as<double>());
            PLS_CHECK_LAUNCH();
        }
        gn_solve_kernel<T><<<solve_grid, GN_SOLVE_THREADS, 0, st>>>(d_head, d_x, d_dT, d_steps, ctx->partials.as<double>(),
                                                                   batch, blocks_per_element, (T)norm_stop);
        PLS_CHECK_LAUNCH();
    }
    GnHead h_head;
    PLS_CUDA(cudaMemcpyAsync(&h_head, d_head, sizeof(h_head), cudaMemcpyDeviceToHost, st));
    finish_out(ctx, o_dT);
    finish_out(ctx, o_x);
    finish_out(ctx, o_loss);
    PLS_CUDA(cudaStreamSynchronize(st));
    if (iters_out) *iters_out = h_head.iters;
    return h_head.status;
}

template <int COST>
int align_dispatch(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t batch, int64_t n,
                   int is_f64, int scheme, double sigma, int max_iters, double norm_stop, const void* x0, void* out_dT,
                   void* out_x, void* out_loss, int* out_iters) {
    const int status =
        is_f64 ? align_impl<double, COST>(ctx, ref, tgt, nrm, batch, n, scheme, sigma, max_iters, norm_stop, x0, out_dT,
                                          out_x, out_loss, out_iters)
               : align_impl<float, COST>(ctx, ref, tgt, nrm, batch, n, scheme, sigma, max_iters, norm_stop, x0, out_dT,
                                         out_x, out_loss, out_iters);
    if (status == PLS_E_SINGULAR) throw pls::Error{PLS_E_SINGULAR, "Invalid Jacobian in Gauss Newton minimization"};
    if (status == PLS_W_TINY_RESIDUAL) ctx->err = "The residual norm is lower than threshold 1e-7";
    return status;
}

__global__ void pose_build_kernel(const float* params, int batch, float* out) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) build_pose(params + 6 * b, out + 16 * b);
}
__global__ void pose_from_kernel(const float* mats, int batch, float* out) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) from_pose(mats + 16 * b, out + 6 * b);
}

}  // namespace
}  // namespace pls

using namespace pls;

extern "C" {

int pls_align_p2plane(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t n, int is_f64,
                      int scheme, double sigma, int max_iters, double norm_stop, const void* x0, void* out_dT,
                      void* out_x, void* out_loss) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(ref && tgt && nrm && n > 0, "pls_align_p2plane: ref/tgt/nrm must be [n,3] with n > 0");
    PLS_REQUIRE(scheme >= 0 && scheme <= PLS_SCHEME_CAUCHY, "pls_align_p2plane: unknown weighting scheme");
    return align_dispatch<COST_PLANE>(ctx, ref, tgt, nrm, 1, n, is_f64, scheme, sigma, max_iters, norm_stop, x0, out_dT,
                                      out_x, out_loss, nullptr);
    PLS_API_END(ctx)
}

int pls_align_p2point(pls_context* ctx, const void* ref, const void* tgt, int64_t n, int is_f64, int scheme, double sigma,
                      int max_iters, double norm_stop, const void* x0, void* out_dT, void* out_x, void* out_loss) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(ref && tgt && n > 0, "pls_align_p2point: ref/tgt must be [n,3] with n > 0");
    PLS_REQUIRE(scheme >= 0 && scheme <= PLS_SCHEME_CAUCHY, "pls_align_p2point: unknown weighting scheme");
    return align_dispatch<COST_POINT>(ctx, ref, tgt, nullptr, 1, n, is_f64, scheme, sigma, max_iters, norm_stop, x0,
                                      out_dT, out_x, out_loss, nullptr);
    PLS_API_END(ctx)
}

int pls_align_p2plane_batch(pls_context* ctx, const void* ref, const void* tgt, const void* nrm, int64_t batch, int64_t n,
                            int is_f64, int scheme, double sigma, int max_iters, double norm_stop, const void* x0,
                            void* out_dT, void* out_x, void* out_loss, int* out_iters) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(ref && tgt && nrm && batch > 0 && n > 0,
                "pls_align_p2plane_batch: ref/tgt/nrm must be [batch,n,3] with batch > 0 and n > 0");
    PLS_REQUIRE(scheme >= 0 && scheme <= PLS_SCHEME_CAUCHY, "pls_align_p2plane_batch: unknown weighting scheme");
    return align_dispatch<COST_PLANE>(ctx, ref, tgt, nrm, batch, n, is_f64, scheme, sigma, max_iters, norm_stop, x0,
                                      out_dT, out_x, out_loss, out_iters);
    PLS_API_END(ctx)
}

int pls_align_p2point_batch(pls_context* ctx, const void* ref, const void* tgt, int64_t batch, int64_t n, int is_f64,
                            int scheme, double sigma, int max_iters, double norm_stop, const void* x0, void* out_dT,
                            void* out_x, void* out_loss, int* out_iters) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(ref && tgt && batch > 0 && n > 0,
                "pls_align_p2point_batch: ref/tgt must be [batch,n,3] with batch > 0 and n > 0");
    PLS_REQUIRE(scheme >= 0 && scheme <= PLS_SCHEME_CAUCHY, "pls_align_p2point_batch: unknown weighting scheme");
    return align_dispatch<COST_POINT>(ctx, ref, tgt, nullptr, batch, n, is_f64, scheme, sigma, max_iters, norm_stop, x0,
                                      out_dT, out_x, out_loss, out_iters);
    PLS_API_END(ctx)
}

int pls_build_pose_matrix(pls_context* ctx, const float* params, int batch, float* out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(params && out && batch > 0, "pls_build_pose_matrix: bad arguments");
    const float* d_in = (const float*)to_device(ctx, params, (size_t)batch * 6 * sizeof(float), ctx->stage_in[0]);
    OutArg o = out_arg(ctx, out, (size_t)batch * 16 * sizeof(float), ctx->stage_out[0]);
    pose_build_kernel<<<(batch + 63) / 64, 64, 0, ctx->stream>>>(d_in, batch, (float*)o.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_from_pose_matrix(pls_context* ctx, const float* mats, int batch, float* out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(mats && out && batch > 0, "pls_from_pose_matrix: bad arguments");
    const float* d_in = (const float*)to_device(ctx, mats, (size_t)batch * 16 * sizeof(float), ctx->stage_in[0]);
    OutArg o = out_arg(ctx, out, (size_t)batch * 6 * sizeof(float), ctx->stage_out[0]);
    pose_from_kernel<<<(batch + 63) / 64, 64, 0, ctx->stream>>>(d_in, batch, (float*)o.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

}  // extern "C"
