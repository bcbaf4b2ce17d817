// Weighted Procrustes / Kabsch rigid registration of two corresponding clouds -- the optional initialiser of the
// point-to-point alignment (GNPointToPointConfig.initialize_with_svd, slam/odometry/alignment.py:170-171) and a
// stand-alone helper (SURVEY.md section 8f rank 2).
//
// Replaces weighted_procrustes, numpy path (slam/common/registration.py:15-76):
//   mu_t = sum w p_t / sum w,  mu_r = sum w p_r / sum w          (the weights only enter the centroids)
//   C    = sum (p_r - mu_r)(p_t - mu_t)^T                          float64, UNWEIGHTED (:44-46)
//   C = U S V^T;  R = U diag(1, 1, sign(det U det V)) V^T;  t = mu_r - R mu_t
//
//   procrustes_moments_kernel : sum w, sum w p_t, sum w p_r  -> one float64 partial row per block
//   procrustes_cross_kernel   : every block folds the moment partials in its prologue, then accumulates the 9
//                               entries of C in float64 (warp shuffle + shared-memory block reduction)
//   procrustes_solve_kernel   : one warp sums the C partials in fixed order; thread 0 runs a one-sided cyclic-Jacobi
//                               SVD of C itself (float64; C^T C would square its condition number), takes u_1, u_2
//                               of the two largest singular values, and closes the frame with u_3 = det(V) u_1 x u_2 -- identical to
//                               U diag(1, 1, +-1) V^T whenever the SVD is unique, and well defined for planar clouds
//                               (sigma_3 = 0) where LAPACK's u_3 is arbitrary up to the same sign rule.
//
// HBM-bound: two streaming passes over 24 (+4) bytes per correspondence.
#include "internal.cuh"
#include "registration_device.cuh"

namespace pls {

namespace {

constexpr int PR_THREADS = 256;

template <int NV>
__device__ __forceinline__ void block_reduce_rows(double* v, double* out) {
    __shared__ double red[PR_THREADS / 32][NV];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < NV; ++a) {
        const double s = warp_sum(v[a]);
        if (lane == 0) red[warp][a] = s;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < PR_THREADS / 32; ++w) s += red[w][threadIdx.x];
        out[threadIdx.x] = s;
    }
    __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(PR_THREADS)
procrustes_moments_kernel(const T* __restrict__ tgt, const T* __restrict__ ref, const T* __restrict__ w, int64_t n,
                          double* __restrict__ partials /*[blocks][7]*/) {
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double wi = w ? (double)w[i] : 1.0;
        acc[0] += wi;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            acc[1 + c] += wi * (double)tgt[3 * i + c];
            acc[4 + c] += wi * (double)ref[3 * i + c];
        }
    }
    block_reduce_rows<7>(acc, partials + 7 * (size_t)blockIdx.x);
}

template <typename T>
__global__ void __launch_bounds__(PR_THREADS)
procrustes_cross_kernel(const T* __restrict__ tgt, const T* __restrict__ ref, int64_t n,
                        const double* __restrict__ moments, int num_moment_rows, double* __restrict__ mu_out /*[6]*/,
                        double* __restrict__ partials /*[blocks][9]*/) {
    __shared__ double s_mu[7];
    {
        double m[7] = {0, 0, 0, 0, 0, 0, 0};
        for (int b = threadIdx.x; b < num_moment_rows; b += PR_THREADS)
#pragma unroll
            for (int a = 0; a < 7; ++a) m[a] += moments[7 * (size_t)b + a];
        block_reduce_rows<7>(m, s_mu);
    }
    const double sw = s_mu[0];
    const double mt[3] = {s_mu[1] / sw, s_mu[2] / sw, s_mu[3] / sw};
    const double mr[3] = {s_mu[4] / sw, s_mu[5] / sw, s_mu[6] / sw};
    if (blockIdx.x == 0 && threadIdx.x < 3) {
        mu_out[threadIdx.x] = mt[threadIdx.x];
        mu_out[3 + threadIdx.x] = mr[threadIdx.x];
    }
    double acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double dt[3] = {(double)tgt[3 * i] - mt[0], (double)tgt[3 * i + 1] - mt[1], (double)tgt[3 * i + 2] - mt[2]};
        const double dr[3] = {(double)ref[3 * i] - mr[0], (double)ref[3 * i + 1] - mr[1], (double)ref[3 * i + 2] - mr[2]};
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) acc[3 * a + b] += dr[a] * dt[b];
    }
    block_reduce_rows<9>(acc, partials + 9 * (size_t)blockIdx.x);
}

__global__ void procrustes_solve_kernel(const double* __restrict__ partials, int num_rows, const double* __restrict__ mu,
                                        double* __restrict__ out_T /*[16]*/) {
    __shared__ double sC[9];
    const int lane = threadIdx.x;
    if (lane < 9) {
        double s = 0.0;
        for (int b = 0; b < num_rows; ++b) s += partials[9 * (size_t)b + lane];
        sC[lane] = s;
    }
    __syncwarp();
    if (lane == 0) kabsch_from_cross(sC, mu, out_T);
}

template <typename T>
void procrustes_impl(pls_context* ctx, const void* tgt, const void* ref, const void* w, int64_t n, double* out_dev) {
    cudaStream_t st = ctx->stream;
    int64_t b = (n + PR_THREADS - 1) / PR_THREADS;
    const int blocks = (int)(b < 1 ? 1 : (b > 4 * kNumSMs ? 4 * kNumSMs : b));
    ctx->next_buf[4].reserve((size_t)blocks * 7 * sizeof(double), st);
    ctx->next_buf[5].reserve((size_t)blocks * 9 * sizeof(double), st);
    ctx->next_buf[6].reserve(6 * sizeof(double), st);
    procrustes_moments_kernel<T><<<blocks, PR_THREADS, 0, st>>>((const T*)tgt, (const T*)ref, (const T*)w, n,
                                                                ctx->next_buf[4].as<double>());
    PLS_CHECK_LAUNCH();
    procrustes_cross_kernel<T><<<blocks, PR_THREADS, 0, st>>>((const T*)tgt, (const T*)ref, n, ctx->next_buf[4].as<double>(),
                                                              blocks, ctx->next_buf[6].as<double>(), ctx->next_buf[5].as<double>());
    PLS_CHECK_LAUNCH();
    procrustes_solve_kernel<<<1, 32, 0, st>>>(ctx->next_buf[5].as<double>(), blocks, ctx->next_buf[6].as<double>(), out_dev);
    PLS_CHECK_LAUNCH();
}

}  // namespace
}  // namespace pls

using namespace pls;

extern "C" {

int pls_weighted_procrustes(pls_context* ctx, const void* tgt, const void* ref, const void* weights, int64_t n, int is_f64,
                            double* out_T) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(tgt && ref && out_T && n > 0, "pls_weighted_procrustes: need two [n,3] clouds");
    const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
    const void* d_t = to_device(ctx, tgt, (size_t)n * 3 * esz, ctx->stage_in[0]);
    const void* d_r = to_device(ctx, ref, (size_t)n * 3 * esz, ctx->stage_in[1]);
    const void* d_w = weights ? to_device(ctx, weights, (size_t)n * esz, ctx->stage_in[2]) : nullptr;
    OutArg o = out_arg(ctx, out_T, 16 * sizeof(double), ctx->stage_out[0]);
    if (is_f64) procrustes_impl<double>(ctx, d_t, d_r, d_w, n, (double*)o.dev);
    else procrustes_impl<float>(ctx, d_t, d_r, d_w, n, (double*)o.dev);
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

}  // extern "C"
