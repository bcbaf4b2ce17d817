// Per-correspondence device math of the point-to-plane Gauss-Newton step, shared by the
// stand-alone alignment kernel (gn.cu) and the fused correspondence+reduction kernels
// (kdmap.cu, projmap.cu); and the joint rules of the stand-alone alignment's batched solve.
#pragma once
#include <cuda_runtime.h>

#include "../../include/plslam_b200.h"
#include "pose_device.cuh"

namespace pls {

constexpr int NACC_DEV = 30;

// r = n . (R p + t - q);  J = [n, (dR_k p) . n]   (slam/common/optimization.py:381-394,424-433)
template <typename T>
__host__ __device__ __forceinline__ T p2plane_residual_jacobian(const T* p, const T* q, const T* n, const T* R, const T* t,
                                                       const T* dR, T* J) {
    T tp0 = p[0] * R[0] + p[1] * R[1] + p[2] * R[2] + t[0];
    T tp1 = p[0] * R[3] + p[1] * R[4] + p[2] * R[5] + t[1];
    T tp2 = p[0] * R[6] + p[1] * R[7] + p[2] * R[8] + t[2];
    T r = (tp0 - q[0]) * n[0] + (tp1 - q[1]) * n[1] + (tp2 - q[2]) * n[2];
    J[0] = n[0];
    J[1] = n[1];
    J[2] = n[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const T* D = dR + 9 * k;
        T v0 = D[0] * p[0] + D[1] * p[1] + D[2] * p[2];
        T v1 = D[3] * p[0] + D[4] * p[1] + D[5] * p[2];
        T v2 = D[6] * p[0] + D[7] * p[1] + D[8] * p[2];
        J[3 + k] = v0 * n[0] + v1 * n[1] + v2 * n[2];
    }
    return r;
}

// At x = 0 (every ICP iteration): R = I, t = 0, J = [n, p x n]; same values, fewer flops.
__device__ __forceinline__ float p2plane_residual_jacobian_identity(const float* p, const float* q, const float* n,
                                                                   float* J) {
    float r = (p[0] - q[0]) * n[0] + (p[1] - q[1]) * n[1] + (p[2] - q[2]) * n[2];
    J[0] = n[0];
    J[1] = n[1];
    J[2] = n[2];
    J[3] = p[1] * n[2] - p[2] * n[1];
    J[4] = p[2] * n[0] - p[0] * n[2];
    J[5] = p[0] * n[1] - p[1] * n[0];
    return r;
}

// Point-to-point cost (slam/common/optimization.py:458-541): r = |d|, d = R p + t - q, and the Jacobian AS THE
// REFERENCE WRITES IT (:485-501): J[k] = (dT/dx_k p~) . d = [d, (dR_k p) . d] -- that is r * dr/dx, the gradient of
// r^2 / 2, not dr/dx.  Restated faithfully: the drop-in must return what the reference returns.
template <typename T>
__host__ __device__ __forceinline__ T p2point_residual_jacobian(const T* p, const T* q, const T* R, const T* t, const T* dR,
                                                       T* J) {
    T d0 = p[0] * R[0] + p[1] * R[1] + p[2] * R[2] + t[0] - q[0];
    T d1 = p[0] * R[3] + p[1] * R[4] + p[2] * R[5] + t[1] - q[1];
    T d2 = p[0] * R[6] + p[1] * R[7] + p[2] * R[8] + t[2] - q[2];
    J[0] = d0;
    J[1] = d1;
    J[2] = d2;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const T* D = dR + 9 * k;
        T v0 = D[0] * p[0] + D[1] * p[1] + D[2] * p[2];
        T v1 = D[3] * p[0] + D[4] * p[1] + D[5] * p[2];
        T v2 = D[6] * p[0] + D[7] * p[1] + D[8] * p[2];
        J[3 + k] = v0 * d0 + v1 * d1 + v2 * d2;
    }
    return sqrt(d0 * d0 + d1 * d1 + d2 * d2);
}

// w = sqrt(cost(r)) / max(|r|, 1e-4)   (optimization.py:45-50 and the cost functions :61-208)
template <typename T>
__host__ __device__ __forceinline__ T ls_weight(int scheme, T sigma, T r, const T* p, const T* q) {
    if (scheme == PLS_SCHEME_DEFAULT || scheme == PLS_SCHEME_LEAST_SQUARE) return (T)1;
    T a = fabs(r);
    T cost;
    switch (scheme) {
        case PLS_SCHEME_HUBER:
            cost = (a < sigma) ? r * r : ((T)2 * sigma * a - sigma * sigma);
            break;
        case PLS_SCHEME_EXP:
            cost = (r * r) * exp(-(r * r) / (sigma * sigma));
            break;
        case PLS_SCHEME_NEIGHBORHOOD: {
            T dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
            T d = sqrt(dx * dx + dy * dy + dz * dz);
            cost = r * r * exp(-(d * d) / (sigma * sigma));
            break;
        }
        case PLS_SCHEME_GEMAN_MCCLURE: {
            T r2 = r * r;
            cost = sigma * r2 / (sigma + r2);
            break;
        }
        case PLS_SCHEME_SQUARE_GEMAN_MCCLURE: {
            T r2 = r * r;
            T f = sigma / (sigma + r2);
            cost = r2 * (f * f);
            break;
        }
        default: {  // PLS_SCHEME_CAUCHY
            T s = r / sigma;
            cost = log((T)1 + s * s);
            break;
        }
    }
    T clamped = a < (T)1e-4 ? (T)1e-4 : a;
    return sqrt(cost) / clamped;
}

// acc += [ (wJ)(wJ)^T upper, (wJ)(wr), (wr)^2, r^2, 1 ] with fp64 accumulation
template <typename T>
__device__ __forceinline__ void accumulate_normal_equations(double* acc, const T* J, T w, T wr, T r) {
    double wj[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) wj[a] = (double)(J[a] * w);
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) acc[k++] += wj[a] * wj[b];
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += wj[a] * (double)wr;
    acc[27] += (double)wr * (double)wr;
    acc[28] += (double)r * (double)r;
    acc[29] += 1.0;
}

// Warp-shuffle + shared-memory block reduction of the N (30, or PLS_EVAL_STATS for the evaluation's rows) accumulators;
// thread a < N of the block writes the block total of accumulator a to out[a].  Only the first WARPS warps hold
// accumulators (a block whose extra warps only search skips them); every thread of the block must call.
template <int THREADS, int WARPS = THREADS / 32, int N = NACC_DEV>
__device__ __forceinline__ void block_reduce_store(double* acc, double* out) {
    static_assert(WARPS >= 1 && WARPS <= THREADS / 32, "block_reduce_store: warps");
    static_assert(N >= 1 && N <= 32, "block_reduce_store: one warp of accumulators");
    __shared__ double red[WARPS][N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (WARPS == THREADS / 32 || warp < WARPS) {  // warp-uniform; always true (no branch) when every warp holds some
#pragma unroll
        for (int a = 0; a < N; ++a) {
            double v = acc[a];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][a] = v;
        }
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) s += red[w][threadIdx.x];
        out[threadIdx.x] = s;
    }
}

// ---- the joint rules of a batched Gauss-Newton iteration (optimization.py:318-341) -----------------------------------
// GaussNewton.compute treats the B elements of a batch as one problem: the tiny-residual guard looks at the norm of all
// B*N residuals, one singular element fails the whole call, and the stop test looks at the norm of all B*6 increments.
// Each element's own 6x6 solve is a GnStep; the functions below turn the B steps into the joint decision and apply it.
// They are shared by gn_solve_kernel (gn.cu) and the host harness of the CPU tests.

struct GnStep {          // one element's solve: H dx = -g, det H, and its sum of unweighted r^2
    double dx[6];
    double det;
    double r2;
};

struct GnHead {          // the batch-wide state of one alignment call
    double dx_norm;      // |dx| over all elements of the last applied step
    int done;            // latched: later iterations are no-ops
    int status;          // PLS_OK, PLS_W_TINY_RESIDUAL or PLS_E_SINGULAR
    int iters;           // iterations executed
    unsigned ticket;     // blocks of the current solve launch that have finished their elements
};

struct GnJoint {         // joint sums: sum r^2 over B*N residuals, sum dx^2 over B*6 increments (as stored in T)
    double r2;
    double dx2;
    int singular;
};

// Adds elements first, first + stride, ... < batch to j, in that order.
template <typename T>
__host__ __device__ inline void gn_joint_reduce(const GnStep* steps, int64_t batch, int64_t first, int64_t stride,
                                                GnJoint& j) {
    for (int64_t b = first; b < batch; b += stride) {
        const GnStep& s = steps[b];
        j.r2 += s.r2;
        double e = 0.0;
        for (int i = 0; i < 6; ++i) {
            const T d = (T)s.dx[i];
            e += (double)d * (double)d;
        }
        j.dx2 += e;
        if (!(fabs(s.det) >= 1e-7)) j.singular = 1;
    }
}

__host__ __device__ inline void gn_joint_merge(GnJoint& a, const GnJoint& b) {
    a.r2 += b.r2;
    a.dx2 += b.dx2;
    a.singular |= b.singular;
}

// The reference's order: tiny residual (warn, x unchanged), then any singular element (raise), then the update and the
// joint stop test.  Returns the status of this iteration; only PLS_OK lets gn_joint_apply move x.
template <typename T>
__host__ __device__ inline int gn_joint_decide(GnHead* head, const GnJoint& j, T norm_stop) {
    head->iters += 1;
    int status = PLS_OK;
    if (sqrt(j.r2) < 1e-7) status = PLS_W_TINY_RESIDUAL;
    else if (j.singular) status = PLS_E_SINGULAR;
    if (status != PLS_OK) {
        head->status = status;
        head->done = 1;
        return status;
    }
    head->dx_norm = sqrt(j.dx2);
    if (head->dx_norm < (double)norm_stop) head->done = 1;
    return status;
}

// Elements first, first + stride, ...: x += (T)dx when the step is taken (status PLS_OK), and dT = pose(x).
template <typename T>
__host__ __device__ inline void gn_joint_apply(const GnStep* steps, int64_t batch, int64_t first, int64_t stride,
                                               int status, T* x /*[B,6]*/, T* dT /*[B,16]*/) {
    for (int64_t b = first; b < batch; b += stride) {
        T* xb = x + 6 * b;
        if (status == PLS_OK)
            for (int i = 0; i < 6; ++i) xb[i] = xb[i] + (T)steps[b].dx[i];
        build_pose(xb, dT + 16 * b);
    }
}

}  // namespace pls
