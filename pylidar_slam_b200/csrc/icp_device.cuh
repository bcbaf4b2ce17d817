// Device-side tail of an ICP iteration, shared by the stand-alone step kernels (odometry.cu) and the
// correspondence kernels that finish the iteration in their last block (kdmap.cu).
#pragma once
#include "eigen_device.cuh"
#include "internal.cuh"
#include "pose_device.cuh"

namespace pls {

// Development builds only (-DPLS_KD_SPLIT, tools/kd_residual_split.py): %globaltimer and clock64 stamps of the kd
// residual-and-solve phase, one record of KD_SPLIT_STAMPS (+ as many clock64 words) per block.  The default build
// compiles none of it: PLS_SPLIT_ARG is empty and PLS_SPLIT(...) nothing.
#ifdef PLS_KD_SPLIT
constexpr int KD_SPLIT_STAMPS = 12;
// `dep` only orders the stamp after the value it is given (no instruction of the stamp reads it)
__device__ __forceinline__ unsigned long long split_now(double dep = 0.0) {
    unsigned long long g;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g) : "d"(dep) : "memory");
    return g;
}
__device__ __forceinline__ void split_stamp(unsigned long long* rec, int i, double dep = 0.0) {
    if (!rec) return;
    rec[i] = split_now(dep);
    rec[KD_SPLIT_STAMPS + i] = (unsigned long long)clock64();
}
#define PLS_SPLIT_ARG , unsigned long long* split = nullptr
#define PLS_SPLIT_PASS , split
#define PLS_SPLIT(...) split_stamp(split, __VA_ARGS__)
#else
#define PLS_SPLIT_ARG
#define PLS_SPLIT_PASS
#define PLS_SPLIT(...) \
    do {           \
    } while (0)
#endif

// Deterministic parallel sum of the block partial rows (THREADS = 512, 256 or 128 threads, all must call): slice w of
// eight sums the rows w, w+8, ... of every accumulator (lane = accumulator, so a row is one coalesced 240-byte read and
// the loads of a lane are independent), then the eight slices are added in fixed order -- the same additions in the
// same order whatever the block size (a 128-thread block gives two slices to each warp, a 512-thread block none to
// its last eight).  N: the accumulators per row (NACC, or PLS_EVAL_STATS for pls_kdmap_evaluate_poses's rows), each
// summed exactly as NACC-wide rows sum it.
template <int THREADS = 256, int N = NACC>
__device__ __forceinline__ void sum_partials_256(const double* __restrict__ partials, int num_blocks, double* sums) {
    static_assert(THREADS == 512 || THREADS == 256 || THREADS == 128, "sum_partials: 4, 8 or 16 warps");
    static_assert(N >= 1 && N <= 32, "sum_partials: a lane per accumulator");
    __shared__ double slice_sum[8][N];
    const int a = threadIdx.x & 31;
    if (a < N) {
        for (int slice = threadIdx.x >> 5; slice < 8; slice += THREADS / 32) {
            // sixteen rows in flight per lane (the additions keep their order; a missing row adds +0.0): the sum of a
            // few hundred rows is a chain of L2 round trips otherwise
            double s = 0.0;
            for (int b0 = slice; b0 < num_blocks; b0 += 8 * 16) {
                double v[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int b = b0 + 8 * j;
                    v[j] = b < num_blocks ? __ldcg(partials + (size_t)b * N + a) : 0.0;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) s += v[j];
            }
            slice_sum[slice][a] = s;
        }
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += slice_sum[k][threadIdx.x];
        sums[threadIdx.x] = s;
    }
}

// The eigenvalue-thresholded solve of a registration (pls_register_scans_degeneracy), a launch argument of the kernels
// that finish an iteration: the threshold, and where the iteration writes the registration's ICP_DEGEN_STRIDE doubles --
// the ascending eigenvalues of H / N, then the number of degenerate directions.  Not a FrameResult field: its stride is
// read by the kernels of every other path.
constexpr int ICP_DEGEN_STRIDE = 8;
struct IcpDegen {
    double min_eigenvalue;
    double* out;      // [ICP_DEGEN_STRIDE]
    double* scratch;  // [72] shared memory: the matrix and the eigenvectors of eigen6_jacobi
};

// The serial tail of an ICP iteration (thread 0): Gauss-Newton guards, 6x6 solve, stop test, pose update.
// DEGEN (pls_register_scans_degeneracy): the step is solve6_projected's with dg.min_eigenvalue, in place of solve6's;
// the iteration is singular when its count N is 0 or no direction is kept, instead of when |det| < 1e-7.  Its
// eigenvalues of H / N and degenerate count go to dg.out whatever the iteration's outcome.
template <bool DEGEN = false>
__device__ __forceinline__ void icp_solve_and_update(FrameResult* fr, const double* sums, float threshold_delta PLS_SPLIT_ARG,
                                                     IcpDegen dg = IcpDegen{}) {
    const int it = fr->iters;
    fr->iters = it + 1;
    double dx[6];
    int kept = 0;
    if constexpr (DEGEN) {
        kept = solve6_projected(sums, dg.min_eigenvalue, dg.scratch, dg.scratch + 36, dx, dg.out);
        dg.out[6] = (double)(6 - kept);
        if (!(sums[29] > 0.0)) {  // no match, or no inlier: nothing to solve, and all-zero sums are no fit
            fr->status = PLS_E_SINGULAR;
            fr->done = 1;
            return;
        }
    }
    // optimization.py:323-327: |r| < 1e-7 -> warning, x stays 0, the residuals are r^2.  The ICP loop then sees delta = 0:
    // it breaks if 0 < threshold_delta_pose (icp_odometry.py:292) and otherwise goes on, the pose unchanged
    // (delta_pose_matrix = I, so `new_pose_matrix` only passes through the Euler round trip again)
    if (sqrt(sums[28]) < 1e-7) {
        fr->losses[it] = (float)sums[28];
        fr->status = PLS_W_TINY_RESIDUAL;
        if (0.f < threshold_delta) {
            fr->done = 1;
        } else {
            float prm[6];
            from_pose(fr->T, prm);
            build_pose(prm, fr->T);
            for (int i = 0; i < 6; ++i) fr->params[i] = prm[i];
        }
        return;
    }
    if constexpr (DEGEN) {
        if (kept == 0) {
            fr->status = PLS_E_SINGULAR;
            fr->done = 1;
            return;
        }
    } else {
        const double det = solve6(sums, dx);
        PLS_SPLIT(7, det + dx[0] + dx[5]);
        if (!(fabs(det) >= 1e-7)) {  // optimization.py:334-336
            fr->status = PLS_E_SINGULAR;
            fr->done = 1;
            return;
        }
    }
    fr->losses[it] = (float)sums[27];
    float delta[6];
    float n2 = 0.f;
    for (int i = 0; i < 6; ++i) {
        delta[i] = (float)dx[i];
        n2 += delta[i] * delta[i];
    }
    if (sqrtf(n2) < threshold_delta) {  // icp_odometry.py:292-293: the last delta is not applied
        fr->done = 1;
        PLS_SPLIT(8, n2);
        return;
    }
    float dT[16], Tn[16], prm[6];
    build_pose(delta, dT);
    mat4_mul(dT, fr->T, Tn);
    from_pose(Tn, prm);          // icp_odometry.py:296
    build_pose(prm, fr->T);      // icp_odometry.py:297
    for (int i = 0; i < 6; ++i) fr->params[i] = prm[i];
    PLS_SPLIT(8, prm[5] + fr->T[10]);
}

// K7: normal-equation solve + ICP bookkeeping of one frame, by one 256-thread block: icp_step_kernel (odometry.cu) and,
// one block per sequence, icp_step_batch_kernel (projmap.cu).  num_blocks == 0: `reduced` holds the (all-reduced) sums.
__device__ __forceinline__ void icp_step_body(FrameResult* fr, const double* __restrict__ partials, int num_blocks,
                                              const double* __restrict__ reduced, float threshold_delta) {
    if (fr->done) return;
    __shared__ double sums[NACC];
    if (num_blocks > 0) {
        sum_partials_256(partials, num_blocks, sums);
    } else if (threadIdx.x < NACC) {
        sums[threadIdx.x] = reduced[threadIdx.x];
    }
    __syncthreads();
    if (threadIdx.x < NACC) fr->last_sums[threadIdx.x] = sums[threadIdx.x];
    if (threadIdx.x != 0) return;
    icp_solve_and_update(fr, sums, threshold_delta);
}

// The shared memory of icp_solve_and_update<true>'s eigen-solve.  Owned by this function rather than by the template,
// so that the kernels without DEGEN keep their shared-memory layout and SASS.
__device__ __forceinline__ double* icp_degen_scratch() {
    __shared__ double s_eig[72];
    return s_eig;
}

// Called by every block of a correspondence kernel (512, 256 or 128 threads) after it stored its partial row: the block
// that arrives last of the num_blocks (ticket in fr->pad) sums all rows in the fixed order and runs the solve -- one
// launch and one dependent-launch gap less per ICP iteration than a separate step kernel.
// DEGEN: icp_solve_and_update<true> with dg, its scratch in this block's shared memory (icp_degen_scratch).
template <int THREADS = 256, bool DEGEN = false>
__device__ __forceinline__ void icp_finish_in_last_block(FrameResult* fr, const double* __restrict__ partials, int num_blocks,
                                                         float threshold_delta PLS_SPLIT_ARG, IcpDegen dg = IcpDegen{}) {
    __shared__ int s_last;
    __shared__ double s_sums[NACC];
    if (threadIdx.x == 0) PLS_SPLIT(4);
    __threadfence();  // this block's partial row is visible before its ticket
    __syncthreads();
    if (threadIdx.x == 0) {
        const int ticket = atomicAdd(&fr->pad, 1);
        s_last = ticket == num_blocks - 1;
        PLS_SPLIT(5, (double)ticket);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    sum_partials_256<THREADS>(partials, num_blocks, s_sums);
    __syncthreads();
    if (threadIdx.x < NACC) fr->last_sums[threadIdx.x] = s_sums[threadIdx.x];
    if (threadIdx.x != 0) return;
    PLS_SPLIT(6, s_sums[0] + s_sums[29]);
    fr->pad = 0;
    if constexpr (DEGEN) dg.scratch = icp_degen_scratch();
    icp_solve_and_update<DEGEN>(fr, s_sums, threshold_delta PLS_SPLIT_PASS, dg);
}

}  // namespace pls
