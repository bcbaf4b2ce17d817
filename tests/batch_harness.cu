// TEST INFRASTRUCTURE ONLY -- host harness around the batched alignment's joint rules (gn_device.cuh).
//
// gn.cu's solve kernel turns the B per-element solves of an iteration into the reference's joint decision with
// gn_joint_reduce / gn_joint_decide / gn_joint_apply, __host__ __device__ functions.  This file runs them on the CPU
// behind a tiny C ABI, with the per-element terms of gn_device.cuh accumulated sequentially, so that
// tests/test_batched_alignment_cpu.py can check the very rules the kernel applies against the goldens of the
// unmodified reference without a GPU.  It is never linked into libplslam_b200.so.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../pylidar_slam_b200/csrc/gn_device.cuh"
#include "../pylidar_slam_b200/csrc/pose_device.cuh"

using namespace pls;

namespace {

// one element's 30 accumulators at x (gn_accumulate_kernel's per-point terms, summed in point order)
template <typename T>
void element_sums(int cost, const T* ref, const T* tgt, const T* nrm, int64_t n, int scheme, T sigma, const T* x,
                  double* acc, T* loss) {
    T M[16], R[9], t[3], dR[27];
    build_pose(x, M);
    R[0] = M[0]; R[1] = M[1]; R[2] = M[2]; R[3] = M[4]; R[4] = M[5]; R[5] = M[6]; R[6] = M[8]; R[7] = M[9]; R[8] = M[10];
    t[0] = M[3]; t[1] = M[7]; t[2] = M[11];
    euler_jacobian(x + 3, dR);
    for (int a = 0; a < NACC_DEV; ++a) acc[a] = 0.0;
    for (int64_t i = 0; i < n; ++i) {
        const T* p = tgt + 3 * i;
        const T* q = ref + 3 * i;
        T J[6];
        const T r = cost == 0 ? p2plane_residual_jacobian<T>(p, q, nrm + 3 * i, R, t, dR, J)
                              : p2point_residual_jacobian<T>(p, q, R, t, dR, J);
        const T w = ls_weight<T>(scheme, sigma, r, p, q);
        const T wr = r * w;
        if (loss) loss[i] = wr * wr;
        double wj[6];
        for (int a = 0; a < 6; ++a) wj[a] = (double)(J[a] * w);
        int k = 0;
        for (int a = 0; a < 6; ++a)
            for (int b = a; b < 6; ++b) acc[k++] += wj[a] * wj[b];
        for (int a = 0; a < 6; ++a) acc[21 + a] += wj[a] * (double)wr;
        acc[27] += (double)wr * (double)wr;
        acc[28] += (double)r * (double)r;
        acc[29] += 1.0;
    }
}

template <typename T>
int align_batch_host(int cost, const T* ref, const T* tgt, const T* nrm, int64_t B, int64_t n, int scheme, T sigma,
                     int max_iters, T norm_stop, const T* x0, T* x, T* dT, T* loss, int* iters) {
    GnHead head;
    memset(&head, 0, sizeof(head));
    for (int64_t i = 0; i < B * 6; ++i) x[i] = x0 ? x0[i] : (T)0;
    std::vector<GnStep> steps(B);
    double acc[NACC_DEV];
    for (int it = 0; it < (max_iters < 1 ? 1 : max_iters) && !head.done; ++it) {
        for (int64_t b = 0; b < B; ++b) {
            element_sums<T>(cost, ref + 3 * n * b, tgt + 3 * n * b, nrm ? nrm + 3 * n * b : nullptr, n, scheme, sigma,
                            x + 6 * b, acc, loss + n * b);
            steps[b].det = solve6(acc, steps[b].dx);
            steps[b].r2 = acc[28];
        }
        GnJoint j = {0.0, 0.0, 0};
        gn_joint_reduce<T>(steps.data(), B, 0, 1, j);
        const int status = gn_joint_decide<T>(&head, j, norm_stop);
        gn_joint_apply<T>(steps.data(), B, 0, 1, status, x, dT);
    }
    *iters = head.iters;
    return head.status;
}

}  // namespace

extern "C" int bh_align_batch(int cost, int is_f64, const void* ref, const void* tgt, const void* nrm, int64_t B,
                              int64_t n, int scheme, double sigma, int max_iters, double norm_stop, const void* x0,
                              void* x, void* dT, void* loss, int* iters) {
    if (is_f64)
        return align_batch_host<double>(cost, (const double*)ref, (const double*)tgt, (const double*)nrm, B, n, scheme,
                                        sigma, max_iters, norm_stop, (const double*)x0, (double*)x, (double*)dT,
                                        (double*)loss, iters);
    return align_batch_host<float>(cost, (const float*)ref, (const float*)tgt, (const float*)nrm, B, n, scheme,
                                   (float)sigma, max_iters, (float)norm_stop, (const float*)x0, (float*)x, (float*)dT,
                                   (float*)loss, iters);
}
