// Closed-form tail of the Procrustes registration, host/device so that the CPU test-suite can exercise the exact
// code the solve kernel runs (tests/test_abi.py builds a host harness with nvcc).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace pls {

// One-sided (Hestenes) cyclic Jacobi SVD of a 3x3 (float64): plane rotations J of column pairs make the columns of
// B = C V mutually orthogonal, so B = U diag(s) with s[k] = |B e_k| and the columns of V orthonormal.  Working on C
// itself rather than on C^T C keeps the small singular directions accurate to eps / (relative gap): squaring C squares
// its condition number, and the eigen-decomposition of C^T C loses the rotation about the long axis of an elongated
// cloud once sigma_2 / sigma_1 falls below ~1e-3.
__host__ __device__ inline void svd3_one_sided(const double C[3][3], double B[3][3], double V[3][3], double s[3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            B[i][j] = C[i][j];
            V[i][j] = (i == j) ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 32; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0.0, beta = 0.0, gamma = 0.0;
                for (int k = 0; k < 3; ++k) {
                    alpha += B[k][p] * B[k][p];
                    beta += B[k][q] * B[k][q];
                    gamma += B[k][p] * B[k][q];
                }
                if (!(fabs(gamma) > 1e-17 * sqrt(alpha * beta))) continue;  // orthogonal to working precision (or zero)
                rotated = true;
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(zeta * zeta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double bkp = B[k][p], bkq = B[k][q];
                    B[k][p] = c * bkp - sn * bkq;
                    B[k][q] = sn * bkp + c * bkq;
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - sn * vkq;
                    V[k][q] = sn * vkp + c * vkq;
                }
            }
        if (!rotated) break;
    }
    for (int k = 0; k < 3; ++k) s[k] = sqrt(B[0][k] * B[0][k] + B[1][k] * B[1][k] + B[2][k] * B[2][k]);
}

// R = U diag(1, 1, sign(det U det V)) V^T of the cross-covariance C (row-major, reference rows x target columns),
// t = mu_r - R mu_t; mu = (mu_t, mu_r).  Registration.py:48-73.
__host__ __device__ inline void kabsch_from_cross(const double* C9, const double* mu, double* out_T /*[16]*/) {
    double Cm[3][3], B[3][3], V[3][3], d[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Cm[i][j] = C9[3 * i + j];
    svd3_one_sided(Cm, B, V, d);
    // order the singular triplets by descending singular value (LAPACK's order)
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = i + 1; j < 3; ++j)
            if (d[o[j]] > d[o[i]]) { const int t = o[i]; o[i] = o[j]; o[j] = t; }
    double v[3][3], u[3][3];  // v[k] = k-th right singular vector, u[k] = k-th left singular vector
    for (int k = 0; k < 3; ++k)
        for (int i = 0; i < 3; ++i) v[k][i] = V[i][o[k]];
    for (int k = 0; k < 2; ++k) {
        for (int i = 0; i < 3; ++i) u[k][i] = B[i][o[k]];  // = sigma_k u_k
        if (k == 1) {  // Gram-Schmidt against u_0: the columns of B are orthogonal only up to rounding
            const double dp = u[1][0] * u[0][0] + u[1][1] * u[0][1] + u[1][2] * u[0][2];
            for (int i = 0; i < 3; ++i) u[1][i] -= dp * u[0][i];
        }
        const double nrm = sqrt(u[k][0] * u[k][0] + u[k][1] * u[k][1] + u[k][2] * u[k][2]);
        for (int i = 0; i < 3; ++i) u[k][i] /= nrm;
    }
    const double detV = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) - v[0][1] * (v[1][0] * v[2][2] - v[1][2] * v[2][0]) +
                        v[0][2] * (v[1][0] * v[2][1] - v[1][1] * v[2][0]);
    const double sg = detV < 0.0 ? -1.0 : 1.0;
    u[2][0] = sg * (u[0][1] * u[1][2] - u[0][2] * u[1][1]);
    u[2][1] = sg * (u[0][2] * u[1][0] - u[0][0] * u[1][2]);
    u[2][2] = sg * (u[0][0] * u[1][1] - u[0][1] * u[1][0]);
    double R[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = u[0][i] * v[0][j] + u[1][i] * v[1][j] + u[2][i] * v[2][j];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) out_T[4 * i + j] = R[i][j];
        out_T[4 * i + 3] = mu[3 + i] - (R[i][0] * mu[0] + R[i][1] * mu[1] + R[i][2] * mu[2]);
    }
    out_T[12] = 0.0; out_T[13] = 0.0; out_T[14] = 0.0; out_T[15] = 1.0;
}

}  // namespace pls
