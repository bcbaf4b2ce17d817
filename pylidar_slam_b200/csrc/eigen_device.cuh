// Smallest-eigenvalue direction of a symmetric 3x3 matrix: the normal of a map point from the second moments of its
// neighbourhood (replaces np.linalg.svd(covs)[2][:, 2, :], slam/odometry/local_map.py:414-416; the sign of the vector
// is arbitrary there and irrelevant downstream: J^T J and J^T r are even in the normal).
//
// Two solvers in float64 (the reference's LAPACK sgesdd works in float32, so both are more accurate than what they
// stand in for):
//   * closed form: eigenvalues by the trigonometric solution of the characteristic cubic, the vector as the largest
//     cross product of two rows of (A - lambda I).  ~300 instructions, no loop.  Accurate to ~eps * lambda_max / gap,
//     gap = lambda_mid - lambda_min: used when the gap is at least 1e-3 of the spectrum;
//   * cyclic Jacobi: unconditionally stable, ~6x the instructions: the fall-back for nearly degenerate
//     neighbourhoods (lines, isotropic blobs), where the direction is ill-defined anyway.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace pls {

__host__ __device__ inline void smallest_eigenvector_jacobi(const float* c /*xx,xy,xz,yy,yz,zz*/, float* n) {
    double A[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 12; ++sweep) {
        double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        double diag = fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2]);
        if (off <= 1e-18 * diag || off == 0.0) break;
#pragma unroll
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0;
            const int q = pq == 0 ? 1 : 2;
            double apq = A[p][q];
            if (apq == 0.0) continue;
            double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
            double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                double akp = A[k][p], akq = A[k][q];
                A[k][p] = cs * akp - sn * akq;
                A[k][q] = sn * akp + cs * akq;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                double apk = A[p][k], aqk = A[q][k];
                A[p][k] = cs * apk - sn * aqk;
                A[q][k] = sn * apk + cs * aqk;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = cs * vkp - sn * vkq;
                V[k][q] = sn * vkp + cs * vkq;
            }
        }
    }
    int m = 0;
    if (A[1][1] < A[m][m]) m = 1;
    if (A[2][2] < A[m][m]) m = 2;
    double nx = V[0][m], ny = V[1][m], nz = V[2][m];
    double inv = 1.0 / sqrt(nx * nx + ny * ny + nz * nz);
    n[0] = (float)(nx * inv);
    n[1] = (float)(ny * inv);
    n[2] = (float)(nz * inv);
}

// Returns false when the closed form should not be trusted (caller falls back to Jacobi).
__host__ __device__ inline bool smallest_eigenvector_closed_form(const float* c, float* n) {
    const double a = c[0], b = c[1], cc = c[2], d = c[3], e = c[4], f = c[5];
    const double q = (a + d + f) / 3.0;
    const double p1 = b * b + cc * cc + e * e;
    const double aq = a - q, dq = d - q, fq = f - q;
    const double p2 = aq * aq + dq * dq + fq * fq + 2.0 * p1;
    if (!(p2 > 0.0)) return false;  // isotropic (or NaN)
    const double p = sqrt(p2 / 6.0);
    const double ip = 1.0 / p;
    // r = det((A - q I) / p) / 2 in [-1, 1]
    const double b11 = aq * ip, b22 = dq * ip, b33 = fq * ip, b12 = b * ip, b13 = cc * ip, b23 = e * ip;
    double r = 0.5 * (b11 * (b22 * b33 - b23 * b23) - b12 * (b12 * b33 - b23 * b13) + b13 * (b12 * b23 - b22 * b13));
    r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
    const double phi = acos(r) / 3.0;
    const double lmax = q + 2.0 * p * cos(phi);
    const double lmin = q + 2.0 * p * cos(phi + 2.0943951023931953);  // + 2 pi / 3
    const double lmid = 3.0 * q - lmax - lmin;
    if (!((lmid - lmin) > 1e-3 * (lmax - lmin))) return false;  // plane direction nearly degenerate
    // rows of A - lmin I; the eigenvector is orthogonal to all of them: take the best-conditioned cross product
    const double r0[3] = {a - lmin, b, cc}, r1[3] = {b, d - lmin, e}, r2[3] = {cc, e, f - lmin};
    const double c01[3] = {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]};
    const double c02[3] = {r0[1] * r2[2] - r0[2] * r2[1], r0[2] * r2[0] - r0[0] * r2[2], r0[0] * r2[1] - r0[1] * r2[0]};
    const double c12[3] = {r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0]};
    const double n01 = c01[0] * c01[0] + c01[1] * c01[1] + c01[2] * c01[2];
    const double n02 = c02[0] * c02[0] + c02[1] * c02[1] + c02[2] * c02[2];
    const double n12 = c12[0] * c12[0] + c12[1] * c12[1] + c12[2] * c12[2];
    const double* v = c01;
    double nn = n01;
    if (n02 > nn) { v = c02; nn = n02; }
    if (n12 > nn) { v = c12; nn = n12; }
    if (!(nn > 0.0)) return false;
    const double inv = 1.0 / sqrt(nn);
    n[0] = (float)(v[0] * inv);
    n[1] = (float)(v[1] * inv);
    n[2] = (float)(v[2] * inv);
    return true;
}

__host__ __device__ inline void smallest_eigenvector(const float* c, float* n) {
    if (!smallest_eigenvector_closed_form(c, n)) smallest_eigenvector_jacobi(c, n);
}

// Eigen-decomposition of a symmetric 6x6 matrix by cyclic Jacobi in float64: A [36] (row-major, both triangles) is
// overwritten, V [36] receives the eigenvectors as columns and w [6] the eigenvalues, ascending (V's columns in the
// same order).  The normal-equation matrix J^T W J of a registration is what it is for: its translation and rotation
// entries differ by the square of the scene's radius, and its degenerate directions have eigenvalues at or near 0.
//   * rotation order: the pairs (p, q), p < q, row by row, in every sweep;
//   * a pair is skipped, its entry set to 0, when |a_pq| <= 2^-53 sqrt(|a_pp|) sqrt(|a_qq|) (0 when a diagonal entry is
//     0).  This relative rule keeps the small eigenvalues of a positive semi-definite matrix accurate to their own size
//     (Demmel and Veselic, "Jacobi's method is more accurate than QR", 1992), so a tiny eigenvalue of a strongly scaled
//     matrix is not drowned by the rounding of its large ones;
//   * it stops after the first sweep that rotates nothing, or after EIGEN6_SWEEPS sweeps;
//   * ties in the ordering keep the lower index first.
// A and V are pointers so that a device caller can keep them in shared memory: in registers, one thread's 72 doubles
// would spill under a 128-register cap.  The same code on the same inputs gives the same bits on every call.
constexpr int EIGEN6_SWEEPS = 30;
__host__ __device__ inline void eigen6_jacobi(double* A, double* V, double* w) {
    for (int i = 0; i < 36; ++i) V[i] = (i % 7 == 0) ? 1.0 : 0.0;
#pragma unroll 1
    for (int sweep = 0; sweep < EIGEN6_SWEEPS; ++sweep) {
        bool rotated = false;
#pragma unroll 1
        for (int p = 0; p < 5; ++p) {
#pragma unroll 1
            for (int q = p + 1; q < 6; ++q) {
                const double apq = A[p * 6 + q];
                if (apq == 0.0) continue;
                const double app = A[p * 6 + p], aqq = A[q * 6 + q];
                if (fabs(apq) <= 0x1p-53 * (sqrt(fabs(app)) * sqrt(fabs(aqq)))) {
                    A[p * 6 + q] = 0.0;
                    A[q * 6 + p] = 0.0;
                    continue;
                }
                rotated = true;
                // the rotation that zeroes a_pq (t = tan of its angle, the smaller root)
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta
                                                     : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                A[p * 6 + p] = app - t * apq;
                A[q * 6 + q] = aqq + t * apq;
                A[p * 6 + q] = 0.0;
                A[q * 6 + p] = 0.0;
#pragma unroll 1
                for (int r = 0; r < 6; ++r) {
                    if (r != p && r != q) {
                        const double arp = A[r * 6 + p], arq = A[r * 6 + q];
                        const double np = c * arp - s * arq, nq = s * arp + c * arq;
                        A[r * 6 + p] = np;
                        A[p * 6 + r] = np;
                        A[r * 6 + q] = nq;
                        A[q * 6 + r] = nq;
                    }
                    const double vrp = V[r * 6 + p], vrq = V[r * 6 + q];
                    V[r * 6 + p] = c * vrp - s * vrq;
                    V[r * 6 + q] = s * vrp + c * vrq;
                }
            }
        }
        if (!rotated) break;
    }
    // insertion sort of the diagonal, V's columns with it: stable, so equal eigenvalues keep their order
#pragma unroll 1
    for (int i = 1; i < 6; ++i)
#pragma unroll 1
        for (int j = i; j > 0 && A[j * 7] < A[(j - 1) * 7]; --j) {
            const double d = A[j * 7];
            A[j * 7] = A[(j - 1) * 7];
            A[(j - 1) * 7] = d;
            for (int r = 0; r < 6; ++r) {
                const double v = V[r * 6 + j];
                V[r * 6 + j] = V[r * 6 + j - 1];
                V[r * 6 + j - 1] = v;
            }
        }
    for (int k = 0; k < 6; ++k) w[k] = A[k * 7];
}

// The Gauss-Newton step of an ICP iteration restricted to the directions the map constrains (Zhang, Kaess and Singh,
// "On degeneracy of optimization-based state estimation problems", ICRA 2016, whose solution remapping is this
// truncated eigen-solve for a step taken from the current pose).  sums: the 30 accumulators of the iteration (21 upper
// entries of H = J^T W J, g = J^T W r, ..., the count N in sums[29]).  With (lambda_k, v_k) the eigen-pairs of H
// (eigen6_jacobi), direction k is kept when N > 0 and lambda_k >= min_eigenvalue * N, and
//   dx = -sum over the kept k, ascending, of v_k (v_k^T g) / lambda_k.
// Returns the number of kept directions (0: dx is all zeros); lambda_n [6] receives the ascending eigenvalues of H / N
// (zeros when N = 0).  A, V: [36] scratch, as eigen6_jacobi's.
__host__ __device__ inline int solve6_projected(const double* sums, double min_eigenvalue, double* A, double* V,
                                                double* dx, double* lambda_n) {
    {
        int k = 0;
        for (int i = 0; i < 6; ++i)
            for (int j = i; j < 6; ++j) {
                A[i * 6 + j] = sums[k];
                A[j * 6 + i] = sums[k];
                ++k;
            }
    }
    eigen6_jacobi(A, V, lambda_n);  // H's eigenvalues, divided by N below
    const double N = sums[29];
    const double thr = min_eigenvalue * N;
    for (int i = 0; i < 6; ++i) dx[i] = 0.0;
    int kept = 0;
    for (int k = 0; k < 6; ++k) {
        const double w = lambda_n[k];
        lambda_n[k] = N > 0.0 ? w / N : 0.0;
        if (!(N > 0.0 && w >= thr)) continue;
        ++kept;
        double vg = 0.0;
        for (int i = 0; i < 6; ++i) vg += V[i * 6 + k] * sums[21 + i];
        const double a = vg / w;
        for (int i = 0; i < 6; ++i) dx[i] -= V[i * 6 + k] * a;
    }
    return kept;
}

}  // namespace pls
