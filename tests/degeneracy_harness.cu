// Host build of the eigenvalue-thresholded solve of pls_register_scans_degeneracy (eigen_device.cuh), for the CPU
// tests of tests/test_degeneracy_cpu.py: the same __host__ __device__ code the kernels run, behind a C ABI.
#include <stdint.h>

#include "../pylidar_slam_b200/csrc/eigen_device.cuh"

using namespace pls;

extern "C" {

// n symmetric 6x6 matrices H [n,36] -> ascending eigenvalues w [n,6] and eigenvectors as columns V [n,36]
void dh_eigen6(const double* H, int64_t n, double* w, double* V) {
    for (int64_t i = 0; i < n; ++i) {
        double A[36];
        for (int j = 0; j < 36; ++j) A[j] = H[36 * i + j];
        eigen6_jacobi(A, V + 36 * i, w + 6 * i);
    }
}

// n rows of 30 sums -> steps dx [n,6], eigenvalues of H / N [n,6] and the kept counts [n]
void dh_solve6_projected(const double* sums, int64_t n, double min_eigenvalue, double* dx, double* lambda_n,
                         int* kept) {
    for (int64_t i = 0; i < n; ++i) {
        double A[36], V[36];
        kept[i] = solve6_projected(sums + 30 * i, min_eigenvalue, A, V, dx + 6 * i, lambda_n + 6 * i);
    }
}

}  // extern "C"
