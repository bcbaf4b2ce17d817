// Spherical projection device math (slam/common/projection.py:11-73,393-401), float32 in the
// reference's operation order.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace pls {

struct ProjConst {
    int H, W;
    float Hf, Wf;
    float abs_down;  // |fov_down| in radians, rounded to float like the torch scalar
    float fov;       // |fov_down| + |fov_up|
};

inline ProjConst make_proj_const(int H, int W, float up_deg, float down_deg) {
    ProjConst pc;
    pc.H = H;
    pc.W = W;
    double up = (double)up_deg / 180.0 * 3.141592653589793;
    double down = (double)down_deg / 180.0 * 3.141592653589793;
    pc.abs_down = (float)fabs(down);
    pc.fov = (float)(fabs(down) + fabs(up));
    pc.Wf = (float)W;
    pc.Hf = (float)H;
    return pc;
}

#ifdef __CUDACC__
// Explicitly rounded arithmetic.  On the device each helper is one PTX instruction with .rn rounding, which the compiler
// never contracts into an FMA, so every kernel that calls a helper below gets the same bits: two kernels that must agree
// on a range or a moved point (a z-buffer and the test of its winner, a single and a batched call) agree by construction.
// They are written as PTX rather than as the __fmul_rn family of intrinsics, which emit the same instructions but reach
// the optimizer as calls that stop it hoisting shared-memory pose loads out of the loops that use them.  On the host the
// helpers are the plain operations, fmaf and sqrtf.
#ifdef __CUDA_ARCH__
#define PLS_RN(T, C, op, ...) \
    T r;                      \
    asm(op : "=" C(r) : __VA_ARGS__); \
    return r;
__device__ __forceinline__ float mul_rn(float a, float b) { PLS_RN(float, "f", "mul.rn.f32 %0, %1, %2;", "f"(a), "f"(b)) }
__device__ __forceinline__ float add_rn(float a, float b) { PLS_RN(float, "f", "add.rn.f32 %0, %1, %2;", "f"(a), "f"(b)) }
__device__ __forceinline__ float fma_rn(float a, float b, float c) {
    PLS_RN(float, "f", "fma.rn.f32 %0, %1, %2, %3;", "f"(a), "f"(b), "f"(c))
}
__device__ __forceinline__ float div_rn(float a, float b) { PLS_RN(float, "f", "div.rn.f32 %0, %1, %2;", "f"(a), "f"(b)) }
__device__ __forceinline__ float sqrt_rn(float a) { PLS_RN(float, "f", "sqrt.rn.f32 %0, %1;", "f"(a)) }
__device__ __forceinline__ double mul_rn(double a, double b) { PLS_RN(double, "d", "mul.rn.f64 %0, %1, %2;", "d"(a), "d"(b)) }
__device__ __forceinline__ double add_rn(double a, double b) { PLS_RN(double, "d", "add.rn.f64 %0, %1, %2;", "d"(a), "d"(b)) }
__device__ __forceinline__ double fma_rn(double a, double b, double c) {
    PLS_RN(double, "d", "fma.rn.f64 %0, %1, %2, %3;", "d"(a), "d"(b), "d"(c))
}
__device__ __forceinline__ double div_rn(double a, double b) { PLS_RN(double, "d", "div.rn.f64 %0, %1, %2;", "d"(a), "d"(b)) }
__device__ __forceinline__ double sqrt_rn(double a) { PLS_RN(double, "d", "sqrt.rn.f64 %0, %1;", "d"(a)) }
#undef PLS_RN
#else
inline float mul_rn(float a, float b) { return a * b; }
inline float add_rn(float a, float b) { return a + b; }
inline float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float div_rn(float a, float b) { return a / b; }
inline float sqrt_rn(float a) { return sqrtf(a); }
#endif

// Which square seeds the range's sum: sqrt(fma(z, z, fma(x, x, y y))) or sqrt(fma(z, z, fma(y, y, x x))).  The two differ
// in the last ulp, and a range one ulp off can change a z-buffer winner, so a z-buffer and every test of its winners use
// one order.  kYFirst, the projections' default, is the order of every z-buffer but the query z-buffers of projmap.cu;
// each kernel keeps the order its z-buffer has always had, so that no winner moves.
enum class RangeOrder { kYFirst, kXFirst };

template <typename T>
__host__ __device__ __forceinline__ T range_rn(T x, T y, T z, RangeOrder order) {
    const T a = order == RangeOrder::kYFirst ? y : x, b = order == RangeOrder::kYFirst ? x : y;
    return sqrt_rn(fma_rn(z, z, fma_rn(b, b, mul_rn(a, a))));
}

// p = T p0, T the first three rows of a row-major 4x4 pose, each row rounded as fma(z, T2, fma(x, T0, y T1)) + T3.
__host__ __device__ __forceinline__ void transform_point(const float* T, const float4& p0, float* p) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
        p[c] = add_rn(fma_rn(p0.z, T[4 * c + 2], fma_rn(p0.x, T[4 * c], mul_rn(p0.y, T[4 * c + 1]))), T[4 * c + 3]);
}

// Float pixel coordinates as torch__spherical_projection returns them: (-1,-1) for the null point.
__host__ __device__ __forceinline__ void project_point(float x, float y, float z, const ProjConst& pc, float& row, float& col,
                                                       float& r_out, RangeOrder order = RangeOrder::kYFirst) {
    const float kPi = 3.14159274101257324f;  // float(np.pi)
    const float r = range_rn(x, y, z, order);
    r_out = r;
    const bool null = (r == 0.0f);
    const float rr = null ? 0.001f : r;
    const float theta = -atan2f(y, x);
    const float phi = asinf(div_rn(z, rr));
    const float c = mul_rn(mul_rn(0.5f, add_rn(div_rn(theta, kPi), 1.0f)), pc.Wf);
    const float rw = mul_rn(add_rn(1.0f, -div_rn(add_rn(phi, pc.abs_down), pc.fov)), pc.Hf);
    row = null ? -1.0f : rw;
    col = null ? -1.0f : c;
}

// Rounded pixel index + validity (projection.py:393-401,408).  False for NaN / null / out of image.
__host__ __device__ __forceinline__ bool project_to_pixel(float x, float y, float z, const ProjConst& pc, int& pix, float& r,
                                                          RangeOrder order = RangeOrder::kYFirst) {
    float row, col;
    project_point(x, y, z, pc, row, col, r, order);
    float pr = rintf(row), pcn = rintf(col);
    bool ok = (pr >= 0.0f) && (pr <= (float)(pc.H - 1)) && (pcn >= 0.0f) && (pcn <= (float)(pc.W - 1)) && (r > 0.0f);
    if (!ok) return false;
    pix = (int)pr * pc.W + (int)pcn;
    return true;
}
#endif

}  // namespace pls
