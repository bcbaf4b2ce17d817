// K2 -- spherical range-image projection with a closest-wins z-buffer.
//
//   pixel math     : r = |p|, theta = -atan2(y, x), phi = asin(z / r),
//                    col = W * 0.5 (theta/pi + 1), row = H (1 - (phi + |fov_down|)/fov), float32
//                    in the reference's operation order (slam/common/projection.py:11-73).
//   zbuf_kernel    : rounds half-to-even, keeps 0 <= row <= H-1, 0 <= col <= W-1, r > 0 and does
//                    one 64-bit atomicMin of (float_bits(r) << 32 | point index) per point --
//                    the closest point per pixel wins, lowest index on exact range ties.  This is
//                    the deterministic form of "sort by descending range, scatter"
//                    (projection.py:393-415).
//   resolve_kernel : one thread per pixel gathers the winner's C channels into the planar
//                    [B,C,H,W] image; empty pixels are 0.
#include "internal.cuh"
#include "projection_device.cuh"

namespace pls {

namespace {

__global__ void project_pixels_kernel(const float* __restrict__ xyz, int64_t n, ProjConst pc,
                                      float* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float row, col, r;
        project_point(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], pc, row, col, r, RangeOrder::kYFirst);
        out[2 * i] = row;
        out[2 * i + 1] = col;
    }
}

__global__ void zbuf_kernel(const float* __restrict__ xyz, int batch, int64_t n, ProjConst pc,
                            unsigned long long* __restrict__ zbuf) {
    const int64_t total = (int64_t)batch * n;
    const int64_t hw = (int64_t)pc.H * pc.W;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t b = g / n, i = g - b * n;
        int pix;
        float r;
        if (project_to_pixel(xyz[3 * g], xyz[3 * g + 1], xyz[3 * g + 2], pc, pix, r, RangeOrder::kYFirst)) {
            unsigned long long key = ((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)i;
            atomicMin(&zbuf[b * hw + pix], key);
        }
    }
}

__global__ void zbuf_points_kernel(const float* __restrict__ xyz, int64_t n, const uint32_t* __restrict__ n_dev, ProjConst pc,
                                   unsigned long long* __restrict__ zbuf) {
    if (n_dev) n = min(n, (int64_t)*n_dev);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int pix;
        float r;
        // the order FrameInputSelect::flags tests this z-buffer's winners with
        if (project_to_pixel(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], pc, pix, r, RangeOrder::kYFirst))
            atomicMin(&zbuf[pix], ((unsigned long long)__float_as_uint(r) << 32) | (unsigned long long)(uint32_t)i);
    }
}

__global__ void resolve_kernel(const unsigned long long* __restrict__ zbuf, const float* __restrict__ values,
                               int batch, int64_t n, int C, int64_t hw, float fill, float* __restrict__ out) {
    const int64_t total = (int64_t)batch * hw;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t b = g / hw, pix = g - b * hw;
        unsigned long long key = zbuf[g];
        float* o = out + (size_t)b * C * hw + pix;
        if (key == ~0ull) {
            for (int c = 0; c < C; ++c) o[(size_t)c * hw] = fill;  // projection.py:378-391: the image starts as default_value
        } else {
            const float* v = values + ((size_t)b * n + (uint32_t)(key & 0xffffffffull)) * C;
            for (int c = 0; c < C; ++c) o[(size_t)c * hw] = v[c];
        }
    }
}

// ---- float64 clouds ----------------------------------------------------------------------------------------------
// With a float64 `input_data` / `numpy_pc` (what the de-skew filter produces) the reference runs the whole projection in
// float64 -- pixel coordinates, rounding, the range the z-buffer sorts by -- and only rounds the finished vertex map to
// float32 (icp_odometry.py:331-352).  Same arithmetic here; a 64-bit range leaves no room for the point index in the
// atomic word, so the winner is found in two passes: the smallest range per pixel, then the lowest index having it.
struct ProjConst64 {
    int H, W;
    double Hf, Wf, abs_down, fov;
};

__device__ __forceinline__ bool project_to_pixel_f64(double x, double y, double z, const ProjConst64& pc, int& pix, double& r) {
    const double kPi = 3.141592653589793;  // np.pi
    r = range_rn(x, y, z, RangeOrder::kYFirst);
    const bool null = (r == 0.0);
    const double rr = null ? 0.001 : r;
    const double theta = -atan2(y, x);
    const double phi = asin(div_rn(z, rr));
    const double c = mul_rn(mul_rn(0.5, add_rn(div_rn(theta, kPi), 1.0)), pc.Wf);
    const double rw = mul_rn(add_rn(1.0, -div_rn(add_rn(phi, pc.abs_down), pc.fov)), pc.Hf);
    const double pr = rint(null ? -1.0 : rw), pcn = rint(null ? -1.0 : c);
    const bool ok = (pr >= 0.0) && (pr <= (double)(pc.H - 1)) && (pcn >= 0.0) && (pcn <= (double)(pc.W - 1)) && (r > 0.0);
    if (!ok) return false;
    pix = (int)pr * pc.W + (int)pcn;
    return true;
}

__global__ void zbuf_range_f64_kernel(const double* __restrict__ xyz, int64_t n, ProjConst64 pc,
                                      unsigned long long* __restrict__ zrange) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int pix;
        double r;
        if (project_to_pixel_f64(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], pc, pix, r))
            atomicMin(&zrange[pix], (unsigned long long)__double_as_longlong(r));  // r > 0: bit order == value order
    }
}

__global__ void zbuf_index_f64_kernel(const double* __restrict__ xyz, int64_t n, ProjConst64 pc,
                                      const unsigned long long* __restrict__ zrange, unsigned int* __restrict__ zindex) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int pix;
        double r;
        if (project_to_pixel_f64(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], pc, pix, r) &&
            (unsigned long long)__double_as_longlong(r) == zrange[pix])
            atomicMin(&zindex[pix], (unsigned int)i);
    }
}

template <typename TO>
__global__ void resolve_f64_kernel(const unsigned int* __restrict__ zindex, const double* __restrict__ xyz, int64_t hw,
                                   TO* __restrict__ out) {
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < hw; pix += (int64_t)gridDim.x * blockDim.x) {
        const unsigned int i = zindex[pix];
        const bool empty = (i == 0xffffffffu);
        out[pix] = empty ? (TO)0 : (TO)xyz[3 * (size_t)i];
        out[hw + pix] = empty ? (TO)0 : (TO)xyz[3 * (size_t)i + 1];
        out[2 * hw + pix] = empty ? (TO)0 : (TO)xyz[3 * (size_t)i + 2];
    }
}

inline int grid_for(int64_t n, int threads = 256) {
    int64_t b = (n + threads - 1) / threads;
    int64_t cap = 16 * kNumSMs;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

void launch_projection(pls_context* ctx, const float* xyz, const float* channels, int batch, int64_t n, int C, int H,
                       int W, float up, float down, float* out, unsigned long long* zbuf, float fill) {
    cudaStream_t st = ctx->stream;
    const int64_t hw = (int64_t)H * W;
    PLS_REQUIRE(n < (1ll << 32), "projection: at most 2^32 points per cloud");
    ProjConst pc = make_proj_const(H, W, up, down);
    PLS_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)batch * hw * sizeof(unsigned long long), st));
    if (n > 0) {
        zbuf_kernel<<<grid_for((int64_t)batch * n), 256, 0, st>>>(xyz, batch, n, pc, zbuf);
        PLS_CHECK_LAUNCH();
    }
    resolve_kernel<<<grid_for((int64_t)batch * hw), 256, 0, st>>>(zbuf, channels ? channels : xyz, batch, n, C, hw, fill, out);
    PLS_CHECK_LAUNCH();
}

void launch_zbuf_points(pls_context* ctx, const float* xyz, int64_t n, const uint32_t* n_dev, int H, int W, float up, float down,
                        unsigned long long* zbuf) {
    PLS_REQUIRE(n > 0 && n < (1ll << 32), "projection: 1 .. 2^32 points per cloud");
    zbuf_points_kernel<<<grid_for(n), 256, 0, ctx->stream>>>(xyz, n, n_dev, make_proj_const(H, W, up, down), zbuf);
    PLS_CHECK_LAUNCH();
}

template <typename TO>
static void launch_projection_f64_impl(pls_context* ctx, const double* xyz, int64_t n, int H, int W, float up, float down, TO* out,
                                       unsigned long long* zbuf) {
    cudaStream_t st = ctx->stream;
    const int64_t hw = (int64_t)H * W;
    PLS_REQUIRE(n < 0xffffffffll, "projection: at most 2^32 - 1 points per cloud");
    ProjConst64 pc;
    pc.H = H;
    pc.W = W;
    pc.Hf = (double)H;
    pc.Wf = (double)W;
    // fov_up = up / 180.0 * np.pi etc. in Python floats (projection.py:47-49)
    pc.abs_down = fabs((double)down / 180.0 * 3.141592653589793);
    pc.fov = pc.abs_down + fabs((double)up / 180.0 * 3.141592653589793);
    // zbuf holds hw 64-bit range words; the 32-bit winner indices live in the scratch of the stateless filters
    ctx->next_buf[7].reserve((size_t)hw * sizeof(unsigned int), st);
    unsigned int* zindex = ctx->next_buf[7].as<unsigned int>();
    PLS_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)hw * sizeof(unsigned long long), st));
    PLS_CUDA(cudaMemsetAsync(zindex, 0xff, (size_t)hw * sizeof(unsigned int), st));
    if (n > 0) {
        zbuf_range_f64_kernel<<<grid_for(n), 256, 0, st>>>(xyz, n, pc, zbuf);
        PLS_CHECK_LAUNCH();
        zbuf_index_f64_kernel<<<grid_for(n), 256, 0, st>>>(xyz, n, pc, zbuf, zindex);
        PLS_CHECK_LAUNCH();
    }
    resolve_f64_kernel<TO><<<grid_for(hw), 256, 0, st>>>(zindex, xyz, hw, out);
    PLS_CHECK_LAUNCH();
}

void launch_projection_f64(pls_context* ctx, const double* xyz, int64_t n, int H, int W, float up, float down, float* out,
                           unsigned long long* zbuf) {
    launch_projection_f64_impl<float>(ctx, xyz, n, H, W, up, down, out, zbuf);
}

// the float64 vertex map itself (what a float64 cloud gives build_projection_map: the dataset loaders' case)
void launch_projection_f64_out64(pls_context* ctx, const double* xyz, int64_t n, int H, int W, float up, float down, double* out,
                                 unsigned long long* zbuf) {
    launch_projection_f64_impl<double>(ctx, xyz, n, H, W, up, down, out, zbuf);
}

}  // namespace pls

using namespace pls;

extern "C" {

int pls_project_pixels(pls_context* ctx, const float* xyz, int64_t n, int height, int width, float up_fov_deg,
                       float down_fov_deg, float* rows_cols_out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(xyz && rows_cols_out && n > 0 && height > 0 && width > 0, "pls_project_pixels: bad arguments");
    const float* d = (const float*)to_device(ctx, xyz, (size_t)n * 3 * sizeof(float), ctx->stage_in[0]);
    OutArg o = out_arg(ctx, rows_cols_out, (size_t)n * 2 * sizeof(float), ctx->stage_out[0]);
    project_pixels_kernel<<<grid_for(n), 256, 0, ctx->stream>>>(d, n, make_proj_const(height, width, up_fov_deg, down_fov_deg),
                                                               (float*)o.dev);
    PLS_CHECK_LAUNCH();
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

static int build_projection_map_impl(pls_context* ctx, const float* xyz, const float* channels, int batch, int64_t n,
                                     int num_channels, int height, int width, float up_fov_deg, float down_fov_deg,
                                     float default_value, float* out) {
    PLS_API_BEGIN(ctx)
    PLS_REQUIRE(xyz && out && batch > 0 && n >= 0 && height > 0 && width > 0, "pls_build_projection_map: bad arguments");
    const int C = channels ? num_channels : 3;
    PLS_REQUIRE(C >= 1 && C <= 64, "pls_build_projection_map: 1..64 channels");
    const int64_t hw = (int64_t)height * width;
    const float* d_xyz = (const float*)to_device(ctx, xyz, (size_t)batch * n * 3 * sizeof(float), ctx->stage_in[0]);
    const float* d_ch = (const float*)to_device(ctx, channels, (size_t)batch * n * C * sizeof(float), ctx->stage_in[1]);
    OutArg o = out_arg(ctx, out, (size_t)batch * C * hw * sizeof(float), ctx->stage_out[0]);
    ctx->tmp[3].reserve((size_t)batch * hw * sizeof(unsigned long long), ctx->stream);
    launch_projection(ctx, d_xyz, d_ch, batch, n, C, height, width, up_fov_deg, down_fov_deg, (float*)o.dev,
                      ctx->tmp[3].as<unsigned long long>(), default_value);
    finish_out(ctx, o);
    PLS_CUDA(cudaStreamSynchronize(ctx->stream));
    PLS_API_END(ctx)
}

int pls_build_projection_map(pls_context* ctx, const float* xyz, const float* channels, int batch, int64_t n,
                             int num_channels, int height, int width, float up_fov_deg, float down_fov_deg,
                             float* out) {
    return build_projection_map_impl(ctx, xyz, channels, batch, n, num_channels, height, width, up_fov_deg, down_fov_deg, 0.f,
                                     out);
}

int pls_build_projection_map_filled(pls_context* ctx, const float* xyz, const float* channels, int batch, int64_t n,
                                    int num_channels, int height, int width, float up_fov_deg, float down_fov_deg,
                                    float default_value, float* out) {
    return build_projection_map_impl(ctx, xyz, channels, batch, n, num_channels, height, width, up_fov_deg, down_fov_deg,
                                     default_value, out);
}

}  // extern "C"
