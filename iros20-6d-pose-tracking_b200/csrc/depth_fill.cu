// Depth hole filling for live sensors (SURVEY.md 8f row 4): the reference's fill_depth (Utils.py:455-514) as its ROS node
// drives it (predict_ros.py:38-41):  uint16 mm -> metres float32 -> invert (max_depth - d where d > 0.1) -> dilate with a 5x5
// diamond -> close 5x5 -> fill the still-empty pixels from a 7x7 dilation -> median 5x5 -> bilateral (d=5, sigmaColor 1.5,
// sigmaSpace 2.0) -> invert back -> x1000 -> uint16.  The reference calls OpenCV for every stage; the stages here restate
// OpenCV's semantics:
//   dilate / erode   BORDER_CONSTANT with the morphology default border value = outside pixels are ignored
//   medianBlur       BORDER_REPLICATE, exact median of 25
//   bilateralFilter  (float path) BORDER_REFLECT_101; range weight from a 4096-bin exp LUT over [min, max] of the image with
//                    linear interpolation, spatial weights exp(-r^2 / (2 sigma_s^2)) for r <= radius
// Everything up to the median is order-free min / max / selection and is bit-identical to OpenCV; the bilateral sum is float32
// accumulation whose order OpenCV's SIMD code does not expose, so the final metres agree to ~5e-7 and the uint16 millimetres
// to +-1 on the rare pixel that sits on a truncation boundary (tests state both tolerances).
// One thread per pixel, seven small launches per frame (1.2 MB images, L2 resident); latency matters here, not bandwidth.
// Every kernel executes griddepcontrol.launch_dependents at entry: inside a track step that fills the frame (se3tn_track_opts)
// the next launch is preprocess_kernel, launched with programmatic dependent launch, which then becomes resident under the
// last fill kernel's tail and reads the filled frame only after its griddepcontrol.wait.  No fill kernel is itself launched
// with that attribute, so each one starts after the previous launch in the stream has completed.
// The two optional branches of the reference (never used by its ROS node) are here too:
//   extrapolate=True   every column's first valid value is extended to the top of the image, then the remaining empty pixels
//                      take the 31x31 dilation (separable row / column maxima; exact)
//   blur_type='gaussian'  cv2.GaussianBlur(5x5, sigma 0 = the fixed [1 4 6 4 1]/16 kernel, BORDER_REFLECT_101) on the valid
//                      pixels instead of the bilateral filter (float32 row pass then column pass, as OpenCV's separable filter)
#include "depth_fill.h"
#include "ptx.cuh"
#include <cfloat>

namespace se3tn {
namespace {
constexpr int kBX = 32, kBY = 8;

__device__ __forceinline__ float inverted(const uint16_t* __restrict__ in, int idx, float max_depth) {
    const float d = static_cast<float>(static_cast<double>(in[idx]) / 1e3);      // depth / 1e3 in float64, then astype(float32)
    return d > 0.1f ? max_depth - d : d;
}

__global__ void __launch_bounds__(kBX * kBY)
invert_dilate_kernel(const uint16_t* __restrict__ in, float* __restrict__ out, int H, int W, float max_depth)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    float m = -FLT_MAX;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) {
            if (abs(dy) + abs(dx) > 2) continue;                                   // 5x5 diamond
            const int yy = y + dy, xx = x + dx;
            if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
            m = fmaxf(m, inverted(in, yy * W + xx, max_depth));
        }
    out[y * W + x] = m;
}

template <int R, bool ERODE>
__global__ void __launch_bounds__(kBX * kBY)
box_morph_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    float m = ERODE ? FLT_MAX : -FLT_MAX;
    for (int dy = -R; dy <= R; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
#pragma unroll
        for (int dx = -R; dx <= R; ++dx) {
            const int xx = x + dx;
            if (xx < 0 || xx >= W) continue;
            const float v = in[yy * W + xx];
            m = ERODE ? fminf(m, v) : fmaxf(m, v);
        }
    }
    out[y * W + x] = m;
}

// depth[empty] = dilate7x7(depth)[empty], empty = depth < 0.1
__global__ void __launch_bounds__(kBX * kBY)
fill_empty_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    float v = in[y * W + x];
    if (v < 0.1f) {
        float m = -FLT_MAX;
        for (int dy = -3; dy <= 3; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= H) continue;
#pragma unroll
            for (int dx = -3; dx <= 3; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= W) continue;
                m = fmaxf(m, in[yy * W + xx]);
            }
        }
        v = m;
    }
    out[y * W + x] = v;
}

__device__ __forceinline__ unsigned ordered_key(float f) {           // monotone float -> unsigned map (negative values occur beyond max_depth)
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float from_key(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// exact median of the 5x5 window (replicated border) + min / max of the result for the bilateral's range LUT
__global__ void __launch_bounds__(kBX * kBY)
median5_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, unsigned* __restrict__ minmax)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    float med = 0.f;
    const bool live = x < W && y < H;
    if (live) {
        float v[25];
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
            for (int dx = -2; dx <= 2; ++dx) {
                const int yy = min(max(y + dy, 0), H - 1), xx = min(max(x + dx, 0), W - 1);
                v[(dy + 2) * 5 + dx + 2] = in[yy * W + xx];
            }
        // partial selection: after pass k the k smallest values sit in v[0..k]
#pragma unroll
        for (int k = 0; k <= 12; ++k)
#pragma unroll
            for (int j = k + 1; j < 25; ++j) {
                const float a = v[k], b = v[j];
                v[k] = fminf(a, b); v[j] = fmaxf(a, b);
            }
        med = v[12];
        out[y * W + x] = med;
    }
    // block-level min / max, one atomic pair per warp
    unsigned kmin = live ? ordered_key(med) : 0xFFFFFFFFu, kmax = live ? ordered_key(med) : 0u;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, off));
        kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, off));
    }
    if (threadIdx.x == 0) { atomicMin(&minmax[0], kmin); atomicMax(&minmax[1], kmax); }
}

__global__ void init_minmax_kernel(unsigned* minmax) { ptx::grid_dep_launch(); minmax[0] = 0xFFFFFFFFu; minmax[1] = 0u; }

// OpenCV's range LUT: expLUT[i] = exp((i / scale)^2 * gauss_color_coeff), scale = 4096 / float(max - min); zero after underflow
__global__ void lut_kernel(const unsigned* __restrict__ minmax, float* __restrict__ lut, float sigma_color)
{
    ptx::grid_dep_launch();
    const float mn = from_key(minmax[0]), mx = from_key(minmax[1]);
    const float len = static_cast<float>(static_cast<double>(mx) - static_cast<double>(mn));
    const float scale = static_cast<float>(1 << 12) / len;
    const double coeff = -0.5 / (static_cast<double>(sigma_color) * sigma_color);
    for (int i = threadIdx.x; i < kFillLutEntries; i += blockDim.x) {
        const double val = static_cast<double>(static_cast<float>(i) / scale);
        lut[i] = static_cast<float>(exp(val * val * coeff));              // (underflow to 0 happens by itself; OpenCV then stops evaluating)
    }
    if (threadIdx.x == 0) lut[kFillLutEntries] = scale;
}

__global__ void __launch_bounds__(kBX * kBY)
bilateral_finish_kernel(const float* __restrict__ in, const float* __restrict__ lut, const unsigned* __restrict__ minmax,
                        int H, int W, float sigma_space, float max_depth, uint16_t* __restrict__ out_mm, float* __restrict__ out_m)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    const float mn = from_key(minmax[0]), mx = from_key(minmax[1]);
    const float v0 = in[y * W + x];
    float res = v0;
    if (!(fabs(static_cast<double>(mn) - static_cast<double>(mx)) < FLT_EPSILON)) {      // constant image: OpenCV copies the source
        const float scale = lut[kFillLutEntries];
        const double gsc = -0.5 / (static_cast<double>(sigma_space) * sigma_space);
        float sum = 0.f, wsum = 0.f;
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
            for (int dx = -2; dx <= 2; ++dx) {
                const int r2 = dy * dy + dx * dx;
                if (r2 > 4) continue;                                             // r <= radius = 2
                int yy = y + dy, xx = x + dx;                                     // BORDER_REFLECT_101
                if (yy < 0) yy = -yy; if (yy >= H) yy = 2 * H - 2 - yy;
                if (xx < 0) xx = -xx; if (xx >= W) xx = 2 * W - 2 - xx;
                yy = min(max(yy, 0), H - 1); xx = min(max(xx, 0), W - 1);         // images narrower than the radius
                const float v = in[yy * W + xx];
                const float sw = static_cast<float>(exp(static_cast<double>(r2) * gsc));
                float alpha = fabsf(v - v0) * scale;
                const int idx = static_cast<int>(floorf(alpha));
                alpha -= static_cast<float>(idx);
                const float w = sw * (lut[idx] + alpha * (lut[idx + 1] - lut[idx]));
                sum += v * w; wsum += w;
            }
        res = sum / wsum;
    }
    if (res > 0.1f) res = max_depth - res;
    if (out_m) out_m[y * W + x] = res;
    if (out_mm) out_mm[y * W + x] = static_cast<uint16_t>(static_cast<int>(res * 1000.0f));      // (depth * 1000).astype(uint16)
}

// extrapolate: depth[0:top, col] = depth[top, col], top = first row with depth > 0.1 (np.argmax of an all-False column = 0: nothing to do)
__global__ void extrapolate_top_kernel(float* __restrict__ d, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    int top = 0;
    for (int y = 0; y < H; ++y) if (d[y * W + x] > 0.1f) { top = y; break; }
    const float v = d[top * W + x];
    for (int y = 0; y < top; ++y) d[y * W + x] = v;
}

// 31x31 dilation, separable: row maxima ...
__global__ void __launch_bounds__(kBX * kBY)
rowmax31_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    float m = -FLT_MAX;
    for (int dx = -15; dx <= 15; ++dx) { const int xx = x + dx; if (xx >= 0 && xx < W) m = fmaxf(m, in[y * W + xx]); }
    out[y * W + x] = m;
}
// ... then column maxima, written only where the image is still empty (depth < 0.1)
__global__ void __launch_bounds__(kBX * kBY)
large_fill_kernel(const float* __restrict__ rowmax, float* __restrict__ d, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    if (!(d[y * W + x] < 0.1f)) return;
    float m = -FLT_MAX;
    for (int dy = -15; dy <= 15; ++dy) { const int yy = y + dy; if (yy >= 0 && yy < H) m = fmaxf(m, rowmax[yy * W + x]); }
    d[y * W + x] = m;
}

__global__ void __launch_bounds__(kBX * kBY)
median5_plain_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    float v[25];
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) {
            const int yy = min(max(y + dy, 0), H - 1), xx = min(max(x + dx, 0), W - 1);
            v[(dy + 2) * 5 + dx + 2] = in[yy * W + xx];
        }
#pragma unroll
    for (int k = 0; k <= 12; ++k)
#pragma unroll
        for (int j = k + 1; j < 25; ++j) { const float a = v[k], b = v[j]; v[k] = fminf(a, b); v[j] = fmaxf(a, b); }
    out[y * W + x] = v[12];
}

__device__ __forceinline__ int reflect101(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return min(max(i, 0), n - 1);
}
// cv2.GaussianBlur(depth, (5,5), 0): rows then columns with the fixed kernel [1 4 6 4 1]/16 in float32; result only where depth > 0.1
__global__ void __launch_bounds__(kBX * kBY)
gaussian_finish_kernel(const float* __restrict__ in, int H, int W, float max_depth, uint16_t* __restrict__ out_mm, float* __restrict__ out_m)
{
    ptx::grid_dep_launch();
    const int x = blockIdx.x * kBX + threadIdx.x, y = blockIdx.y * kBY + threadIdx.y;
    if (x >= W || y >= H) return;
    const float k0 = 0.375f, k1 = 0.25f, k2 = 0.0625f;
    float res = in[y * W + x];
    if (res > 0.1f) {
        float rows[5];
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy) {
            const float* r = in + reflect101(y + dy, H) * W;
            const float c = r[x], l1 = r[reflect101(x - 1, W)], r1 = r[reflect101(x + 1, W)], l2 = r[reflect101(x - 2, W)], r2 = r[reflect101(x + 2, W)];
            rows[dy + 2] = __fadd_rn(__fadd_rn(__fmul_rn(c, k0), __fmul_rn(__fadd_rn(l1, r1), k1)), __fmul_rn(__fadd_rn(l2, r2), k2));
        }
        res = __fadd_rn(__fadd_rn(__fmul_rn(rows[2], k0), __fmul_rn(__fadd_rn(rows[1], rows[3]), k1)), __fmul_rn(__fadd_rn(rows[0], rows[4]), k2));
    }
    if (res > 0.1f) res = max_depth - res;
    if (out_m) out_m[y * W + x] = res;
    if (out_mm) out_mm[y * W + x] = static_cast<uint16_t>(static_cast<int>(res * 1000.0f));
}
}  // namespace

cudaError_t launch_fill_depth(const uint16_t* depth_mm, int H, int W, float max_depth, bool extrapolate, bool gaussian, const FillScratch& sc,
                              uint16_t* out_mm, float* out_m, cudaStream_t s) {
    if (H <= 0 || W <= 0) return cudaSuccess;
    const dim3 block(kBX, kBY), grid((W + kBX - 1) / kBX, (H + kBY - 1) / kBY);
    invert_dilate_kernel<<<grid, block, 0, s>>>(depth_mm, sc.a, H, W, max_depth);
    box_morph_kernel<2, false><<<grid, block, 0, s>>>(sc.a, sc.b, H, W);            // close = dilate ...
    box_morph_kernel<2, true><<<grid, block, 0, s>>>(sc.b, sc.a, H, W);             // ... then erode
    fill_empty_kernel<<<grid, block, 0, s>>>(sc.a, sc.b, H, W);
    if (extrapolate) {
        extrapolate_top_kernel<<<(W + 127) / 128, 128, 0, s>>>(sc.b, H, W);
        rowmax31_kernel<<<grid, block, 0, s>>>(sc.b, sc.a, H, W);
        large_fill_kernel<<<grid, block, 0, s>>>(sc.a, sc.b, H, W);
    }
    if (gaussian) {
        median5_plain_kernel<<<grid, block, 0, s>>>(sc.b, sc.a, H, W);
        gaussian_finish_kernel<<<grid, block, 0, s>>>(sc.a, H, W, max_depth, out_mm, out_m);
        return cudaGetLastError();
    }
    init_minmax_kernel<<<1, 1, 0, s>>>(sc.minmax);
    median5_kernel<<<grid, block, 0, s>>>(sc.b, sc.a, H, W, sc.minmax);
    lut_kernel<<<1, 256, 0, s>>>(sc.minmax, sc.lut, 1.5f);
    bilateral_finish_kernel<<<grid, block, 0, s>>>(sc.a, sc.lut, sc.minmax, H, W, 2.0f, max_depth, out_mm, out_m);
    return cudaGetLastError();
}

}  // namespace se3tn
