// The reference's train-time augmentations of input B on the device (data_augmentation.py:48-121, 217-267): two launches per
// batch.  augment_draws_kernel forms each pair's draws and BlackCover's corner from whole-image counts of maskB;
// augment_pixels_kernel runs HSVJitter -> ChangeBright -> GaussianNoise pointwise and GaussianBlur -> BlackCover over a band of
// rows.  The arithmetic is augment.cuh's.
#include "augment.h"
#include "launch.h"

namespace se3tn {
namespace {

using namespace aug;

constexpr int kDrawThreads = 512;

__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, unsigned long long* acc) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(acc, v);
    return v;
}

__global__ void __launch_bounds__(kDrawThreads) augment_draws_kernel(Config cfg, const uint16_t* __restrict__ depthB,
                                                                      const uint8_t* __restrict__ segB,
                                                                      const int64_t* __restrict__ pair_index, double* __restrict__ params) {
    __shared__ uint8_t ones[kPixels];                  // maskB == 1
    __shared__ double p[kNumParams];
    __shared__ unsigned long long s_valid, s_ones, s_quad[4];
    __shared__ int s_corner[3], s_done;
    const int i = blockIdx.x;
    const int64_t pair = pair_index[i];
    if (threadIdx.x == 0) {
        scalar_draws(cfg, pair, p);
        s_valid = s_ones = 0;
    }
    __syncthreads();
    if (p[kCoverBranch] != 0.0) {
        // num_valid = np.sum(maskB) (the values, as uint8), and the pixels equal to 1, which the reference counts after a cover
        unsigned long long valid = 0, one = 0;
        for (int px = threadIdx.x; px < kPixels; px += blockDim.x) {
            const size_t g = static_cast<size_t>(i) * kPixels + px;
            const uint8_t m = segB ? segB[g] : static_cast<uint8_t>(depthB[g] > 100);
            ones[px] = m == 1;
            valid += m; one += m == 1;
        }
        block_sum(valid, &s_valid);
        block_sum(one, &s_ones);
        for (int a = 0; a < kMaxCorners; ++a) {
            if (threadIdx.x == 0) {
                cover_corner(cfg, pair, a, &s_corner[0], &s_corner[1], &s_corner[2]);
                for (int q = 0; q < 4; ++q) s_quad[q] = 0;
            }
            __syncthreads();
            const int u = s_corner[0], v = s_corner[1];
            unsigned long long cnt[4] = {0, 0, 0, 0};
            for (int px = threadIdx.x; px < kPixels; px += blockDim.x)
                if (ones[px]) ++cnt[quadrant(px / kImg, px % kImg, u, v)];
            for (int q = 0; q < 4; ++q) block_sum(cnt[q], &s_quad[q]);
            __syncthreads();
            if (threadIdx.x == 0) {
                // quadrants tried cyclically from the drawn one; a cover is kept unless fewer than half of num_valid stay ones
                s_done = 0;
                for (int t = 0; t < 4 && !s_done; ++t) {
                    const int q = (s_corner[2] + t) & 3;
                    const unsigned long long remained = s_ones - s_quad[q];
                    if (!(2 * remained < s_valid)) {
                        p[kCoverU] = u; p[kCoverV] = v; p[kCoverQuadrant] = q; p[kCoverRemained] = static_cast<double>(remained);
                        s_done = 1;
                    }
                }
                p[kCoverCorners] = a + 1;
            }
            __syncthreads();
            if (s_done) break;
        }
        if (threadIdx.x == 0) p[kCoverValid] = static_cast<double>(s_valid);
        __syncthreads();
    }
    if (threadIdx.x < kNumParams) params[static_cast<size_t>(i) * kNumParams + threadIdx.x] = p[threadIdx.x];
}

// A band of kBand rows per CTA, with the blur's 3-row halo on each side (reflected at the image's edges, as cv2's border).
constexpr int kBand = 11, kBands = kImg / kBand, kHalo = 3, kRows = kBand + 2 * kHalo, kPixThreads = 256;
static_assert(kBand * kBands == kImg, "the bands tile the image");

__global__ void __launch_bounds__(kPixThreads) augment_pixels_kernel(Config cfg, const uint8_t* __restrict__ rgbB,
                                                                      const uint16_t* __restrict__ depthB,
                                                                      const int64_t* __restrict__ pair_index,
                                                                      const double* __restrict__ params, uint8_t* __restrict__ out_rgb,
                                                                      uint16_t* __restrict__ out_depth) {
    __shared__ uint8_t s_rgb[kRows][kImg * 3];      // after HSVJitter, ChangeBright and GaussianNoise
    __shared__ uint16_t s_dep[kRows][kImg];
    __shared__ uint16_t h_rgb[kRows][kImg * 3];     // the blur's row pass: 8 fractional bits
    __shared__ uint32_t h_dep[kRows][kImg];         // 16 fractional bits
    __shared__ double p[kNumParams];
    const int i = blockIdx.y, r0 = blockIdx.x * kBand;
    if (threadIdx.x < kNumParams) p[threadIdx.x] = params[static_cast<size_t>(i) * kNumParams + threadIdx.x];
    __syncthreads();
    const int64_t pair = pair_index[i];
    const bool hsv = p[kHsvOn] != 0.0, bright = p[kBrightOn] != 0.0;
    const bool hsv_br[3] = {p[kHsvBranch] != 0.0, p[kHsvBranch + 1] != 0.0, p[kHsvBranch + 2] != 0.0};
    const double hsv_mag[3] = {p[kHsvMag], p[kHsvMag + 1], p[kHsvMag + 2]};
    const bool noise_rgb = p[kNoiseRgbBranch] != 0.0, noise_dep = p[kNoiseDepthBranch] != 0.0;
    const size_t img = static_cast<size_t>(i) * kPixels;

    for (int t = threadIdx.x; t < kRows * kImg; t += blockDim.x) {
        const int sr = t / kImg, col = t % kImg, row = reflect101(r0 - kHalo + sr, kImg);
        const int px = row * kImg + col;
        uint8_t c[3] = {rgbB[(img + px) * 3], rgbB[(img + px) * 3 + 1], rgbB[(img + px) * 3 + 2]};
        uint16_t d = depthB[img + px];
        const bool mask = d > 100;                   // depthB > 100 of the input: no stage before the noise changes depth
        if (hsv && mask) hsv_jitter(c, col, hsv_br, hsv_mag);
        if (bright)
            for (int k = 0; k < 3; ++k) c[k] = clip_u8(dmul(static_cast<double>(c[k]), p[kBright]));
        if (noise_rgb && mask)
            for (int k = 0; k < 3; ++k)
                c[k] = store_u8(dadd(static_cast<double>(c[k]), gaussian(cfg, pair, kNoiseRgb, px * 3 + k, p[kNoiseRgbStd])));
        if (noise_dep && mask) d = store_u16(dadd(static_cast<double>(d), gaussian(cfg, pair, kNoiseDepth, px, p[kNoiseDepthStd])));
        for (int k = 0; k < 3; ++k) s_rgb[sr][col * 3 + k] = c[k];
        s_dep[sr][col] = d;
    }
    __syncthreads();
    const bool blur_rgb = p[kBlurRgbBranch] != 0.0, blur_dep = p[kBlurDepthBranch] != 0.0;
    const int krgb = static_cast<int>(p[kBlurRgbK]), kdep = static_cast<int>(p[kBlurDepthK]);
    if (blur_rgb || blur_dep) {
        for (int t = threadIdx.x; t < kRows * kImg; t += blockDim.x) {
            const int sr = t / kImg, col = t % kImg;
            if (blur_rgb) {
                uint32_t acc[3] = {0, 0, 0};
                for (int j = 0; j < krgb; ++j) {
                    const int x = reflect101(col + j - krgb / 2, kImg);
                    const uint32_t w = blur_tap8(krgb, j);
                    for (int k = 0; k < 3; ++k) acc[k] += w * s_rgb[sr][x * 3 + k];
                }
                for (int k = 0; k < 3; ++k) h_rgb[sr][col * 3 + k] = static_cast<uint16_t>(acc[k]);
            }
            if (blur_dep) {
                uint32_t acc = 0;
                for (int j = 0; j < kdep; ++j) acc += blur_tap16(kdep, j) * s_dep[sr][reflect101(col + j - kdep / 2, kImg)];
                h_dep[sr][col] = acc;
            }
        }
        __syncthreads();
    }
    const int q = static_cast<int>(p[kCoverQuadrant]), cu = static_cast<int>(p[kCoverU]), cv = static_cast<int>(p[kCoverV]);
    for (int t = threadIdx.x; t < kBand * kImg; t += blockDim.x) {
        const int sr = kHalo + t / kImg, col = t % kImg, row = r0 + t / kImg;
        uint8_t c[3] = {s_rgb[sr][col * 3], s_rgb[sr][col * 3 + 1], s_rgb[sr][col * 3 + 2]};
        uint16_t d = s_dep[sr][col];
        // the column pass reads the band's own rows plus the halo: row r0 + j - k/2 sits at shared row sr + j - k/2
        if (blur_rgb) {
            uint32_t acc[3] = {0, 0, 0};
            for (int j = 0; j < krgb; ++j) {
                const uint32_t w = blur_tap8(krgb, j);
                for (int k = 0; k < 3; ++k) acc[k] += w * h_rgb[sr + j - krgb / 2][col * 3 + k];
            }
            for (int k = 0; k < 3; ++k) c[k] = blur_round8(acc[k]);
        }
        if (blur_dep) {
            uint64_t acc = 0;
            for (int j = 0; j < kdep; ++j) acc += static_cast<uint64_t>(blur_tap16(kdep, j)) * h_dep[sr + j - kdep / 2][col];
            d = blur_round16(acc);
        }
        if (q >= 0 && quadrant(row, col, cu, cv) == q) {
            c[0] = c[1] = c[2] = 0;
            d = static_cast<uint16_t>(kDepthCover);
        }
        const size_t g = img + static_cast<size_t>(row) * kImg + col;
        out_rgb[g * 3] = c[0]; out_rgb[g * 3 + 1] = c[1]; out_rgb[g * 3 + 2] = c[2];
        out_depth[g] = d;
    }
}

__global__ void augment_noise_kernel(Config cfg, const int64_t* __restrict__ pair_index, const double* __restrict__ params,
                                     double* __restrict__ noise_rgb, double* __restrict__ noise_depth) {
    const int i = blockIdx.y;
    const int64_t pair = pair_index[i];
    const double srgb = params[static_cast<size_t>(i) * kNumParams + kNoiseRgbStd];
    const double sdep = params[static_cast<size_t>(i) * kNumParams + kNoiseDepthStd];
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < kPixels * 3; e += gridDim.x * blockDim.x) {
        if (noise_rgb) noise_rgb[static_cast<size_t>(i) * kPixels * 3 + e] = gaussian(cfg, pair, kNoiseRgb, e, srgb);
        if (noise_depth && e < kPixels) noise_depth[static_cast<size_t>(i) * kPixels + e] = gaussian(cfg, pair, kNoiseDepth, e, sdep);
    }
}

}  // namespace

cudaError_t launch_augment_draws(const aug::Config& cfg, const uint16_t* depthB, const uint8_t* segB, const int64_t* pair_index, int n,
                                 double* params, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    return launch_kernel(augment_draws_kernel, dim3(n), dim3(kDrawThreads), 0, s, false, cfg, depthB, segB, pair_index, params);
}

cudaError_t launch_augment_pixels(const aug::Config& cfg, const uint8_t* rgbB, const uint16_t* depthB, const int64_t* pair_index,
                                  const double* params, int n, uint8_t* out_rgb, uint16_t* out_depth, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    return launch_kernel(augment_pixels_kernel, dim3(kBands, n), dim3(kPixThreads), 0, s, false, cfg, rgbB, depthB, pair_index, params,
                         out_rgb, out_depth);
}

cudaError_t launch_augment_noise(const aug::Config& cfg, const int64_t* pair_index, const double* params, int n, double* noise_rgb,
                                 double* noise_depth, cudaStream_t s) {
    if (n <= 0 || (!noise_rgb && !noise_depth)) return cudaSuccess;
    return launch_kernel(augment_noise_kernel, dim3(64, n), dim3(256), 0, s, false, cfg, pair_index, params, noise_rgb, noise_depth);
}

}  // namespace se3tn
