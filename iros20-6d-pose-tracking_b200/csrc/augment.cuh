// The reference's train-time augmentations of input B (data_augmentation.py:48-121, 217-267) as per-pixel functions and per-pair
// draws.  Everything here except the Gaussian draws is __host__ __device__: the host build (tests/test_augment_cpu.py compiles
// this header with g++ -ffp-contract=off) and the device build compute the same bits, because every float / double operation
// whose rounding matters is spelt with an explicit round-to-nearest intrinsic on the device (nvcc would contract a * b + c).
#pragma once
#include <cstdint>
#include "philox.cuh"
#ifndef __CUDACC__
#include <cmath>
#define AUG_HD inline
#else
#define AUG_HD __host__ __device__ __forceinline__
#endif

namespace se3tn {
namespace aug {

constexpr int kImg = 176;
constexpr int kPixels = kImg * kImg;
constexpr int kMaxCorners = 64;        // BlackCover: corners drawn at most (each tries four quadrants); the reference loops forever
constexpr int kDepthCover = 55537;     // -9999 stored into uint16 (numpy 1.x): what BlackCover leaves in depthB

// One pair's draws, as se3tn_augment_draws returns them (doubles, include/se3tn.h SE3TN_AUG_*).
enum Param {
    kHsvOn = 0, kHsvBranch = 1, kHsvMag = 4, kBrightOn = 7, kBright = 8, kNoiseRgbBranch = 9, kNoiseRgbStd = 10,
    kNoiseDepthBranch = 11, kNoiseDepthStd = 12, kBlurRgbBranch = 13, kBlurRgbK = 14, kBlurDepthBranch = 15, kBlurDepthK = 16,
    kCoverBranch = 17, kCoverU = 18, kCoverV = 19, kCoverQuadrant = 20, kCoverCorners = 21, kCoverValid = 22, kCoverRemained = 23,
    kNumParams = 24
};

// The configuration as the kernels take it (se3tn_augment without the refused DepthMissing).
struct Config {
    uint64_t seed;
    int hsv, bright, noise, blur, cover;   // stage enables
    int blur_half_max;                     // randint(1, max_kernel_size // 2 + 1): 1..3
    double hsv_prob, hsv_noise[3], bright_lo, bright_hi, noise_prob, noise_rgb, noise_depth, blur_prob, cover_prob;
};

// ---------------------------------------------------------------------------------------------------- exact arithmetic
#ifdef __CUDA_ARCH__
AUG_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
AUG_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
AUG_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
AUG_HD float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
AUG_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
AUG_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
AUG_HD int round_even(float x) { return __float2int_rn(x); }
AUG_HD int round_even(double x) { return __double2int_rn(x); }
AUG_HD long long trunc_ll(double x) { return __double2ll_rz(x); }
#else
AUG_HD float fadd(float a, float b) { return a + b; }
AUG_HD float fsub(float a, float b) { return a - b; }
AUG_HD float fmul(float a, float b) { return a * b; }
AUG_HD float ffma(float a, float b, float c) { return std::fma(a, b, c); }
AUG_HD double dadd(double a, double b) { return a + b; }
AUG_HD double dmul(double a, double b) { return a * b; }
AUG_HD int round_even(float x) { return static_cast<int>(std::nearbyint(x)); }
AUG_HD int round_even(double x) { return static_cast<int>(std::nearbyint(x)); }
AUG_HD long long trunc_ll(double x) { return static_cast<long long>(x); }
#endif

// numpy's store of a float64 into a uint8 / uint16 array on x86-64: truncate toward zero, keep the low bits (256.4 -> 0,
// -1.5 -> 255).  Pinned against numpy by tests/test_augment_cpu.py for values within +-2^31.
AUG_HD uint8_t store_u8(double x) { return static_cast<uint8_t>(static_cast<uint64_t>(trunc_ll(x))); }
AUG_HD uint16_t store_u16(double x) { return static_cast<uint16_t>(static_cast<uint64_t>(trunc_ll(x))); }

// np.clip(x, 0, 255).astype(np.uint8) of a float64
AUG_HD uint8_t clip_u8(double x) { return static_cast<uint8_t>(x < 0.0 ? 0.0 : (x > 255.0 ? 255.0 : x)); }

// ---------------------------------------------------------------------------------------------------- cv2 8-bit HSV
// cv2.cvtColor(rgb, COLOR_RGB2HSV) on uint8: H in [0, 180), integer tables with 12 fractional bits (cv2 RGB2HSV_b).
AUG_HD void rgb2hsv(uint8_t r, uint8_t g, uint8_t b, uint8_t* hsv) {
    const int v = r > g ? (r > b ? r : b) : (g > b ? g : b);
    const int vmin = r < g ? (r < b ? r : b) : (g < b ? g : b);
    const int diff = v - vmin;
    const int sdiv = v ? round_even(static_cast<double>(255 << 12) / v) : 0;
    const int hdiv = diff ? round_even(static_cast<double>(180 << 12) / (6.0 * diff)) : 0;
    const int s = (diff * sdiv + (1 << 11)) >> 12;
    int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
    h = (h * hdiv + (1 << 11)) >> 12;
    h += h < 0 ? 180 : 0;
    hsv[0] = static_cast<uint8_t>(h > 255 ? 255 : h);
    hsv[1] = static_cast<uint8_t>(s);
    hsv[2] = static_cast<uint8_t>(v);
}

// cv2.cvtColor(hsv, COLOR_HSV2RGB) on uint8, every stored H (0-255) included, as OpenCV 4.13 computes it on x86-64 with AVX2:
// float math with h * (6/180), the sector taken modulo 6, 1 - s h and 1 - s (1 - h) each one fused multiply-add, and the result
// times 255 converted to uint8.  cv2 converts each row in blocks of 32 pixels, which truncate, and converts the last
// (width % 32) pixels one at a time, rounding half to even: `col` is the pixel's column in a row of kImg pixels.
constexpr int kHsvVectorCols = kImg / 32 * 32;
AUG_HD void hsv2rgb(uint8_t H, uint8_t S, uint8_t V, uint8_t* rgb, int col) {
    const float hscale = 6.0f / 180.0f;
    float h = fmul(static_cast<float>(H), hscale);
    const float s = fmul(static_cast<float>(S), 1.0f / 255.0f), v = fmul(static_cast<float>(V), 1.0f / 255.0f);
    const int pre = static_cast<int>(h);             // h >= 0: truncation is the floor
    h = fsub(h, static_cast<float>(pre));
    const int sector = pre % 6;
    float tab[4];
    tab[0] = v;
    tab[1] = fmul(v, fsub(1.0f, s));
    tab[2] = fmul(v, ffma(-s, h, 1.0f));
    tab[3] = fmul(v, ffma(-s, fsub(1.0f, h), 1.0f));
    // (b, g, r) = tab[sector_data[sector]], cv2's table {{1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}}; nibble s of each
    // constant is the entry of sector s
    const int bi = (0x200311 >> (4 * sector)) & 0xF;
    const int gi = (0x112003 >> (4 * sector)) & 0xF;
    const int ri = (0x031120 >> (4 * sector)) & 0xF;
    const int idx[3] = {ri, gi, bi};
    for (int c = 0; c < 3; ++c) {
        const float x = fmul(tab[idx[c]], 255.0f);
        rgb[c] = static_cast<uint8_t>(col < kHsvVectorCols ? static_cast<int>(x) : round_even(x));
    }
}

// HSVJitter's per-pixel arithmetic at a mask pixel: the float32 channel plus float32(delta) when its branch is taken, clipped to
// [0, 255], truncated to uint8, converted back.
AUG_HD void hsv_jitter(uint8_t* rgb, int col, const bool branch[3], const double mag[3]) {
    uint8_t hsv[3];
    rgb2hsv(rgb[0], rgb[1], rgb[2], hsv);
    for (int c = 0; c < 3; ++c) {
        float x = static_cast<float>(hsv[c]);
        if (branch[c]) x = fadd(x, static_cast<float>(mag[c]));
        x = x < 0.0f ? 0.0f : (x > 255.0f ? 255.0f : x);
        hsv[c] = static_cast<uint8_t>(x);
    }
    hsv2rgb(hsv[0], hsv[1], hsv[2], rgb, col);
}

// ---------------------------------------------------------------------------------------------------- cv2 GaussianBlur
// cv2.GaussianBlur(img, (k, k), sigmaX=2) for k = 3, 5, 7 is separable fixed point: 8-bit images with kernels of 8 fractional
// bits (16 for the 16-bit path), the row pass exact in integers, the column pass rounded half up at the end.  The taps below
// are cv2's (Gaussian of sigma 2 normalised, then error-diffused to the fixed-point grid); tests/test_augment_cpu.py checks
// the host build against cv2 bit for bit.
AUG_HD int blur_tap8(int k, int t) {    // t in [0, k)
    const int c = t < k / 2 ? t : k - 1 - t;
    return k == 3 ? (c == 0 ? 82 : 92) : k == 5 ? (c == 0 ? 39 : c == 1 ? 57 : 64) : (c == 0 ? 18 : c == 1 ? 34 : c == 2 ? 48 : 56);
}
AUG_HD uint32_t blur_tap16(int k, int t) {
    const int c = t < k / 2 ? t : k - 1 - t;
    return k == 3 ? (c == 0 ? 20917u : 23702u)
         : k == 5 ? (c == 0 ? 9992u : c == 1 ? 14539u : 16474u)
                  : (c == 0 ? 4598u : c == 1 ? 8590u : c == 2 ? 12499u : 14162u);
}
// cv2's default border, BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba), for offsets of at most n - 1
AUG_HD int reflect101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }
AUG_HD uint8_t blur_round8(uint32_t acc) { return static_cast<uint8_t>((acc + (1u << 15)) >> 16); }
AUG_HD uint16_t blur_round16(uint64_t acc) { return static_cast<uint16_t>((acc + (1ull << 31)) >> 32); }

// ---------------------------------------------------------------------------------------------------- draws
// Philox4x32-10 (philox.cuh): counter (pair index low, high, stream, slot), key = the seed's two words.
using rng::U4;
using rng::philox;
using rng::u53;

enum Stream : uint32_t { kScalars = 0, kNoiseRgb = 1, kNoiseDepth = 2 };
AUG_HD U4 draw_words(const Config& c, int64_t pair, uint32_t stream, uint32_t slot) {
    const uint64_t p = static_cast<uint64_t>(pair);
    return philox({static_cast<uint32_t>(p), static_cast<uint32_t>(p >> 32), stream, slot}, static_cast<uint32_t>(c.seed),
                  static_cast<uint32_t>(c.seed >> 32));
}
AUG_HD double uniform(const Config& c, int64_t pair, uint32_t slot) {
    const U4 w = draw_words(c, pair, kScalars, slot);
    return u53(w.x, w.y);
}
AUG_HD double uniform(const Config& c, int64_t pair, uint32_t slot, double lo, double hi) {   // lo + (hi - lo) U, numpy's form
    return dadd(lo, dmul(hi - lo, uniform(c, pair, slot)));
}
AUG_HD int randint(const Config& c, int64_t pair, uint32_t slot, int count) {   // uniform over [0, count)
    const int v = static_cast<int>(uniform(c, pair, slot) * count);
    return v < count ? v : count - 1;
}

// Scalar slots: what each stage draws, whether or not its branch is taken.
enum Slot : uint32_t {
    kSlotHsvBranch = 0, kSlotHsvMag = 3, kSlotBright = 6, kSlotNoiseRgbBranch = 7, kSlotNoiseRgbStd = 8, kSlotNoiseDepthBranch = 9,
    kSlotNoiseDepthStd = 10, kSlotBlurRgbBranch = 11, kSlotBlurRgbK = 12, kSlotBlurDepthBranch = 13, kSlotBlurDepthK = 14,
    kSlotCoverBranch = 15, kSlotCorner = 16   // corner a: u, v, quadrant at kSlotCorner + 3a + {0, 1, 2}
};

// Every draw of one pair except the cover's accepted corner (cover_corner / the cover kernel).
AUG_HD void scalar_draws(const Config& c, int64_t pair, double* p) {
    for (int i = 0; i < kNumParams; ++i) p[i] = 0.0;
    p[kHsvOn] = c.hsv;
    for (int ch = 0; ch < 3; ++ch) {
        p[kHsvBranch + ch] = c.hsv && uniform(c, pair, kSlotHsvBranch + ch) < c.hsv_prob;
        p[kHsvMag + ch] = c.hsv ? uniform(c, pair, kSlotHsvMag + ch, -c.hsv_noise[ch], c.hsv_noise[ch]) : 0.0;
    }
    p[kBrightOn] = c.bright;
    p[kBright] = c.bright ? uniform(c, pair, kSlotBright, c.bright_lo, c.bright_hi) : 1.0;
    if (c.noise) {
        p[kNoiseRgbBranch] = uniform(c, pair, kSlotNoiseRgbBranch) < c.noise_prob;
        p[kNoiseRgbStd] = uniform(c, pair, kSlotNoiseRgbStd, 0.0, c.noise_rgb);
        p[kNoiseDepthBranch] = uniform(c, pair, kSlotNoiseDepthBranch) < c.noise_prob;
        p[kNoiseDepthStd] = uniform(c, pair, kSlotNoiseDepthStd, 0.0, c.noise_depth);
    }
    if (c.blur) {
        p[kBlurRgbBranch] = uniform(c, pair, kSlotBlurRgbBranch) < c.blur_prob;
        p[kBlurRgbK] = 2 * (1 + randint(c, pair, kSlotBlurRgbK, c.blur_half_max)) + 1;
        p[kBlurDepthBranch] = uniform(c, pair, kSlotBlurDepthBranch) < c.blur_prob;
        p[kBlurDepthK] = 2 * (1 + randint(c, pair, kSlotBlurDepthK, c.blur_half_max)) + 1;
    }
    p[kCoverBranch] = c.cover && uniform(c, pair, kSlotCoverBranch) < c.cover_prob;
    p[kCoverQuadrant] = -1.0;
}

// BlackCover's corner a: (u, v) = (randint(0, W), randint(0, H)), then the first quadrant choice([0, 1, 2, 3]).
AUG_HD void cover_corner(const Config& c, int64_t pair, int a, int* u, int* v, int* q) {
    *u = randint(c, pair, kSlotCorner + 3 * a, kImg);
    *v = randint(c, pair, kSlotCorner + 3 * a + 1, kImg);
    *q = randint(c, pair, kSlotCorner + 3 * a + 2, 4);
}
// quadrant of pixel (row, col) for the corner (u, v): 0 top left, 1 top right, 2 bottom left, 3 bottom right
AUG_HD int quadrant(int row, int col, int u, int v) { return (row >= v ? 2 : 0) + (col >= u ? 1 : 0); }

#ifdef __CUDACC__
// N(0, std) of element e of a noise field (stream kNoiseRgb: (176,176,3) in HWC order, kNoiseDepth: (176,176)).  Elements 2j and
// 2j + 1 are the two Box-Muller normals of Philox slot j.  Device only: the host never forms the noise, it is handed the fields.
__device__ __forceinline__ double gaussian(const Config& c, int64_t pair, uint32_t stream, uint32_t e, double stddev) {
    return dmul(stddev, rng::box_muller(draw_words(c, pair, stream, e >> 1), e & 1));
}
#endif

}  // namespace aug
}  // namespace se3tn
