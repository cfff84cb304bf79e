// Storage formats of the tensor-core precisions (SE3TN_PREC_* of include/se3tn.h): how an activation or weight value of
// each mode is laid out in bytes.  Every kernel that reads or writes these formats goes through this header.
//
//   SE3TN_PREC_TF32   : 4 bytes per channel, fp32 words rounded to tf32 (rna).
//   SE3TN_PREC_BF16X3 : 4 bytes per channel, x = hi + lo as two bf16; per 32-channel (128-byte) chunk [32 x hi | 32 x lo],
//                       so channel c's lo half sits 64 bytes behind its hi half.
//   SE3TN_PREC_BF16   : 2 bytes per channel, plain bf16, 64 channels per 128-byte chunk.
//   SE3TN_PREC_FP8    : 1 byte per channel, e4m3 (cvt.rn.satfinite: |x| > 448 saturates), 128 channels per 128-byte chunk.
//                       Only the trunk's tensors (and CAT) are in this format; the mode's other layers store bf16
//                       (resident_prec).  A code means code * s with a power-of-two scale s per tensor (activations) or
//                       per row (weights); encode / decode here work on the unscaled codes, their callers scale.
//   SE3TN_PREC_FP16   : 2 bytes per channel, IEEE fp16 (cvt.rn.satfinite: |x| > 65504 saturates to +-65504), laid out as
//                       SE3TN_PREC_BF16.  Decoding is exact.
// Weight matrices use the same formats with a K-major row as the "pixel" and K as the channel.
//
// The helpers below are conversions, adds and address arithmetic only (no multiply-add), so they compile to the same
// instructions in files built with and without -fmad=false.  They never load: a call site loads the raw words with the
// cache policy it needs and hands them to decode().
#pragma once
#include "se3tn.h"
#include "ptx.cuh"
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace se3tn {

// The 2-byte formats (bf16, fp16): 64 channels per 128-byte chunk, one k16 MMA per 32-byte K step
__host__ __device__ constexpr bool prec_2byte(int prec) { return prec == SE3TN_PREC_BF16 || prec == SE3TN_PREC_FP16; }
__host__ __device__ constexpr int prec_bytes_per_channel(int prec) { return prec == SE3TN_PREC_FP8 ? 1 : (prec_2byte(prec) ? 2 : 4); }

// The stem INPUT (4 channels, 16 bytes per pixel in every mode) has a format of its own: tf32 words in SE3TN_PREC_TF32, and in
// the bf16, fp16 and fp8 modes the bf16x3 split of the 4 channels as [2 words hi | 2 words lo] (no 64-byte gap), raw fp32 in
// SE3TN_PREC_FP32.  So the stems of those modes run the bf16x3 arithmetic: stacked hi / lo weight rows (conv_wgmma.cu RCfg::kStack).
__host__ __device__ constexpr int stem_input_prec(int prec) {
    return (prec_2byte(prec) || prec == SE3TN_PREC_FP8) ? SE3TN_PREC_BF16X3 : prec;
}
// The format and arithmetic of the stems and 64-channel layers (conv_resident_kernel) in mode prec: SE3TN_PREC_FP8 runs them
// as SE3TN_PREC_BF16 (a 64-channel e4m3 pixel is half a SWIZZLE_128B row).
__host__ __device__ constexpr int resident_prec(int prec) { return prec == SE3TN_PREC_FP8 ? SE3TN_PREC_BF16 : prec; }
// Format of the input of layer li (0..13; 8 on: the trunk) in mode prec (the stems: stem_input_prec)
__host__ __device__ constexpr int layer_input_prec(int li, int prec) {
    return li < 2 ? stem_input_prec(prec) : (li < 8 ? resident_prec(prec) : prec);
}

// e4m3: element 0 in the low byte.  Saturating (satfinite: +-inf -> +-448), NaN stays NaN.
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    uint16_t lo, hi;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));   // first source -> upper byte
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
    return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}
__device__ __forceinline__ float2 unpack_e4m3x2(uint16_t v) {   // exact: every e4m3 value is an f16 value
    uint32_t h;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(v));
    return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

// The one hi / lo split: fp32 -> (bf16 hi, bf16 lo) with x ~= hi + lo, two values per 32-bit word (element 0 in the low half)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
// fp16: element 0 in the low half.  Saturating (satfinite: +-inf -> +-65504), NaN stays NaN.
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
    uint32_t h;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));   // first source -> upper half
    return h;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t w) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
}
__device__ __forceinline__ float2 unpack2(uint32_t w) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}

// N consecutive channels (N = 4 or 8) of format PREC as the raw words they occupy: kPieces vector pieces of kPieceWords
// words, piece q at byte offset q * kStride from Storage<PREC>::addr() (BF16X3: hi piece, lo piece).
template <int PREC, int N> struct Raw {
    static constexpr bool kHiLo = PREC == SE3TN_PREC_BF16X3;
    static constexpr int kWords = N * prec_bytes_per_channel(PREC) / 4;
    static constexpr int kPieces = kHiLo ? 2 : (kWords > 4 ? kWords / 4 : 1);
    static constexpr int kPieceWords = kWords / kPieces;
    static constexpr int kStride = kHiLo ? 64 : 16;
    using Piece = std::conditional_t<kPieceWords == 4, uint4, std::conditional_t<kPieceWords == 2, uint2, uint32_t>>;
    uint32_t w[kWords];
    __device__ __forceinline__ static const Piece* at(const uint8_t* p, int q) { return reinterpret_cast<const Piece*>(p + q * kStride); }
    __device__ __forceinline__ Piece get(int q) const { Piece v; memcpy(&v, w + q * kPieceWords, sizeof v); return v; }
    __device__ __forceinline__ void set(int q, Piece v) { memcpy(w + q * kPieceWords, &v, sizeof v); }
    __device__ __forceinline__ void store(uint8_t* p) const {
#pragma unroll
        for (int q = 0; q < kPieces; ++q) *reinterpret_cast<Piece*>(p + q * kStride) = get(q);
    }
};

template <int PREC> struct Storage {
    static_assert(PREC == SE3TN_PREC_TF32 || PREC == SE3TN_PREC_BF16X3 || PREC == SE3TN_PREC_BF16 || PREC == SE3TN_PREC_FP8 ||
                  PREC == SE3TN_PREC_FP16, "tensor-core precision");
    static constexpr int kBytes = prec_bytes_per_channel(PREC);     // per channel
    static constexpr bool kHiLo = PREC == SE3TN_PREC_BF16X3;

    // Byte address of channel c (c % 4 == 0 for a group of 4 or 8) of pixel `pix` in an NHWC buffer of C channels per pixel.
    // In BF16X3 this is the hi half; the lo half is 64 bytes further.
    __host__ __device__ __forceinline__ static size_t addr(size_t pix, int C, int c) {
        if (kHiLo) return (pix * C + (c & ~31)) * 4 + (c & 31) * 2;
        return (pix * C + c) * kBytes;
    }

    template <int N> __device__ __forceinline__ static Raw<PREC, N> encode(const float (&v)[N]) {
        Raw<PREC, N> r;
        if constexpr (PREC == SE3TN_PREC_TF32) {
#pragma unroll
            for (int i = 0; i < N; ++i) r.w[i] = __float_as_uint(ptx::to_tf32(v[i]));
        } else if constexpr (kHiLo) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) split2(v[2 * i], v[2 * i + 1], r.w[i], r.w[N / 2 + i]);
        } else if constexpr (PREC == SE3TN_PREC_FP8) {
#pragma unroll
            for (int i = 0; i < N / 4; ++i) r.w[i] = pack_e4m3x4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
        } else if constexpr (PREC == SE3TN_PREC_FP16) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) r.w[i] = pack_f16(v[2 * i], v[2 * i + 1]);
        } else {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) r.w[i] = pack_bf16(v[2 * i], v[2 * i + 1]);
        }
        return r;
    }

    template <int N> __device__ __forceinline__ static void decode(const Raw<PREC, N>& r, float (&v)[N]) {
        if constexpr (PREC == SE3TN_PREC_TF32) {
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = __uint_as_float(r.w[i]);
        } else if constexpr (PREC == SE3TN_PREC_FP8) {
#pragma unroll
            for (int i = 0; i < N / 4; ++i) {
                const float2 a = unpack_e4m3x2(static_cast<uint16_t>(r.w[i] & 0xFFFFu)), b = unpack_e4m3x2(static_cast<uint16_t>(r.w[i] >> 16));
                v[4 * i] = a.x; v[4 * i + 1] = a.y; v[4 * i + 2] = b.x; v[4 * i + 3] = b.y;
            }
        } else if constexpr (PREC == SE3TN_PREC_FP16) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {
                const float2 h = unpack_f16x2(r.w[i]);
                v[2 * i] = h.x; v[2 * i + 1] = h.y;
            }
        } else {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {
                const float2 h = unpack2(r.w[i]);
                if constexpr (kHiLo) {
                    const float2 l = unpack2(r.w[N / 2 + i]);
                    v[2 * i] = h.x + l.x; v[2 * i + 1] = h.y + l.y;
                } else {
                    v[2 * i] = h.x; v[2 * i + 1] = h.y;
                }
            }
        }
    }
};

// One stem-input pixel (stem_input_prec above), as the 16 bytes stored
__device__ __forceinline__ float4 encode_stem_pixel(float4 v, int prec) {
    const float f[4] = {v.x, v.y, v.z, v.w};
    uint4 w;
    switch (stem_input_prec(prec)) {
        case SE3TN_PREC_TF32: w = Storage<SE3TN_PREC_TF32>::encode(f).get(0); break;
        case SE3TN_PREC_BF16X3: { const auto r = Storage<SE3TN_PREC_BF16X3>::encode(f); w = make_uint4(r.w[0], r.w[1], r.w[2], r.w[3]); break; }
        default: return v;
    }
    return make_float4(__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), __uint_as_float(w.w));
}

}  // namespace se3tn
