// The counter-based generator every random draw of the library comes from: Philox4x32-10 (Salmon et al., SC'11), the 53-bit
// uniform numpy forms from two words, and a Box-Muller normal.  A draw depends on (key, counter) alone, so any thread can form
// any draw without state, and a captured step replayed with new counters in device memory draws anew.  __host__ __device__
// except the normal: host builds (tests/test_augment_cpu.py, oracle/*_ref.py's restatements) reproduce the words bit for bit.
#pragma once
#include <cstdint>
#ifndef __CUDACC__
#define PHILOX_HD inline
#else
#define PHILOX_HD __host__ __device__ __forceinline__
#endif

namespace se3tn {
namespace rng {

struct U4 { uint32_t x, y, z, w; };
PHILOX_HD uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
    const uint64_t p = static_cast<uint64_t>(a) * b;
    *hi = static_cast<uint32_t>(p >> 32);
    return static_cast<uint32_t>(p);
}
PHILOX_HD U4 philox(U4 c, uint32_t k0, uint32_t k1) {
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0, hi1;
        const uint32_t lo0 = mulhilo(0xD2511F53u, c.x, &hi0), lo1 = mulhilo(0xCD9E8D57u, c.z, &hi1);
        c = {hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}
// a uniform double in [0, 1) with 53 random bits, as numpy forms one from two 32-bit words
PHILOX_HD double u53(uint32_t a, uint32_t b) { return ((a >> 5) * 67108864.0 + (b >> 6)) * (1.0 / 9007199254740992.0); }

#ifdef __CUDACC__
// The two standard normals of one block of words by Box-Muller: u1 = 1 - u53(x, y) in (0, 1], u2 = u53(z, w),
// sqrt(-2 ln u1) times cos(2 pi u2) (second = false) or sin(2 pi u2) (second = true).  Device only: log, sqrt and sincospi are
// CUDA's, within a few ulps of libm's but not always equal to them.
__device__ __forceinline__ double box_muller(const U4& w, bool second) {
    const double u1 = 1.0 - u53(w.x, w.y);
    const double u2 = u53(w.z, w.w);
    double s, co;
    sincospi(2.0 * u2, &s, &co);
    const double r = sqrt(__dmul_rn(-2.0, log(u1)));
    return __dmul_rn(r, second ? s : co);
}
#endif

}  // namespace rng
}  // namespace se3tn
