// Depth hole filling for live sensors (see depth_fill.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
constexpr int kFillLutEntries = (1 << 12) + 2;
struct FillScratch { float* a; float* b; float* lut; unsigned* minmax; };   // a, b: H*W floats each; lut: kFillLutEntries + 1 floats (scale at the end)
cudaError_t launch_fill_depth(const uint16_t* depth_mm, int H, int W, float max_depth, bool extrapolate, bool gaussian, const FillScratch& sc,
                              uint16_t* out_mm, float* out_m, cudaStream_t s);
// kernels launch_fill_depth launches: 8 (bilateral), 6 (gaussian), 3 more with extrapolate
inline int fill_depth_launches(bool extrapolate, bool gaussian) { return (gaussian ? 6 : 8) + (extrapolate ? 3 : 0); }
}  // namespace se3tn
