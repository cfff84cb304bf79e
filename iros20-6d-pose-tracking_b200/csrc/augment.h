// Launch wrappers of the augmentation kernels (augment.cu); the per-pixel arithmetic and the draws are in augment.cuh.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "augment.cuh"

namespace se3tn {

// Every draw of pairs pair_index[0..n) (aug::Param layout, n x aug::kNumParams doubles), BlackCover's accepted corner included:
// maskB is segB (uint8 (n,176,176)) or, when segB is NULL, depthB (uint16 (n,176,176)) > 100.  One CTA per pair.
cudaError_t launch_augment_draws(const aug::Config& cfg, const uint16_t* depthB, const uint8_t* segB, const int64_t* pair_index, int n,
                                 double* params, cudaStream_t s);
// The five stages on rgbB / depthB with the draws of launch_augment_draws -> out_rgb (n,176,176,3), out_depth (n,176,176).
cudaError_t launch_augment_pixels(const aug::Config& cfg, const uint8_t* rgbB, const uint16_t* depthB, const int64_t* pair_index,
                                  const double* params, int n, uint8_t* out_rgb, uint16_t* out_depth, cudaStream_t s);
// GaussianNoise's N(0, std) fields (every element, whatever the branch and mask): rgb (n,176,176,3), depth (n,176,176); nullable.
cudaError_t launch_augment_noise(const aug::Config& cfg, const int64_t* pair_index, const double* params, int n, double* noise_rgb,
                                 double* noise_depth, cudaStream_t s);

}  // namespace se3tn
