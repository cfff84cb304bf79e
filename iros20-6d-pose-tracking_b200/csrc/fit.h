// Depth agreement of each track's model at its new pose with the observed frame (see fit.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
constexpr int kFitCols = 6;              // model, observed, inlier, front, behind, residual (include/se3tn.h, se3tn_track_opts)
struct FitArgs {
    const double* poses;                 // [n][16] the step's poses_out
    const double* object_width;          // [n] mm
    double fx, fy, cx, cy;
    const uint16_t* frame_depth;         // H x W mm: the frame K0 crops B from (the filled one when the step fills)
    int H, W;
    const uint16_t* rendered;            // [n][176][176] mm: the models drawn at `poses`, 0 = background
    int tau;                             // mm, 1..1000
    int32_t* rows;                       // [n][kFitCols]
};
// One 4-CTA cluster per track; launched with programmatic dependent launch behind the render that draws `rendered`.
cudaError_t launch_fit(const FitArgs& a, int n, cudaStream_t s);
}  // namespace se3tn
