// Depth refinement of a render step (se3tn_track_opts.icp): projective point-to-plane ICP of every track's model against the
// observed depth, one Gauss-Newton iteration per accumulate + solve pair (see icp.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "render.h"
namespace se3tn {
constexpr int kIcpSums = 32;             // per track: JtJ upper triangle (21), Jte (6), sum e^2, inlier count, 3 unused
constexpr int kIcpCols = 4;              // stats row: inliers, rms_mm, step_mm, step_deg (include/se3tn.h, se3tn_icp_opts)

struct IcpArgs {
    double* poses;                       // [n][16] the step's poses_out: read by the accumulation, updated in place by the solve
    const double* object_width;          // [n] mm
    const int32_t* mesh_ids;             // [n] or null (mesh 0), as the render draws them
    const MeshDev* meshes;               // device table indexed by mesh id
    int n_meshes;
    double fx, fy, cx, cy;
    const uint16_t* frame_depth;         // H x W mm: the frame K0 crops B from (the filled one when the step fills)
    int H, W;
    const int32_t* tri;                  // [n][176][176] the triangle each crop pixel of the render at `poses` shows, -1 = none
    int tau;                             // mm, 1..1000: the association gate
    int min_inliers;                     // fewer inliers leave the pose as it is
    double* sums;                        // [n][kIcpSums] scratch between the two kernels
    double* stats;                       // [n][kIcpCols] or null
};
// accumulate: one 4-CTA cluster per track, launched with programmatic dependent launch behind the render that wrote `tri`.
// solve: one thread per track, launched with programmatic dependent launch behind the accumulation.
cudaError_t launch_icp(const IcpArgs& a, int n, cudaStream_t s);
}  // namespace se3tn
