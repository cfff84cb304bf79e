// The fit check of a track step (se3tn_track_opts): after the last round, every track's model is drawn at its new pose
// (render_kernel, depth only) and compared pixel by pixel with the observed depth in the crop window of that pose -- the
// window K0 would crop input B from in the next frame's step: bbox_window (bbox.cuh) and cv2's nearest source index
// floor(dst * (1 / (176 / size))), clamped, 0 outside the frame.  R is the rendered depth, O the raw observed uint16 mm (the
// filled frame when the step fills), both before any clipping.  Per track, over the 176 x 176 pixels with R > 0:
//   model = #R>0, observed = #(O>0), inlier = #|O-R| <= tau, front = #O < R-tau, behind = #O > R+tau, residual = sum |O-R| of
//   the inliers.
// Integer counts and sums of integers: the rows are exact and do not depend on the order of the reduction.
// One cluster of 4 CTAs per track, each CTA a quarter of the rows; CTA 0 of the cluster adds the four partial rows through
// distributed shared memory and writes the track's row, so one launch needs no zeroed output and no atomics.
#include "fit.h"
#include "aux_kernels.h"
#include "bbox.cuh"
#include "launch.h"
#include "ptx.cuh"
#include <cooperative_groups.h>

namespace se3tn {
namespace {
namespace cg = cooperative_groups;
constexpr int kFitCtas = 4, kFitThreads = 512, kFitRows = kImg / kFitCtas;
static_assert(kImg % kFitCtas == 0, "whole rows per CTA");

__global__ void __cluster_dims__(kFitCtas, 1, 1) __launch_bounds__(kFitThreads)
fit_kernel(const FitArgs a)
{
    __shared__ int s_win[4];
    __shared__ int s_sx[kImg], s_sy[kFitRows];
    __shared__ int s_warp[kFitThreads / 32][kFitCols];
    __shared__ int s_part[kFitCols];
    ptx::grid_dep_launch();
    const int n = blockIdx.y, row0 = blockIdx.x * kFitRows;
    // poses_out comes from the last round's head / pose update, `rendered` from the render launched right before this one:
    // every read of either, and of the frame, stays behind this wait
    ptx::grid_dep_wait();
    if (threadIdx.x == 0) {
        int top, left, ch, cw;
        bbox_window(a.poses + 16 * n, a.fx, a.fy, a.cx, a.cy, a.object_width[n], 1000.0, 1000.0, 1000.0, top, left, ch, cw);
        s_win[0] = top; s_win[1] = left; s_win[2] = ch; s_win[3] = cw;
    }
    __syncthreads();
    const int top = s_win[0], left = s_win[1], ch = s_win[2], cw = s_win[3];
    const bool inside = ch > 0 && cw > 0;
    // the nearest source indices exactly as preprocess_kernel computes them
    if (threadIdx.x < kImg) s_sx[threadIdx.x] = nearest_source(threadIdx.x, kImg, cw);
    else if (threadIdx.x >= 256 && threadIdx.x < 256 + kFitRows) s_sy[threadIdx.x - 256] = nearest_source(row0 + threadIdx.x - 256, kImg, ch);
    __syncthreads();
    const uint16_t* R = a.rendered + (static_cast<size_t>(n) * kImg + row0) * kImg;
    int model = 0, observed = 0, inlier = 0, front = 0, behind = 0, residual = 0;
    for (int p = threadIdx.x; p < kFitRows * kImg; p += kFitThreads) {
        const int r = R[p];
        if (r == 0) continue;
        ++model;
        if (!inside) continue;
        const int ly = p / kImg, x = p - ly * kImg;
        const int fy = top + s_sy[ly], fx = left + s_sx[x];
        if (fy < 0 || fy >= a.H || fx < 0 || fx >= a.W) continue;
        const int o = a.frame_depth[static_cast<size_t>(fy) * a.W + fx];
        if (o == 0) continue;
        ++observed;
        const int d = o - r;
        if (d < -a.tau) ++front;
        else if (d > a.tau) ++behind;
        else { ++inlier; residual += d < 0 ? -d : d; }
    }
    const int v[kFitCols] = {model, observed, inlier, front, behind, residual};
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < kFitCols; ++k) {
        const int s = static_cast<int>(__reduce_add_sync(0xffffffffu, static_cast<unsigned>(v[k])));
        if (lane == 0) s_warp[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < kFitCols) {
        int s = 0;
        for (int w = 0; w < kFitThreads / 32; ++w) s += s_warp[w][threadIdx.x];
        s_part[threadIdx.x] = s;
    }
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();                                          // every CTA's partial row is written
    if (cluster.block_rank() == 0 && threadIdx.x < kFitCols) {
        int s = 0;
        for (int r = 0; r < kFitCtas; ++r) s += cluster.map_shared_rank(s_part, r)[threadIdx.x];
        a.rows[n * kFitCols + threadIdx.x] = s;
    }
    cluster.sync();                                          // no CTA exits while CTA 0 still reads its shared memory
}
}  // namespace

cudaError_t launch_fit(const FitArgs& a, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (!a.poses || !a.object_width || !a.frame_depth || !a.rendered || !a.rows || a.tau < 1 || a.tau > 1000) return cudaErrorInvalidValue;
    return launch_kernel(fit_kernel, dim3(kFitCtas, n), dim3(kFitThreads), 0, s, true, a);
}

}  // namespace se3tn
