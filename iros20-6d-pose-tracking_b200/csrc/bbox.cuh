// Crop / render window of a track: reference Utils.py:302-316 (compute_bbox) + the min/max of Utils.py:321-324 /
// predict.py:204-207.  float64 with the reference's association, np.round = rint (half to even).
#pragma once
#include <cuda_runtime.h>
namespace se3tn {
__device__ __forceinline__ void bbox_window(const double* pose, double fx, double fy, double cx, double cy,
                                            double width, double sx, double sy, double sz,
                                            int& top, int& left, int& ch, int& cw)
{
    const double ox = __dmul_rn(pose[3], sx), oy = __dmul_rn(pose[7], sy), oz = __dmul_rn(pose[11], sz);
    const double half = width / 2;
    // u for x-half / x+half, v for y-half / y+half (the 4 corners share these two values each)
    const double u0 = rint(__dadd_rn(__ddiv_rn(__dmul_rn(ox - half, fx), oz), cx));
    const double u1 = rint(__dadd_rn(__ddiv_rn(__dmul_rn(ox + half, fx), oz), cx));
    const double v0 = rint(__dadd_rn(__ddiv_rn(__dmul_rn(oy - half, fy), oz), cy));
    const double v1 = rint(__dadd_rn(__ddiv_rn(__dmul_rn(oy + half, fy), oz), cy));
    const double umin = fmin(u0, u1), umax = fmax(u0, u1), vmin = fmin(v0, v1), vmax = fmax(v0, v1);
    // clamp to int range so degenerate poses (z ~ 0) cannot overflow
    const double lim = 1.0e9;
    if (!(umin == umin && umax == umax && vmin == vmin && vmax == vmax)) { top = left = 0; ch = cw = 0; return; }
    left = static_cast<int>(fmax(-lim, fmin(lim, umin)));
    top = static_cast<int>(fmax(-lim, fmin(lim, vmin)));
    cw = static_cast<int>(fmax(-lim, fmin(lim, umax))) - left;
    ch = static_cast<int>(fmax(-lim, fmin(lim, vmax))) - top;
}

// The source row / column cv2 INTER_NEAREST reads for output pixel dst when `size` source pixels are resized to `out`:
// floor(dst * (1 / (out / size))) in float64, clamped to size - 1 -- as the crop kernels cut B (no meaning for size <= 0).
__device__ __forceinline__ int nearest_source(int dst, int out, int size)
{
    const double inv = size > 0 ? 1.0 / (static_cast<double>(out) / size) : 0.0;
    const int s = static_cast<int>(floor(dst * inv));
    return s > size - 1 ? size - 1 : s;
}

}  // namespace se3tn
