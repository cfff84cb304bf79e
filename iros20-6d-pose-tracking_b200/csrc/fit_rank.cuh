// The one order of fit-check rows (fit.h): the hypothesis choice (hypotheses.cu) keeps the start that ranks highest by it, and
// re-initialisation (reinit.cu) replaces a lost track's pose only by a start that ranks strictly above it (include/se3tn.h).
#pragma once
#include <cstdint>

namespace se3tn {
// true when fit row x ranks strictly above row y: the higher inlier fraction inlier / model (int64 cross products; model = 0
// ranks last), then the lower mean inlier residual residual / inlier (inlier = 0 ranks last).  Equal rows: false.
__device__ __forceinline__ bool fit_better(const int32_t* x, const int32_t* y) {
    const long long xm = x[0], ym = y[0], xi = x[2], yi = y[2], xr = x[5], yr = y[5];
    if ((xm == 0) != (ym == 0)) return ym == 0;
    if (xm != 0 && xi * ym != yi * xm) return xi * ym > yi * xm;
    if ((xi == 0) != (yi == 0)) return yi == 0;
    if (xi != 0 && xr * yi != yr * xi) return xr * yi < yr * xi;
    return false;
}
}  // namespace se3tn
