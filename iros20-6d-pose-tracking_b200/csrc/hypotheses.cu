// Multi-hypothesis tracking: start every track from S poses and keep the one whose model best fits the observed depth.
//
// hypotheses_kernel expands n tracks into n x S rows, track-major (track i's hypothesis h is row i S + h).  Hypothesis 0 is the
// track's previous pose P, copied.  Hypothesis h >= 1 is P . inv(D), D = random_gaussian_magnitude(max_t, max_r) (reference
// Utils.py:372-404), composed as produce_train_pair_data.py:110 composes a training pair's A_in_cam = B_in_cam . inv(B_in_A).
// Every uniform comes from Philox4x32-10 (philox.cuh), key = the seed, counter = (the track's draw key low, high, h, slot):
//   slot 0        the translation's direction: U_theta = u53(x, y), U_phi = u53(z, w); random_direction's theta = U_theta * pi * 2,
//                 phi = acos(2 U_phi - 1)
//   slot 1        the rotation axis, the same way
//   slot 2 + j    the j-th N(0, max_t) draw of the translation magnitude (Box-Muller's first normal of the block)
//   slot 66 + j   the j-th N(0, max_r) draw of the rotation magnitude, degrees
// A magnitude is redrawn until |m| <= max, as the reference's loop does, at most kHypMaxTries times; one that never lands inside
// (probability ~1e-32 per magnitude) is clamped to +-max with the sign of its last draw.  The rotation is cv2.Rodrigues of
// axis / |axis| * m / 180 * pi in fp64.  The row's weight id and object width are track i's.
//
// select_kernel picks, per track, the hypothesis whose fit row has the highest inlier fraction inlier / model (int64 cross
// products; model = 0 ranks last), then the lowest mean inlier residual residual / inlier (inlier = 0 ranks last), then the
// lowest h, and writes its pose, network outputs, fit row and index.  A frame without depth gives every row inlier = 0 and
// keeps hypothesis 0, unless hypothesis 0's model = 0 (nothing drawn in its window): then the first h >= 1 with model > 0 wins.
#include "hypotheses.h"
#include "fit.h"
#include "fit_rank.cuh"
#include "launch.h"
#include "philox.cuh"
#include <cfloat>
#include <math_constants.h>

namespace se3tn {
namespace {
constexpr int kHypThreads = 128;
constexpr uint32_t kSlotDirT = 0, kSlotDirR = 1, kSlotMagT = 2, kSlotMagR = 2 + kHypMaxTries;

__device__ rng::U4 words(const HypArgs& a, uint64_t key, int h, uint32_t slot) {
    return rng::philox({static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32), static_cast<uint32_t>(h), slot},
                       static_cast<uint32_t>(a.seed), static_cast<uint32_t>(a.seed >> 32));
}

// random_direction (Utils.py:393-404): sph2cart(acos(2 U1 - 1), U0 * pi * 2, 1)
__device__ void direction(double u_theta, double u_phi, double* d) {
    const double theta = (u_theta * CUDART_PI) * 2.0;
    const double phi = acos(2.0 * u_phi - 1.0);
    d[0] = sin(phi) * cos(theta);
    d[1] = sin(phi) * sin(theta);
    d[2] = cos(phi);
}

// np.random.normal(0, max) until |m| <= max; *tries: the draws taken
__device__ double magnitude(const HypArgs& a, uint64_t key, int h, uint32_t slot0, double max, int* tries) {
    double m = 0.0;
    for (int j = 0; j < kHypMaxTries; ++j) {
        m = max * rng::box_muller(words(a, key, h, slot0 + j), false);
        if (fabs(m) <= max) { *tries = j + 1; return m; }
    }
    *tries = kHypMaxTries;
    return copysign(max, m);
}

__global__ void __launch_bounds__(kHypThreads) hypotheses_kernel(const HypArgs a)
{
    const int row = blockIdx.x * kHypThreads + threadIdx.x;
    if (row >= a.n * a.S) return;
    const int i = row / a.S, h = row - i * a.S;
    if (a.wid) a.wid[row] = a.wid_in[i];
    if (a.width) a.width[row] = a.width_in[i];
    const double* P = a.poses_in + 16 * static_cast<size_t>(i);
    double* out = a.poses + 16 * static_cast<size_t>(row);
    double* dr = a.draws ? a.draws + kHypDraws * static_cast<size_t>(row) : nullptr;
    if (h == 0) {
        for (int k = 0; k < 16; ++k) out[k] = P[k];
        if (dr) for (int k = 0; k < kHypDraws; ++k) dr[k] = 0.0;
        return;
    }
    const uint64_t key = static_cast<uint64_t>(a.keys[i]);
    const rng::U4 wt = words(a, key, h, kSlotDirT), wr = words(a, key, h, kSlotDirR);
    const double u[4] = {rng::u53(wt.x, wt.y), rng::u53(wt.z, wt.w), rng::u53(wr.x, wr.y), rng::u53(wr.z, wr.w)};
    double dt[3], ax[3];
    direction(u[0], u[1], dt);
    int tries_t, tries_r;
    const double mt = magnitude(a, key, h, kSlotMagT, a.max_t, &tries_t);
    direction(u[2], u[3], ax);
    const double norm = sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
    const double mr = magnitude(a, key, h, kSlotMagR, a.max_r_deg, &tries_r);
    double T[3], rod[3];
    for (int k = 0; k < 3; ++k) {
        T[k] = dt[k] * mt;
        rod[k] = ((ax[k] / norm) * mr / 180.0) * CUDART_PI;
    }
    // cv2.Rodrigues: R = cos(t) I + (1 - cos(t)) r r^T + sin(t) [r]x, r = rod / t; the identity below DBL_EPSILON
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    const double t = sqrt(rod[0] * rod[0] + rod[1] * rod[1] + rod[2] * rod[2]);
    if (t >= DBL_EPSILON) {
        const double c = cos(t), s = sin(t), c1 = 1.0 - c, it = 1.0 / t;
        const double r[3] = {rod[0] * it, rod[1] * it, rod[2] * it};
        const double rx[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
        for (int p = 0; p < 3; ++p)
            for (int q = 0; q < 3; ++q) R[3 * p + q] = (p == q ? c : 0.0) + c1 * (r[p] * r[q]) + s * rx[3 * p + q];
    }
    // inv(D) = [R^T, -R^T T; 0 0 0 1], then P . inv(D)
    double Di[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1};
    for (int p = 0; p < 3; ++p) {
        for (int q = 0; q < 3; ++q) Di[4 * p + q] = R[3 * q + p];
        Di[4 * p + 3] = -(R[p] * T[0] + R[3 + p] * T[1] + R[6 + p] * T[2]);
    }
    for (int p = 0; p < 4; ++p)
        for (int q = 0; q < 4; ++q)
            out[4 * p + q] = P[4 * p] * Di[q] + P[4 * p + 1] * Di[4 + q] + P[4 * p + 2] * Di[8 + q] + P[4 * p + 3] * Di[12 + q];
    if (dr) {
        for (int k = 0; k < 4; ++k) dr[k] = u[k];
        dr[4] = mt; dr[5] = mr; dr[6] = tries_t; dr[7] = tries_r;
    }
}

__global__ void __launch_bounds__(kHypThreads) select_kernel(const SelectArgs a)
{
    const int i = blockIdx.x * kHypThreads + threadIdx.x;
    if (i >= a.n) return;
    const size_t base = static_cast<size_t>(i) * a.S;
    int best = 0;
    for (int h = 1; h < a.S; ++h)
        if (fit_better(a.rows + (base + h) * kFitCols, a.rows + (base + best) * kFitCols)) best = h;
    const size_t r = base + best;
    for (int k = 0; k < 16; ++k) a.poses_out[16 * static_cast<size_t>(i) + k] = a.poses[16 * r + k];
    for (int k = 0; k < kFitCols; ++k) a.fit_out[kFitCols * static_cast<size_t>(i) + k] = a.rows[kFitCols * r + k];
    for (int k = 0; k < 3; ++k) {
        if (a.trans_out) a.trans_out[3 * static_cast<size_t>(i) + k] = a.trans[3 * r + k];
        if (a.rot_out) a.rot_out[3 * static_cast<size_t>(i) + k] = a.rot[3 * r + k];
    }
    a.choice[i] = best;
}
}  // namespace

cudaError_t launch_hypotheses(const HypArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    if (!a.poses_in || !a.poses || a.S < 1 || (a.S > 1 && !a.keys) || (a.wid && !a.wid_in) || (a.width && !a.width_in))
        return cudaErrorInvalidValue;
    const int rows = a.n * a.S;
    return launch_kernel(hypotheses_kernel, dim3((rows + kHypThreads - 1) / kHypThreads), dim3(kHypThreads), 0, s, false, a);
}

cudaError_t launch_select(const SelectArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    if (!a.rows || !a.poses || !a.trans || !a.rot || !a.poses_out || !a.choice || !a.fit_out || a.S < 1) return cudaErrorInvalidValue;
    return launch_kernel(select_kernel, dim3((a.n + kHypThreads - 1) / kHypThreads), dim3(kHypThreads), 0, s, false, a);
}

}  // namespace se3tn
