// Start poses without a previous pose (se3tn_init_poses): render-and-compare of a rotation grid against an object's
// segmentation mask and the observed depth.  Five kinds of launch, all on the caller's stream:
//
// mask_pass_kernel / mask_finish_kernel: for object i with label l_i, over the whole H x W frame, mask = #(seg == l_i),
//   depth_px = #(seg == l_i, depth > 0), sum_u / sum_v = the sums of the mask pixels' columns / rows, and z_med = the lower
//   median (sorted index (depth_px - 1) / 2) of the depths > 0 under the mask, from a 65536-bin histogram.  Integer atomics
//   only: the statistics are exact and do not depend on the order of the reduction.  status 1: mask = 0; 2: depth_px <
//   min_pixels.  t0 = z_med / 1000 * ((u - cx) / fx, (v - cy) / fy, 1), (u, v) = (sum_u, sum_v) / mask, in fp64; an object
//   with status != 0 gets the placeholder t0 = (0, 0, 1), which keeps every later launch on finite poses.
// box_pass_kernel (se3tn_init_boxes): the same statistics over the pixels of object i's half-open box (x0, y0, x1, y1)
//   instead of seg == l_i, one grid slice per object.  mask_finish_kernel then also takes D depth candidates z_d = the sorted
//   depth at index max(0, floor(((2 d + 1) depth_px - D) / (2 D))), d < D, with t0_d = z_d / 1000 K^-1 (u, v, 1): t0 is
//   [n][D][3]; D = 1 is the lower median, the mask call's t0.
// grid_kernel: candidate c = d V R + v R + r (d = 0 with a mask).  d_v = (sqrt(1 - z^2) cos phi, sqrt(1 - z^2) sin phi, z), z = 1 - (2 v + 1) / V,
//   phi = v pi (3 - sqrt 5): a Fibonacci-sphere direction in the object frame.  The camera axes in object coordinates are
//   z_c = -d_v, x_c = (z_c x up) / |z_c x up|, y_c = z_c x x_c with up = +z (+y when |d_v.z| > 0.99), so R_c = [x_c; y_c; z_c]
//   maps d_v to the camera's -z axis; the candidate turns that about the camera's z axis by th = 2 pi r / R:
//   rows (cos th x_c - sin th y_c, sin th x_c + cos th y_c, z_c).  Translation t0_d.  fp64, restated in oracle/init_ref.py.
// score_kernel: one 4-CTA cluster per rendered row, as fit_kernel: the crop window of the row's pose (bbox_window, cv2's
//   nearest source index, 0 outside the frame) gives the observed depth O and the mask M = (seg == l_i) under each of the
//   176 x 176 pixels of the rendered depth R (with boxes, M = the source pixel lies in object i's box).  model #(R>0), maskc #M, overlap #(R>0, M), pairs #(R>0, M, O>0) and
//   S = sum (O - R) over the pairs; after a cluster barrier delta = floor((2 S + pairs) / (2 pairs)) mm (0 without pairs,
//   or when the row is scored where it is), then inlier #(R>0, M, O>0, |O - (R + delta)| <= tau).
// keep_kernel: per object, the K best rows in rank order; the kept grid pose moves along its ray: t = t0 (1 + delta / (1000 t0_z)).
// choose_kernel: per object, the best of its K (refined and rescored) rows; NaN pose when the status is not 0.
//
// Rank: the higher inlier / union (union = model + maskc - overlap; a row with union 0 scores 0), compared as int64 cross
// products; then the higher overlap; then the lower candidate index.  Compiled with -fmad=false.
#include "init.h"
#include "aux_kernels.h"
#include "bbox.cuh"
#include "launch.h"
#include "ptx.cuh"
#include <algorithm>
#include <cooperative_groups.h>
#include <math_constants.h>

namespace se3tn {
namespace {
namespace cg = cooperative_groups;

// ---- mask statistics ----------------------------------------------------------------------------------------------------
constexpr int kMaskThreads = 256, kMaskBlocks = 264;

__global__ void __launch_bounds__(kMaskThreads) mask_pass_kernel(const MaskArgs a)
{
    extern __shared__ unsigned long long s_acc[];            // [n][kInitAcc], then the n labels as int
    int* s_lab = reinterpret_cast<int*>(s_acc + static_cast<size_t>(a.n) * kInitAcc);
    for (int k = threadIdx.x; k < a.n * kInitAcc; k += kMaskThreads) s_acc[k] = 0;
    for (int k = threadIdx.x; k < a.n; k += kMaskThreads) s_lab[k] = a.labels[k];
    __syncthreads();
    const size_t total = static_cast<size_t>(a.H) * a.W;
    for (size_t p = blockIdx.x * static_cast<size_t>(kMaskThreads) + threadIdx.x; p < total; p += static_cast<size_t>(gridDim.x) * kMaskThreads) {
        const int l = a.seg[p];
        if (l == 0) continue;
        const int d = a.depth[p];
        const unsigned long long u = p % a.W, v = p / a.W;
        for (int i = 0; i < a.n; ++i) {
            if (s_lab[i] != l) continue;
            unsigned long long* acc = s_acc + i * kInitAcc;
            atomicAdd(acc, 1ull);
            atomicAdd(acc + 2, u);
            atomicAdd(acc + 3, v);
            if (d > 0) {
                atomicAdd(acc + 1, 1ull);
                atomicAdd(a.hist + static_cast<size_t>(i) * kInitBins + d, 1u);
            }
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < a.n * kInitAcc; k += kMaskThreads)
        if (s_acc[k]) atomicAdd(a.acc + k, s_acc[k]);
}

// se3tn_init_boxes: blockIdx.y is the object, the x CTAs stride over its own box's pixels only (the same accumulators and
// histogram as mask_pass_kernel)
__global__ void __launch_bounds__(kMaskThreads) box_pass_kernel(const MaskArgs a)
{
    __shared__ unsigned long long s_acc[kInitAcc];
    const int i = blockIdx.y;
    const int x0 = a.boxes[4 * i], y0 = a.boxes[4 * i + 1], x1 = a.boxes[4 * i + 2], y1 = a.boxes[4 * i + 3];
    if (threadIdx.x < kInitAcc) s_acc[threadIdx.x] = 0;
    __syncthreads();
    const long long bw = x1 - x0, total = bw * (y1 - y0);
    unsigned* hist = a.hist + static_cast<size_t>(i) * kInitBins;
    unsigned long long own[kInitAcc] = {0, 0, 0, 0};        // integer sums: exact in any order
    for (long long p = blockIdx.x * static_cast<long long>(kMaskThreads) + threadIdx.x; p < total; p += static_cast<long long>(gridDim.x) * kMaskThreads) {
        const long long v = y0 + p / bw, u = x0 + p % bw;
        const int d = a.depth[v * a.W + u];
        ++own[0]; own[2] += u; own[3] += v;
        if (d > 0) {
            ++own[1];
            atomicAdd(hist + d, 1u);
        }
    }
    for (int k = 0; k < kInitAcc; ++k)
        if (own[k]) atomicAdd(s_acc + k, own[k]);
    __syncthreads();
    if (threadIdx.x < kInitAcc && s_acc[threadIdx.x]) atomicAdd(a.acc + i * kInitAcc + threadIdx.x, s_acc[threadIdx.x]);
}

constexpr int kFinishThreads = 1024, kBinsPerThread = kInitBins / kFinishThreads;
static_assert(kInitBins % kFinishThreads == 0, "whole bins per thread");

// The sorted index of depth candidate d of D among depth_px depths: the quantile (2 d + 1) / 2 D, floored and clamped at 0.
// D = 1 gives the lower median (depth_px - 1) / 2.
__device__ __forceinline__ unsigned long long quantile_index(int d, int D, unsigned long long depth_px) {
    const long long num = static_cast<long long>(2 * d + 1) * static_cast<long long>(depth_px) - D;
    return num < 0 ? 0ull : static_cast<unsigned long long>(num / (2 * D));
}

__global__ void __launch_bounds__(kFinishThreads) mask_finish_kernel(const MaskArgs a)
{
    __shared__ unsigned s_scan[kFinishThreads];
    __shared__ int s_z[1 + kInitMaxDepths];                  // the lower median, then the D depth candidates
    const int i = blockIdx.x, t = threadIdx.x;
    const unsigned long long* acc = a.acc + i * kInitAcc;
    const unsigned long long mask = acc[0], depth_px = acc[1];
    const unsigned* h = a.hist + static_cast<size_t>(i) * kInitBins + t * kBinsPerThread;
    unsigned own = 0;
    for (int b = 0; b < kBinsPerThread; ++b) own += h[b];
    s_scan[t] = own;
    if (t <= a.D) s_z[t] = 0;
    __syncthreads();
    for (int off = 1; off < kFinishThreads; off <<= 1) {     // inclusive Hillis-Steele scan
        const unsigned x = t >= off ? s_scan[t - off] : 0u;
        __syncthreads();
        s_scan[t] += x;
        __syncthreads();
    }
    if (depth_px > 0) {
        const unsigned long long hi = s_scan[t], lo = hi - own;
        for (int q = 0; q <= a.D; ++q) {
            const unsigned long long k = q == 0 ? (depth_px - 1) / 2 : quantile_index(q - 1, a.D, depth_px);   // sorted index
            if (k < lo || k >= hi) continue;
            unsigned long long c = lo;
            for (int b = 0; b < kBinsPerThread; ++b) {
                c += h[b];
                if (k < c) { s_z[q] = t * kBinsPerThread + b; break; }
            }
        }
    }
    __syncthreads();
    if (t != 0) return;
    const int status = mask == 0 ? 1 : (depth_px < static_cast<unsigned long long>(a.min_pixels) ? 2 : 0);
    long long* st = a.stats + i * kInitStats;
    st[0] = status; st[1] = static_cast<long long>(mask); st[2] = static_cast<long long>(depth_px);
    st[3] = static_cast<long long>(acc[2]); st[4] = static_cast<long long>(acc[3]); st[5] = s_z[0];
    const double m = static_cast<double>(mask);
    const double u = static_cast<double>(acc[2]) / m, v = static_cast<double>(acc[3]) / m;
    for (int d = 0; d < a.D; ++d) {
        double* t0 = a.t0 + 3 * (static_cast<size_t>(i) * a.D + d);
        if (status) { t0[0] = 0.0; t0[1] = 0.0; t0[2] = 1.0; continue; }
        const double z = static_cast<double>(s_z[1 + d]) / 1000.0;
        t0[0] = z * ((u - a.cx) / a.fx);
        t0[1] = z * ((v - a.cy) / a.fy);
        t0[2] = z;
    }
}

// ---- rotation grid ------------------------------------------------------------------------------------------------------
constexpr int kGridThreads = 128;

__global__ void __launch_bounds__(kGridThreads) grid_kernel(const GridArgs a)
{
    const int VR = a.V * a.R, per = a.D * VR;
    const long long g = static_cast<long long>(blockIdx.x) * kGridThreads + threadIdx.x;
    if (g >= static_cast<long long>(a.n) * per) return;
    const int i = static_cast<int>(g / per), cd = static_cast<int>(g - static_cast<long long>(i) * per), dz = cd / VR;
    const int c = cd - dz * VR, v = c / a.R, r = c - v * a.R;
    const double z = 1.0 - (2.0 * v + 1.0) / a.V;
    const double rad = sqrt(1.0 - z * z);
    const double phi = v * (CUDART_PI * (3.0 - sqrt(5.0)));
    const double d[3] = {rad * cos(phi), rad * sin(phi), z};
    const double up[3] = {0.0, fabs(z) > 0.99 ? 1.0 : 0.0, fabs(z) > 0.99 ? 0.0 : 1.0};
    const double zc[3] = {-d[0], -d[1], -d[2]};
    double xc[3] = {zc[1] * up[2] - zc[2] * up[1], zc[2] * up[0] - zc[0] * up[2], zc[0] * up[1] - zc[1] * up[0]};
    const double il = 1.0 / sqrt((xc[0] * xc[0] + xc[1] * xc[1]) + xc[2] * xc[2]);
    for (int k = 0; k < 3; ++k) xc[k] = xc[k] * il;
    const double yc[3] = {zc[1] * xc[2] - zc[2] * xc[1], zc[2] * xc[0] - zc[0] * xc[2], zc[0] * xc[1] - zc[1] * xc[0]};
    const double th = (2.0 * CUDART_PI) * r / a.R;
    const double ct = cos(th), st = sin(th);
    double* P = a.poses + 16 * g;
    const double* t0 = a.t0 + 3 * (static_cast<long long>(i) * a.D + dz);
    for (int k = 0; k < 3; ++k) {
        P[k] = ct * xc[k] - st * yc[k];
        P[4 + k] = st * xc[k] + ct * yc[k];
        P[8 + k] = zc[k];
    }
    P[3] = t0[0]; P[7] = t0[1]; P[11] = t0[2];
    P[12] = 0.0; P[13] = 0.0; P[14] = 0.0; P[15] = 1.0;
    a.width[g] = a.width_in[i];
    if (a.ids) a.ids[g] = a.ids_in[i];
}

// ---- render and score ---------------------------------------------------------------------------------------------------
constexpr int kScoreCtas = 4, kScoreThreads = 512, kScoreRows = kImg / kScoreCtas, kScoreSums = 6;
static_assert(kImg % kScoreCtas == 0, "whole rows per CTA");

__device__ __forceinline__ long long floor_div(long long a, long long b) {   // b > 0
    const long long q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

// true when score row x ranks strictly above row y (columns as kInitCols)
__device__ __forceinline__ bool ranks_above(const int32_t* x, const int32_t* y) {
    const long long ux = static_cast<long long>(x[2]) + x[3] - x[4], uy = static_cast<long long>(y[2]) + y[3] - y[4];
    const long long ix = x[6], iy = y[6];
    const long long lhs = ix * (uy > 0 ? uy : 1), rhs = iy * (ux > 0 ? ux : 1);
    if (lhs != rhs) return lhs > rhs;
    if (x[4] != y[4]) return x[4] > y[4];
    return x[1] < y[1];
}

__global__ void __cluster_dims__(kScoreCtas, 1, 1) __launch_bounds__(kScoreThreads)
score_kernel(const ScoreArgs a)
{
    __shared__ int s_win[4];
    __shared__ int s_sx[kImg], s_sy[kScoreRows];
    __shared__ long long s_warp[kScoreThreads / 32][kScoreSums];
    __shared__ long long s_part[kScoreSums];
    __shared__ long long s_tot[4], s_delta;           // CTA 0: the cluster's model, maskc, overlap, pairs; delta
    ptx::grid_dep_launch();
    const int r = blockIdx.y, row0 = blockIdx.x * kScoreRows;
    const long long g = static_cast<long long>(a.row0) + r;
    const int obj = static_cast<int>(g / a.per_object);
    // the poses come from the grid or ICP, `rendered` from the render launched right before this one: every read stays
    // behind this wait
    ptx::grid_dep_wait();
    const int label = a.boxes ? 0 : a.labels[obj];
    const int* box = a.boxes ? a.boxes + 4 * obj : nullptr;
    const int bx0 = box ? box[0] : 0, by0 = box ? box[1] : 0, bx1 = box ? box[2] : 0, by1 = box ? box[3] : 0;
    if (threadIdx.x == 0) {
        int top, left, ch, cw;
        bbox_window(a.poses + 16 * g, a.fx, a.fy, a.cx, a.cy, a.object_width[g], 1000.0, 1000.0, 1000.0, top, left, ch, cw);
        s_win[0] = top; s_win[1] = left; s_win[2] = ch; s_win[3] = cw;
    }
    __syncthreads();
    const int top = s_win[0], left = s_win[1], ch = s_win[2], cw = s_win[3];
    const bool inside = ch > 0 && cw > 0;
    if (threadIdx.x < kImg) s_sx[threadIdx.x] = nearest_source(threadIdx.x, kImg, cw);      // as fit_kernel and K0 crop B
    else if (threadIdx.x >= 256 && threadIdx.x < 256 + kScoreRows) s_sy[threadIdx.x - 256] = nearest_source(row0 + threadIdx.x - 256, kImg, ch);
    __syncthreads();
    const uint16_t* R = a.rendered + (static_cast<size_t>(r) * kImg + row0) * kImg;
    // the frame pixel under crop pixel p (-1: outside the frame or no window)
    auto source = [&](int p) -> long long {
        if (!inside) return -1;
        const int ly = p / kImg, x = p - ly * kImg;
        const int fy = top + s_sy[ly], fx = left + s_sx[x];
        if (fy < 0 || fy >= a.H || fx < 0 || fx >= a.W) return -1;
        return static_cast<long long>(fy) * a.W + fx;
    };
    // M of frame pixel q >= 0: its label, or with boxes whether it lies in the object's box (H x W < 2^31: q fits an int)
    auto member = [&](long long q) -> bool {
        if (!box) return a.seg[q] == label;
        const int fy = static_cast<int>(q) / a.W, fx = static_cast<int>(q) - fy * a.W;
        return fx >= bx0 && fx < bx1 && fy >= by0 && fy < by1;
    };
    int model = 0, maskc = 0, overlap = 0, pairs = 0, sum = 0;     // sum: at most 16 pixels x 65535 per thread
    for (int p = threadIdx.x; p < kScoreRows * kImg; p += kScoreThreads) {
        const int rd = R[p];
        const long long q = source(p);
        const bool m = q >= 0 && member(q);
        model += rd > 0; maskc += m;
        if (!(rd > 0 && m)) continue;
        ++overlap;
        const int o = a.frame_depth[q];
        if (o == 0) continue;
        ++pairs; sum += o - rd;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    cg::cluster_group cluster = cg::this_cluster();
    {
        const int v[5] = {model, maskc, overlap, pairs, sum};
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int s = static_cast<int>(__reduce_add_sync(0xffffffffu, static_cast<unsigned>(v[k])));   // |warp sum| < 2^31
            if (lane == 0) s_warp[warp][k] = s;
        }
        __syncthreads();
        if (threadIdx.x < 5) {
            long long s = 0;
            for (int w = 0; w < kScoreThreads / 32; ++w) s += s_warp[w][threadIdx.x];
            s_part[threadIdx.x] = s;
        }
        cluster.sync();                                      // every CTA's partial sums are written
        if (cluster.block_rank() == 0 && threadIdx.x == 0) {
            long long tot[5] = {0, 0, 0, 0, 0};
            for (int q = 0; q < kScoreCtas; ++q)
                for (int k = 0; k < 5; ++k) tot[k] += cluster.map_shared_rank(s_part, q)[k];
            const long long np = tot[3];
            s_delta = (a.fixed_delta || np == 0) ? 0 : floor_div(2 * tot[4] + np, 2 * np);
            for (int k = 0; k < 4; ++k) s_tot[k] = tot[k];
        }
        cluster.sync();                                      // delta is set
    }
    const long long delta = *cluster.map_shared_rank(&s_delta, 0);
    int inlier = 0;
    for (int p = threadIdx.x; p < kScoreRows * kImg; p += kScoreThreads) {
        const int rd = R[p];
        if (rd == 0) continue;
        const long long q = source(p);
        if (q < 0 || !member(q)) continue;
        const int o = a.frame_depth[q];
        if (o == 0) continue;
        const long long e = static_cast<long long>(o) - (rd + delta);
        inlier += (e < 0 ? -e : e) <= a.tau;
    }
    const int s = static_cast<int>(__reduce_add_sync(0xffffffffu, static_cast<unsigned>(inlier)));
    __shared__ int s_in[kScoreThreads / 32];
    __shared__ int s_inl;
    if (lane == 0) s_in[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int x = 0;
        for (int w = 0; w < kScoreThreads / 32; ++w) x += s_in[w];
        s_inl = x;
    }
    cluster.sync();                                          // every CTA's inlier count is written
    if (cluster.block_rank() == 0 && threadIdx.x == 0) {
        int tot = 0;
        for (int q = 0; q < kScoreCtas; ++q) tot += *cluster.map_shared_rank(&s_inl, q);
        int32_t* o = a.rows + kInitCols * g;
        const int cand = a.cand_rows ? a.cand_rows[kInitCols * g + 1] : static_cast<int>(g - static_cast<long long>(obj) * a.per_object);
        o[0] = static_cast<int32_t>(a.stats[kInitStats * obj]); o[1] = cand;
        for (int k = 0; k < 4; ++k) o[2 + k] = static_cast<int32_t>(s_tot[k]);
        o[6] = tot; o[7] = static_cast<int32_t>(delta);
    }
    cluster.sync();                                          // no CTA exits while CTA 0 still reads its shared memory
}

// ---- keep K, choose one -------------------------------------------------------------------------------------------------
constexpr int kKeepThreads = 1024;

__global__ void __launch_bounds__(kKeepThreads) keep_kernel(const KeepArgs a)
{
    __shared__ int s_best[kKeepThreads / 32];
    __shared__ int s_prev;
    const int i = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t* rows = a.rows + static_cast<size_t>(i) * a.per_object * kInitCols;
    for (int k = 0; k < a.K; ++k) {
        const int prev = k == 0 ? -1 : s_prev;
        int best = -1;
        for (int j = threadIdx.x; j < a.per_object; j += kKeepThreads) {
            if (prev >= 0 && !ranks_above(rows + kInitCols * prev, rows + kInitCols * j)) continue;   // kept already
            if (best < 0 || ranks_above(rows + kInitCols * j, rows + kInitCols * best)) best = j;
        }
        for (int off = 16; off > 0; off >>= 1) {
            const int o = __shfl_down_sync(0xffffffffu, best, off);
            if (o >= 0 && (best < 0 || ranks_above(rows + kInitCols * o, rows + kInitCols * best))) best = o;
        }
        if (lane == 0) s_best[warp] = best;
        __syncthreads();
        if (threadIdx.x == 0) {
            int b = -1;
            for (int w = 0; w < kKeepThreads / 32; ++w) {
                const int o = s_best[w];
                if (o >= 0 && (b < 0 || ranks_above(rows + kInitCols * o, rows + kInitCols * b))) b = o;
            }
            s_prev = b;                                      // K <= per_object: there always is one
            const size_t dst = static_cast<size_t>(i) * a.K + k, src = static_cast<size_t>(i) * a.per_object + b;
            for (int c = 0; c < kInitCols; ++c) a.kept_rows[kInitCols * dst + c] = rows[kInitCols * b + c];
            const double* P = a.poses + 16 * src;
            double* Q = a.kept_poses + 16 * dst;
            for (int c = 0; c < 16; ++c) Q[c] = P[c];
            const double f = 1.0 + static_cast<double>(rows[kInitCols * b + 7]) / (1000.0 * P[11]);
            Q[3] = P[3] * f; Q[7] = P[7] * f; Q[11] = P[11] * f;
            a.kept_width[dst] = a.width_in[i];
            if (a.kept_ids) a.kept_ids[dst] = a.ids_in[i];
        }
        __syncthreads();
    }
}

__global__ void choose_kernel(const ChooseArgs a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const size_t base = static_cast<size_t>(i) * a.K;
    size_t best = base;
    for (int k = 1; k < a.K; ++k)
        if (ranks_above(a.rows + kInitCols * (base + k), a.rows + kInitCols * best)) best = base + k;
    const bool ok = a.stats[kInitStats * i] == 0;
    for (int c = 0; c < 16; ++c) a.poses_out[16 * i + c] = ok ? a.poses[16 * best + c] : CUDART_NAN;
    for (int c = 0; c < kInitCols; ++c) a.rows_out[kInitCols * i + c] = a.rows[kInitCols * best + c];
}
}  // namespace

cudaError_t launch_mask_stats(const MaskArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    if (!a.depth || !(a.boxes || (a.seg && a.labels)) || !a.acc || !a.hist || !a.stats || !a.t0 || a.H <= 0 || a.W <= 0 ||
        a.D < 1 || a.D > kInitMaxDepths || (!a.boxes && a.D != 1) || a.box_px_max < 0)
        return cudaErrorInvalidValue;
    cudaError_t e = cudaMemsetAsync(a.acc, 0, sizeof(unsigned long long) * kInitAcc * a.n, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.hist, 0, sizeof(unsigned) * kInitBins * static_cast<size_t>(a.n), s);
    if (e != cudaSuccess) return e;
    if (a.boxes) {
        const int blocks = static_cast<int>(std::max<long long>(1, std::min<long long>(kMaskBlocks, (a.box_px_max + kMaskThreads - 1) / kMaskThreads)));
        if ((e = launch_kernel(box_pass_kernel, dim3(blocks, a.n), dim3(kMaskThreads), 0, s, false, a)) != cudaSuccess) return e;
        return launch_kernel(mask_finish_kernel, dim3(a.n), dim3(kFinishThreads), 0, s, false, a);
    }
    const size_t smem = static_cast<size_t>(a.n) * (kInitAcc * sizeof(unsigned long long) + sizeof(int));
    if ((e = set_max_dynamic_smem<mask_pass_kernel>(smem)) != cudaSuccess) return e;
    const long long px = static_cast<long long>(a.H) * a.W;
    const int blocks = static_cast<int>(std::min<long long>(kMaskBlocks, (px + kMaskThreads - 1) / kMaskThreads));
    if ((e = launch_kernel(mask_pass_kernel, dim3(blocks), dim3(kMaskThreads), smem, s, false, a)) != cudaSuccess) return e;
    return launch_kernel(mask_finish_kernel, dim3(a.n), dim3(kFinishThreads), 0, s, false, a);
}

cudaError_t launch_grid(const GridArgs& a, cudaStream_t s) {
    const long long rows = static_cast<long long>(a.n) * a.D * a.V * a.R;
    if (rows <= 0) return cudaSuccess;
    if (a.D < 1 || a.D > kInitMaxDepths || !a.t0 || !a.width_in || !a.poses || !a.width || (a.ids && !a.ids_in)) return cudaErrorInvalidValue;
    return launch_kernel(grid_kernel, dim3(static_cast<unsigned>((rows + kGridThreads - 1) / kGridThreads)), dim3(kGridThreads), 0, s,
                         false, a);
}

cudaError_t launch_score(const ScoreArgs& a, int chunk_rows, cudaStream_t s) {
    if (chunk_rows <= 0) return cudaSuccess;
    if (!a.poses || !a.object_width || !a.frame_depth || !(a.boxes || (a.seg && a.labels)) || !a.rendered || !a.stats || !a.rows ||
        a.per_object <= 0 || a.tau < 1 || a.tau > 1000)
        return cudaErrorInvalidValue;
    return launch_kernel(score_kernel, dim3(kScoreCtas, chunk_rows), dim3(kScoreThreads), 0, s, true, a);
}

cudaError_t launch_keep(const KeepArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    if (!a.rows || !a.poses || !a.width_in || !a.kept_rows || !a.kept_poses || !a.kept_width || a.K < 1 || a.K > kInitMaxKeep ||
        a.K > a.per_object || (a.kept_ids && !a.ids_in))
        return cudaErrorInvalidValue;
    return launch_kernel(keep_kernel, dim3(a.n), dim3(kKeepThreads), 0, s, false, a);
}

cudaError_t launch_choose(const ChooseArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    if (!a.rows || !a.poses || !a.stats || !a.poses_out || !a.rows_out || a.K < 1) return cudaErrorInvalidValue;
    return launch_kernel(choose_kernel, dim3((a.n + 127) / 128), dim3(128), 0, s, false, a);
}

}  // namespace se3tn
