// Depth refinement of a track step (se3tn_icp_opts): projective point-to-plane ICP of each track's model against the observed
// depth.  One iteration is render (depth + triangle ids at the current pose, render.cu) -> icp_accumulate_kernel ->
// icp_solve_kernel.  Pose T = (R, t), object -> OpenCV camera, metres, fp64.
//
// Association, per track, over the 176 x 176 crop pixels u = (row j, column i) with tri[u] >= 0, in the crop window of the
// current pose exactly as fit_kernel takes it (bbox_window at scale 1000, cv2's nearest source index floor(dst * (1 / (176 /
// size))), clamped):
//   p = (left + sx[i], top + sy[j]), skipped outside the frame; d_obs = frame_depth[p] mm, skipped when 0
//   r = K^-1 (p_x, p_y, 1)
//   the triangle tri[u] of the track's mesh in the camera frame: vertices a_k = R v_k + t, unit normal n of (a1 - a0) x (a2 - a0)
//   q = r (n.a0) / (n.r), d_model = 1000 q_z mm; skipped when |n.r| / |r| < 0.1 (grazing) or d_model <= 0
//   inlier: |d_obs - d_model| <= tau; o = r d_obs / 1000
//   e = n.(q - o), J = [(q x n)^T, n^T] for the left increment xi = (w, v): q' ~ q + w x q + v
// Sums per track: the 21 upper entries of J^T J (row-major), J^T e, sum e^2, the inlier count.  All per-pixel arithmetic is
// fp64 in the association written here, and this file is compiled with -fmad=false: every term and every inlier decision
// equals oracle/icp_ref.py's bit for bit; only the order of the sums differs.  Those run in a fixed order -- each thread's
// pixels in turn, a shuffle tree per warp, the warps in order, then the four CTAs of the track's cluster in rank order through
// distributed shared memory -- so they are bit-reproducible across runs and graph replays, with no atomics and no zeroed
// output.
//
// Solve, one thread per track: Cholesky of J^T J; with fewer than min_inliers inliers or a pivot <= 1e-12 x the largest
// diagonal entry the pose stays bit for bit.  Otherwise xi = -(J^T J)^-1 J^T e, R <- Exp(w) R, t <- Exp(w) t + v (Rodrigues).
#include "icp.h"
#include "aux_kernels.h"
#include "bbox.cuh"
#include "launch.h"
#include "ptx.cuh"
#include <cooperative_groups.h>

namespace se3tn {
namespace {
namespace cg = cooperative_groups;
constexpr int kIcpCtas = 4, kIcpThreads = 512, kIcpRows = kImg / kIcpCtas, kIcpTerms = 29;
static_assert(kImg % kIcpCtas == 0, "whole rows per CTA");
static_assert(kIcpTerms <= kIcpSums, "the sums fit their row");

__global__ void __cluster_dims__(kIcpCtas, 1, 1) __launch_bounds__(kIcpThreads)
icp_accumulate_kernel(const IcpArgs a)
{
    __shared__ int s_win[4];
    __shared__ int s_sx[kImg], s_sy[kIcpRows];
    __shared__ double s_warp[kIcpThreads / 32][kIcpTerms];
    __shared__ double s_part[kIcpTerms];
    ptx::grid_dep_launch();
    const int n = blockIdx.y, row0 = blockIdx.x * kIcpRows;
    // the poses come from the last solve or the last round's head, `tri` from the render launched right before this one:
    // every read of either, and of the frame, stays behind this wait
    ptx::grid_dep_wait();
    const double* P = a.poses + 16 * n;
    if (threadIdx.x == 0) {
        int top, left, ch, cw;
        bbox_window(P, a.fx, a.fy, a.cx, a.cy, a.object_width[n], 1000.0, 1000.0, 1000.0, top, left, ch, cw);
        s_win[0] = top; s_win[1] = left; s_win[2] = ch; s_win[3] = cw;
    }
    __syncthreads();
    const int top = s_win[0], left = s_win[1], ch = s_win[2], cw = s_win[3];
    const bool inside = ch > 0 && cw > 0;
    if (threadIdx.x < kImg) s_sx[threadIdx.x] = nearest_source(threadIdx.x, kImg, cw);       // as fit_kernel and K0 crop B
    else if (threadIdx.x >= 256 && threadIdx.x < 256 + kIcpRows) s_sy[threadIdx.x - 256] = nearest_source(row0 + threadIdx.x - 256, kImg, ch);
    __syncthreads();
    int mid = a.mesh_ids ? a.mesh_ids[n] : 0;
    if (mid < 0 || mid >= a.n_meshes) mid = 0;
    const MeshDev m = a.meshes[mid];
    double acc[kIcpTerms];
#pragma unroll
    for (int k = 0; k < kIcpTerms; ++k) acc[k] = 0.0;
    const int32_t* T = a.tri + (static_cast<size_t>(n) * kImg + row0) * kImg;
    for (int p = threadIdx.x; inside && p < kIcpRows * kImg; p += kIcpThreads) {
        const int t = T[p];
        if (t < 0 || t >= m.nf) continue;
        const int ly = p / kImg, x = p - ly * kImg;
        const int py = top + s_sy[ly], px = left + s_sx[x];
        if (py < 0 || py >= a.H || px < 0 || px >= a.W) continue;
        const int obs = a.frame_depth[static_cast<size_t>(py) * a.W + px];
        if (obs == 0) continue;
        const int i0 = m.faces[3 * t], i1 = m.faces[3 * t + 1], i2 = m.faces[3 * t + 2];
        double v[3][3];
        const int ids[3] = {i0, i1, i2};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double vx = m.pos[3 * ids[k]], vy = m.pos[3 * ids[k] + 1], vz = m.pos[3 * ids[k] + 2];
#pragma unroll
            for (int r = 0; r < 3; ++r) v[k][r] = ((P[4 * r] * vx + P[4 * r + 1] * vy) + P[4 * r + 2] * vz) + P[4 * r + 3];
        }
        const double e1x = v[1][0] - v[0][0], e1y = v[1][1] - v[0][1], e1z = v[1][2] - v[0][2];
        const double e2x = v[2][0] - v[0][0], e2y = v[2][1] - v[0][1], e2z = v[2][2] - v[0][2];
        const double cx_ = e1y * e2z - e1z * e2y, cy_ = e1z * e2x - e1x * e2z, cz_ = e1x * e2y - e1y * e2x;
        const double len = sqrt((cx_ * cx_ + cy_ * cy_) + cz_ * cz_);
        if (!(len > 0.0)) continue;
        const double il = 1.0 / len;
        const double nx = cx_ * il, ny = cy_ * il, nz = cz_ * il;
        const double rx = (static_cast<double>(px) - a.cx) / a.fx, ry = (static_cast<double>(py) - a.cy) / a.fy;
        const double ndr = (nx * rx + ny * ry) + nz;
        const double rl = sqrt((rx * rx + ry * ry) + 1.0);
        if (!(fabs(ndr / rl) >= 0.1)) continue;                  // grazing
        const double nda = (nx * v[0][0] + ny * v[0][1]) + nz * v[0][2];
        const double s = nda / ndr;
        const double dmodel = 1000.0 * s;
        if (!(dmodel > 0.0)) continue;
        const double dobs = static_cast<double>(obs);
        if (!(fabs(dobs - dmodel) <= static_cast<double>(a.tau))) continue;
        const double zo = dobs / 1000.0;
        const double qx = rx * s, qy = ry * s, qz = s;
        const double ox = rx * zo, oy = ry * zo, oz = zo;
        const double e = (nx * (qx - ox) + ny * (qy - oy)) + nz * (qz - oz);
        const double J[6] = {qy * nz - qz * ny, qz * nx - qx * nz, qx * ny - qy * nx, nx, ny, nz};
        int k = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int c = r; c < 6; ++c) acc[k++] += J[r] * J[c];
#pragma unroll
        for (int r = 0; r < 6; ++r) acc[21 + r] += J[r] * e;
        acc[27] += e * e;
        acc[28] += 1.0;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < kIcpTerms; ++k) {
        double x = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_down_sync(0xffffffffu, x, off);
        if (lane == 0) s_warp[warp][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < kIcpTerms) {
        double x = 0.0;
        for (int w = 0; w < kIcpThreads / 32; ++w) x += s_warp[w][threadIdx.x];
        s_part[threadIdx.x] = x;
    }
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();                                          // every CTA's partial sums are written
    if (cluster.block_rank() == 0 && threadIdx.x < kIcpTerms) {
        double x = 0.0;
        for (int r = 0; r < kIcpCtas; ++r) x += cluster.map_shared_rank(s_part, r)[threadIdx.x];
        a.sums[n * kIcpSums + threadIdx.x] = x;
    }
    cluster.sync();                                          // no CTA exits while CTA 0 still reads its shared memory
}

constexpr int kSolveThreads = 64;
__global__ void __launch_bounds__(kSolveThreads)
icp_solve_kernel(const IcpArgs a, int n_tracks)
{
    ptx::grid_dep_launch();
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    ptx::grid_dep_wait();                                    // the sums come from the accumulation right before this launch
    if (n >= n_tracks) return;
    const double* S = a.sums + n * kIcpSums;
    double A[6][6], b[6];
    int k = 0;
    for (int r = 0; r < 6; ++r)
        for (int c = r; c < 6; ++c) { A[r][c] = S[k]; A[c][r] = S[k]; ++k; }
    for (int r = 0; r < 6; ++r) b[r] = S[21 + r];
    const double e2 = S[27], cnt = S[28];
    double maxd = 0.0;
    for (int r = 0; r < 6; ++r) maxd = fmax(maxd, A[r][r]);
    bool ok = cnt >= static_cast<double>(a.min_inliers) && maxd > 0.0 && isfinite(maxd);
    double L[6][6] = {};
    for (int j = 0; ok && j < 6; ++j) {
        double d = A[j][j];
        for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
        if (!(d > 1e-12 * maxd)) { ok = false; break; }
        L[j][j] = sqrt(d);
        for (int i = j + 1; i < 6; ++i) {
            double x = A[i][j];
            for (int q = 0; q < j; ++q) x -= L[i][q] * L[j][q];
            L[i][j] = x / L[j][j];
        }
    }
    double step_mm = 0.0, step_deg = 0.0;
    if (ok) {
        double y[6], xi[6];
        for (int i = 0; i < 6; ++i) {                        // L y = -b
            double x = -b[i];
            for (int q = 0; q < i; ++q) x -= L[i][q] * y[q];
            y[i] = x / L[i][i];
        }
        for (int i = 5; i >= 0; --i) {                       // L^T xi = y
            double x = y[i];
            for (int q = i + 1; q < 6; ++q) x -= L[q][i] * xi[q];
            xi[i] = x / L[i][i];
        }
        const double th = sqrt((xi[0] * xi[0] + xi[1] * xi[1]) + xi[2] * xi[2]);
        double E[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
        if (th > 0.0) {                                      // Rodrigues: cos th I + sin th [k]x + (1 - cos th) k k^T
            const double kx = xi[0] / th, ky = xi[1] / th, kz = xi[2] / th, c = cos(th), s = sin(th), c1 = 1.0 - c;
            E[0][0] = c + c1 * kx * kx;      E[0][1] = c1 * kx * ky - s * kz; E[0][2] = c1 * kx * kz + s * ky;
            E[1][0] = c1 * ky * kx + s * kz; E[1][1] = c + c1 * ky * ky;      E[1][2] = c1 * ky * kz - s * kx;
            E[2][0] = c1 * kz * kx - s * ky; E[2][1] = c1 * kz * ky + s * kx; E[2][2] = c + c1 * kz * kz;
        }
        double* P = a.poses + 16 * n;
        double R[3][3], t[3];
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) R[r][c] = P[4 * r + c]; t[r] = P[4 * r + 3]; }
        double d2 = 0.0;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) P[4 * r + c] = (E[r][0] * R[0][c] + E[r][1] * R[1][c]) + E[r][2] * R[2][c];
            const double tn = ((E[r][0] * t[0] + E[r][1] * t[1]) + E[r][2] * t[2]) + xi[3 + r];
            P[4 * r + 3] = tn;
            d2 += (tn - t[r]) * (tn - t[r]);
        }
        step_mm = sqrt(d2) * 1000.0;
        step_deg = th * (180.0 / 3.14159265358979323846);
    }
    if (a.stats) {
        double* o = a.stats + n * kIcpCols;
        o[0] = cnt; o[1] = cnt > 0.0 ? sqrt(e2 / cnt) * 1000.0 : 0.0; o[2] = step_mm; o[3] = step_deg;
    }
}
}  // namespace

cudaError_t launch_icp(const IcpArgs& a, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (!a.poses || !a.object_width || !a.meshes || !a.frame_depth || !a.tri || !a.sums || a.tau < 1 || a.tau > 1000)
        return cudaErrorInvalidValue;
    cudaError_t e = launch_kernel(icp_accumulate_kernel, dim3(kIcpCtas, n), dim3(kIcpThreads), 0, s, true, a);
    if (e != cudaSuccess) return e;
    return launch_kernel(icp_solve_kernel, dim3((n + kSolveThreads - 1) / kSolveThreads), dim3(kSolveThreads), 0, s, true, a, n);
}

}  // namespace se3tn
