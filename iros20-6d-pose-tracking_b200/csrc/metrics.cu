// Pose-error metrics on the GPU -- the first row of SURVEY.md 8(f) ("next"): what the reference's evaluation
// scripts compute on the CPU with open3d + scipy for every key-frame pose (eval_ycb.py:96-106).
//   ADD   (reference Utils.py:72-82):  mean_i || (R_p x_i + t_p) - (R_g x_i + t_g) ||
//   ADD-S (reference Utils.py:84-98):  mean_i min_j || (R_g x_i + t_g) - (R_p x_j + t_p) ||   (cKDTree, k=1)
//   VOCap (reference eval_ycb.py:45-64): area under the accuracy-threshold curve below 0.1 m, x10
// float64 throughout, no FMA contraction (-fmad=false) so distances match numpy/scipy to the last few ulps.
// The nearest-neighbour search is exhaustive (m^2 distance evaluations per pose, a few 1e6): exact by
// construction, so there is no kd-tree to mirror.
#include "metrics.h"
#include "ptx.cuh"
#include <cub/cub.cuh>
#include <algorithm>

namespace se3tn {

namespace {
constexpr int kMetricThreads = 256;
constexpr int kPredTile = 512;

__device__ __forceinline__ void xform(const double* T, double x, double y, double z, double& ox, double& oy, double& oz) {
    ox = T[0] * x + T[1] * y + T[2] * z + T[3];
    oy = T[4] * x + T[5] * y + T[6] * z + T[7];
    oz = T[8] * x + T[9] * y + T[10] * z + T[11];
}

__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
    if (threadIdx.x == 0) for (int w = 0; w < kMetricThreads / 32; ++w) s += red[w];
    __syncthreads();
    return s;                       // valid in thread 0
}

// ADD / ADD-S of one (pred, gt) pair of 4x4 poses against m model points, computed by one CTA of kMetricThreads threads; the
// values are valid in thread 0 (ADD-S only with want_adi).  Every metric kernel runs this body, so a pose scored against its own
// point set gives the same bits in each.
__device__ __forceinline__ void score_pose(const double* __restrict__ model, int m, const double* __restrict__ pred16,
                                           const double* __restrict__ gt16, bool want_adi, double& add, double& adi)
{
    __shared__ double sp[kPredTile * 3];
    __shared__ double red[kMetricThreads / 32];
    __shared__ double Tp[12], Tg[12];
    if (threadIdx.x < 12) { Tp[threadIdx.x] = pred16[threadIdx.x]; Tg[threadIdx.x] = gt16[threadIdx.x]; }
    __syncthreads();
    double sum_add = 0, sum_adi = 0;
    for (int base = 0; base < m; base += kMetricThreads) {
        const int i = base + threadIdx.x;
        const bool have = i < m;
        double gx = 0, gy = 0, gz = 0;
        if (have) {
            const double x = model[i * 3], y = model[i * 3 + 1], z = model[i * 3 + 2];
            double px, py, pz;
            xform(Tp, x, y, z, px, py, pz);
            xform(Tg, x, y, z, gx, gy, gz);
            const double dx = px - gx, dy = py - gy, dz = pz - gz;
            sum_add += sqrt(dx * dx + dy * dy + dz * dz);
        }
        if (want_adi) {
            double best = 1.0e300;
            for (int t0 = 0; t0 < m; t0 += kPredTile) {
                __syncthreads();
                for (int j = threadIdx.x; j < kPredTile && t0 + j < m; j += kMetricThreads) {
                    double px, py, pz;
                    xform(Tp, model[(t0 + j) * 3], model[(t0 + j) * 3 + 1], model[(t0 + j) * 3 + 2], px, py, pz);
                    sp[j * 3] = px; sp[j * 3 + 1] = py; sp[j * 3 + 2] = pz;
                }
                __syncthreads();
                const int cnt = min(kPredTile, m - t0);
                if (have)
                    for (int j = 0; j < cnt; ++j) {
                        const double dx = sp[j * 3] - gx, dy = sp[j * 3 + 1] - gy, dz = sp[j * 3 + 2] - gz;
                        const double d2 = dx * dx + dy * dy + dz * dz;
                        best = d2 < best ? d2 : best;
                    }
            }
            if (have) sum_adi += sqrt(best);
        }
    }
    add = block_sum(sum_add, red) / m;
    if (want_adi) adi = block_sum(sum_adi, red) / m;
}

__global__ void __launch_bounds__(kMetricThreads)
add_adi_kernel(const double* __restrict__ model, int m, const double* __restrict__ pred, const double* __restrict__ gt,
               double* __restrict__ out_add, double* __restrict__ out_adi)
{
    const int pose = blockIdx.x;
    double a, b;
    score_pose(model, m, pred + pose * 16, gt + pose * 16, out_adi != nullptr, a, b);
    if (threadIdx.x == 0) {
        if (out_add) out_add[pose] = a;
        if (out_adi) out_adi[pose] = b;
    }
}

// One CTA per pose; pose p is scored against points [offsets[s], offsets[s+1]) of the table, s = pose_set[p].
__global__ void __launch_bounds__(kMetricThreads)
add_adi_sets_kernel(const double* __restrict__ pts, const int* __restrict__ offsets, const int* __restrict__ pose_set,
                    const double* __restrict__ pred, const double* __restrict__ gt, double* __restrict__ out_add,
                    double* __restrict__ out_adi)
{
    const int pose = blockIdx.x;
    const int s = pose_set[pose], first = offsets[s];
    double a, b;
    score_pose(pts + static_cast<size_t>(first) * 3, offsets[s + 1] - first, pred + pose * 16, gt + pose * 16, out_adi != nullptr, a, b);
    if (threadIdx.x == 0) {
        if (out_add) out_add[pose] = a;
        if (out_adi) out_adi[pose] = b;
    }
}

// One CTA per row: out[row] = translation error (mm), rotation geodesic angle (degrees), ADD, ADD-S of pred against gt, the two
// metrics from score_pose on the row's point set.  keep (nullable): a row whose byte is 0 is not scored; its four values are NaN and
// its out_set entry is -1, every other row's out_set entry its set id.
__global__ void __launch_bounds__(kMetricThreads)
pose_errors_sets_kernel(const double* __restrict__ pts, const int* __restrict__ offsets, const int* __restrict__ pose_set,
                        const double* __restrict__ pred, const double* __restrict__ gt, const uint8_t* __restrict__ keep,
                        double* __restrict__ out, int* __restrict__ out_set)
{
    const int row = blockIdx.x;
    const int s = pose_set[row];
    if (keep && !keep[row]) {
        if (threadIdx.x < 4) out[row * 4 + threadIdx.x] = __longlong_as_double(0x7ff8000000000000ll);
        if (threadIdx.x == 0 && out_set) out_set[row] = -1;
        return;
    }
    const int first = offsets[s];
    const double* P = pred + row * 16;
    const double* G = gt + row * 16;
    double a, b;
    score_pose(pts + static_cast<size_t>(first) * 3, offsets[s + 1] - first, P, G, true, a, b);
    if (threadIdx.x == 0) {
        const double dx = P[3] - G[3], dy = P[7] - G[7], dz = P[11] - G[11];
        double tr = 0;                                  // tr(R^T R_gt) = sum_ij R_ij R_gt_ij, row-major order
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) tr += P[i * 4 + j] * G[i * 4 + j];
        const double cosang = fmin(1.0, fmax(-1.0, (tr - 1.0) / 2.0));
        out[row * 4 + 0] = sqrt(dx * dx + dy * dy + dz * dz) * 1000.0;
        out[row * 4 + 1] = acos(cosang) * (180.0 / 3.14159265358979323846);
        out[row * 4 + 2] = a;
        out[row * 4 + 3] = b;
        if (out_set) out_set[row] = s;
    }
}

// errs sorted ascending; ap = 10 * [ sum_j (r_j - r_{j-1}) * j/n  +  (0.1 - r_c) * c/n ],  r_0 = 0, c = #(r < 0.1).
// One CTA of kVocapThreads threads; the additions happen in an order fixed by n alone.
constexpr int kVocapThreads = 1024;

__device__ __forceinline__ void vocap_block(const double* __restrict__ rec, int n, double* __restrict__ out)
{
    __shared__ double red[32];
    __shared__ int s_c;
    if (threadIdx.x == 0) s_c = 0;
    __syncthreads();
    int c_local = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c_local += rec[i] < 0.1 ? 1 : 0;
    atomicAdd(&s_c, c_local);
    __syncthreads();
    const int c = s_c;
    double s = 0;
    for (int j = threadIdx.x + 1; j <= c; j += blockDim.x) {
        const double prev = (j == 1) ? 0.0 : rec[j - 2];
        s += (rec[j - 1] - prev) * (static_cast<double>(j) / static_cast<double>(n));
    }
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0;
        for (int w = 0; w < 32; ++w) tot += red[w];
        if (c > 0) tot += (0.1 - rec[c - 1]) * (static_cast<double>(c) / static_cast<double>(n));
        out[0] = c > 0 ? tot * 10.0 : 0.0;
    }
}

__global__ void __launch_bounds__(kVocapThreads)
vocap_kernel(const double* __restrict__ rec, int n, double* __restrict__ out)
{
    vocap_block(rec, n, out);
}

// CTA s < n_sets: the AP of segment s of seg_sorted (each segment sorted); CTA n_sets: the AP of all_sorted (all n errors).
__global__ void __launch_bounds__(kVocapThreads)
vocap_sets_kernel(const double* __restrict__ seg_sorted, const int* __restrict__ offsets, int n_sets,
                  const double* __restrict__ all_sorted, int n, double* __restrict__ out)
{
    const int s = blockIdx.x;
    if (s < n_sets) vocap_block(seg_sorted + offsets[s], offsets[s + 1] - offsets[s], out + s);
    else vocap_block(all_sorted, n, out + n_sets);
}

// counts[s] = #(set[i] == s); an id outside [0, n_sets) sets *bad instead.  counts has n_sets + 1 zeroed entries (the last
// stays 0, so an exclusive scan over all of them ends in the total).
__global__ void count_sets_kernel(const int* __restrict__ set, int n, int n_sets, int* __restrict__ counts, int* __restrict__ bad)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int s = set[i];
        if (s >= 0 && s < n_sets) atomicAdd(&counts[s], 1);
        else atomicOr(bad, 1);
    }
}
}  // namespace

cudaError_t launch_add_adi(const double* model, int m, const double* pred, const double* gt, int n,
                           double* out_add, double* out_adi, cudaStream_t s) {
    if (n <= 0 || m <= 0) return cudaSuccess;
    add_adi_kernel<<<n, kMetricThreads, 0, s>>>(model, m, pred, gt, out_add, out_adi);
    return cudaGetLastError();
}

cudaError_t launch_add_adi_sets(const double* pts, const int* offsets, const int* pose_set, const double* pred, const double* gt,
                                int n, double* out_add, double* out_adi, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    add_adi_sets_kernel<<<n, kMetricThreads, 0, s>>>(pts, offsets, pose_set, pred, gt, out_add, out_adi);
    return cudaGetLastError();
}

cudaError_t launch_pose_errors_sets(const double* pts, const int* offsets, const int* pose_set, const double* pred, const double* gt,
                                    const uint8_t* keep, int n, double* out, int* out_set, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    pose_errors_sets_kernel<<<n, kMetricThreads, 0, s>>>(pts, offsets, pose_set, pred, gt, keep, out, out_set);
    return cudaGetLastError();
}

cudaError_t vocap(const double* errs, int n, double* out_host, cudaStream_t s) {
    if (n <= 0) { *out_host = 0.0; return cudaSuccess; }
    double *sorted = nullptr, *d_out = nullptr; void* tmp = nullptr; size_t tmp_bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, errs, sorted, n, 0, 64, s);
    if (e != cudaSuccess) return e;
    if ((e = cudaMalloc(&sorted, sizeof(double) * n)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&d_out, sizeof(double))) != cudaSuccess) { cudaFree(sorted); return e; }
    if ((e = cudaMalloc(&tmp, tmp_bytes ? tmp_bytes : 1)) != cudaSuccess) { cudaFree(sorted); cudaFree(d_out); return e; }
    e = cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, errs, sorted, n, 0, 64, s);
    if (e == cudaSuccess) {
        vocap_kernel<<<1, kVocapThreads, 0, s>>>(sorted, n, d_out);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_host, d_out, sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFree(tmp); cudaFree(sorted); cudaFree(d_out);
    return e;
}


namespace {
inline size_t up256(size_t v) { return (v + 255) & ~size_t(255); }

// The scratch of vocap_sets, carved in this order: grouped ids | grouped errors | segments sorted | all sorted | counts (n_sets + 1)
// then the bad-id flag | offsets (n_sets + 1) | APs (n_sets + 1) | cub temporary storage.
struct VocapSetsLayout {
    size_t keys, grouped, seg_sorted, all_sorted, counts, offsets, out, temp, temp_bytes, total;
};

cudaError_t vocap_sets_layout(int n, int n_sets, VocapSetsLayout& L) {
    size_t a = 0, b = 0, c = 0, d = 0;
    const int* ki = nullptr; int* ko = nullptr; const double* vi = nullptr; double* vo = nullptr;
    cudaError_t e;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, a, ki, ko, vi, vo, n, 0, 32)) != cudaSuccess) return e;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, b, ki, ko, n_sets + 1)) != cudaSuccess) return e;
    if ((e = cub::DeviceSegmentedRadixSort::SortKeys(nullptr, c, vi, vo, n, n_sets, ki, ki + 1, 0, 64)) != cudaSuccess) return e;
    if ((e = cub::DeviceRadixSort::SortKeys(nullptr, d, vi, vo, n, 0, 64)) != cudaSuccess) return e;
    const size_t nd = up256(sizeof(double) * n), ni = up256(sizeof(int) * n), sets = static_cast<size_t>(n_sets) + 1;
    L.keys = 0; L.grouped = ni; L.seg_sorted = L.grouped + nd; L.all_sorted = L.seg_sorted + nd;
    L.counts = L.all_sorted + nd; L.offsets = L.counts + up256(sizeof(int) * (sets + 1));
    L.out = L.offsets + up256(sizeof(int) * sets); L.temp = L.out + up256(sizeof(double) * sets);
    L.temp_bytes = std::max(std::max(a, b), std::max(c, d));
    L.total = L.temp + up256(L.temp_bytes ? L.temp_bytes : 1);
    return cudaSuccess;
}
}  // namespace

cudaError_t vocap_sets_scratch_bytes(int n, int n_sets, size_t* bytes) {
    VocapSetsLayout L;
    const cudaError_t e = vocap_sets_layout(n, n_sets, L);
    if (e == cudaSuccess) *bytes = L.total;
    return e;
}

cudaError_t vocap_sets(const double* errs, const int* err_set, int n, int n_sets, uint8_t* scratch, double* out_host, int* bad_host,
                       cudaStream_t s) {
    VocapSetsLayout L;
    cudaError_t e = vocap_sets_layout(n, n_sets, L);
    if (e != cudaSuccess) return e;
    int* keys = reinterpret_cast<int*>(scratch + L.keys);
    double* grouped = reinterpret_cast<double*>(scratch + L.grouped);
    double* seg_sorted = reinterpret_cast<double*>(scratch + L.seg_sorted);
    double* all_sorted = reinterpret_cast<double*>(scratch + L.all_sorted);
    int* counts = reinterpret_cast<int*>(scratch + L.counts);
    int* bad = counts + n_sets + 1;
    int* offsets = reinterpret_cast<int*>(scratch + L.offsets);
    double* out = reinterpret_cast<double*>(scratch + L.out);
    void* temp = scratch + L.temp;
    size_t tb = L.temp_bytes;
    // group the errors by set (a stable sort on the ids), count each set, and turn the counts into segment offsets
    if ((e = cub::DeviceRadixSort::SortPairs(temp, tb, err_set, keys, errs, grouped, n, 0, 32, s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(counts, 0, sizeof(int) * (n_sets + 2), s)) != cudaSuccess) return e;
    count_sets_kernel<<<std::min((n + 255) / 256, 1024), 256, 0, s>>>(err_set, n, n_sets, counts, bad);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    tb = L.temp_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(temp, tb, counts, offsets, n_sets + 1, s)) != cudaSuccess) return e;
    // each segment sorted on its own, and all errors sorted together, as se3tn_vocap sorts them
    tb = L.temp_bytes;
    if ((e = cub::DeviceSegmentedRadixSort::SortKeys(temp, tb, grouped, seg_sorted, n, n_sets, offsets, offsets + 1, 0, 64, s)) != cudaSuccess) return e;
    tb = L.temp_bytes;
    if ((e = cub::DeviceRadixSort::SortKeys(temp, tb, errs, all_sorted, n, 0, 64, s)) != cudaSuccess) return e;
    vocap_sets_kernel<<<n_sets + 1, kVocapThreads, 0, s>>>(seg_sorted, offsets, n_sets, all_sorted, n, out);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(out_host, out, sizeof(double) * (n_sets + 1), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(bad_host, bad, sizeof(int), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
    return cudaStreamSynchronize(s);
}

}  // namespace se3tn
