// Track overlays for the sequence drivers' result videos: the drawing of the reference's getResultsYcb (predict.py:424-433) and
// predictSequenceYcb / predictSequenceYcbInEOAT (predict.py:549-560, 612-624), for n tracks of one frame at once.
//   points   model points moved by the track's pose, x' = ((R00 x + R01 y) + R02 z) + t0 (no FMA), then project_points
//            (predict.py:81-86): u = (x' fx) / z' + cx, v = (y' fy) / z' + cy, rounded half to even.  A point whose u or v is
//            not finite or beyond +-2^30 is not drawn; z' < 0 is drawn wherever it lands, as the reference draws it.
//   circles  cv2.circle(radius=1, thickness=-1) sets the plus of 5 pixels (u, v), (u+-1, v), (u, v+-1), clipped to the image,
//            all in (0,255,255): one bit per pixel in a per-track mask (splat_kernel).
//   label    the pixels cv2.putText sets (a host-rendered 0 / 255 mask of full-width rows) in (255,0,0), under or over the dots.
//   resize   cv2.resize(.., (W/2, H/2)) with INTER_LINEAR at an exact factor of 2 is (a + b + c + d + 2) >> 2 over each 2 x 2
//            block (compose_kernel, which also swaps RGB to BGR).
#include "overlay.h"
#include <algorithm>

namespace se3tn {

namespace {
constexpr int kThreads = 256;
constexpr double kMaxCoord = 1073741824.0;   // 2^30

__device__ __forceinline__ double row(const double* T, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[1], y)), __dmul_rn(T[2], z)), T[3]);
}

__device__ __forceinline__ void set_bit(uint32_t* mask, int H, int W, int u, int v) {
    if (u < 0 || u >= W || v < 0 || v >= H) return;
    const size_t p = static_cast<size_t>(v) * W + u;
    atomicOr(mask + (p >> 5), 1u << (p & 31));
}

// grid (points / kThreads, tracks): thread p of track i draws point p of the track's set into mask i
__global__ void __launch_bounds__(kThreads)
splat_kernel(const double* __restrict__ pts, const int* __restrict__ offsets, const int* __restrict__ track_set,
             const double* __restrict__ poses, int n, double fx, double fy, double cx, double cy, int H, int W, size_t words,
             uint32_t* __restrict__ masks)
{
    const int p = blockIdx.x * kThreads + threadIdx.x;
    for (int i = blockIdx.y; i < n; i += gridDim.y) {
        const int s = track_set[i], first = offsets[s];
        if (p >= offsets[s + 1] - first) continue;
        const double* T = poses + 16 * static_cast<size_t>(i);
        const double* q = pts + 3 * (static_cast<size_t>(first) + p);
        const double x = q[0], y = q[1], z = q[2];
        const double X = row(T, x, y, z), Y = row(T + 4, x, y, z), Z = row(T + 8, x, y, z);
        const double u = rint(__dadd_rn(__ddiv_rn(__dmul_rn(X, fx), Z), cx));
        const double v = rint(__dadd_rn(__ddiv_rn(__dmul_rn(Y, fy), Z), cy));
        if (!(fabs(u) <= kMaxCoord && fabs(v) <= kMaxCoord)) continue;      // also NaN and inf
        const int iu = static_cast<int>(u), iv = static_cast<int>(v);
        uint32_t* m = masks + words * i;
        set_bit(m, H, W, iu, iv);
        set_bit(m, H, W, iu - 1, iv);
        set_bit(m, H, W, iu + 1, iv);
        set_bit(m, H, W, iu, iv - 1);
        set_bit(m, H, W, iu, iv + 1);
    }
}

// one thread per output pixel of every track: the 2 x 2 source pixels drawn, then averaged
__global__ void __launch_bounds__(kThreads)
compose_kernel(const uint8_t* __restrict__ rgb, int H, int W, const uint32_t* __restrict__ masks, size_t words,
               const uint8_t* __restrict__ label, int label_y0, int label_h, int label_over, int n, uint8_t* __restrict__ out)
{
    const int h2 = H / 2, w2 = W / 2;
    const size_t per = static_cast<size_t>(h2) * w2, total = per * n;
    for (size_t k = blockIdx.x * static_cast<size_t>(kThreads) + threadIdx.x; k < total; k += static_cast<size_t>(gridDim.x) * kThreads) {
        const int i = static_cast<int>(k / per);
        const size_t r = k - i * per;
        const int oy = static_cast<int>(r / w2), ox = static_cast<int>(r - static_cast<size_t>(oy) * w2);
        const uint32_t* m = masks + words * i;
        unsigned sb = 0, sg = 0, sr = 0;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            const int y = 2 * oy + (d >> 1), x = 2 * ox + (d & 1);
            const size_t p = static_cast<size_t>(y) * W + x;
            const bool dot = (m[p >> 5] >> (p & 31)) & 1u;
            const bool lab = label && static_cast<unsigned>(y - label_y0) < static_cast<unsigned>(label_h) &&
                             label[static_cast<size_t>(y - label_y0) * W + x] != 0;
            if (lab && (label_over || !dot)) sb += 255;
            else if (dot) { sg += 255; sr += 255; }
            else { sb += rgb[3 * p + 2]; sg += rgb[3 * p + 1]; sr += rgb[3 * p]; }
        }
        out[3 * k] = static_cast<uint8_t>((sb + 2) >> 2);
        out[3 * k + 1] = static_cast<uint8_t>((sg + 2) >> 2);
        out[3 * k + 2] = static_cast<uint8_t>((sr + 2) >> 2);
    }
}
}  // namespace

size_t overlay_mask_words(int H, int W) { return (static_cast<size_t>(H) * W + 31) / 32; }

cudaError_t launch_draw_tracks(const uint8_t* frame_rgb, int H, int W, const double* K, const double* poses, int n, const double* pts,
                               const int* offsets, const int* track_set, int max_m, const uint8_t* label, int label_y0, int label_h,
                               int label_over, uint32_t* masks, uint8_t* out_bgr, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const size_t words = overlay_mask_words(H, W);
    cudaError_t e = cudaMemsetAsync(masks, 0, sizeof(uint32_t) * words * n, s);
    if (e != cudaSuccess) return e;
    const dim3 grid((max_m + kThreads - 1) / kThreads, std::min(n, 65535));
    splat_kernel<<<grid, kThreads, 0, s>>>(pts, offsets, track_set, poses, n, K[0], K[1], K[2], K[3], H, W, words, masks);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const size_t total = static_cast<size_t>(H / 2) * (W / 2) * n;
    const int blocks = static_cast<int>(std::min<size_t>((total + kThreads - 1) / kThreads, 132 * 16));
    compose_kernel<<<blocks, kThreads, 0, s>>>(frame_rgb, H, W, masks, words, label, label_y0, label_h, label_over, n, out_bgr);
    return cudaGetLastError();
}

}  // namespace se3tn
