// HBM-bound fp32/fp64 kernels either side of the conv stack: frame crop + depth clip + channel
// normalisation (K0), layout packing, 3x3/s2 max-pool, avg-pool + FC + tanh head (K4), and the
// R^3 x so(3) pose update / label (K6 / K5).  Each replaces numpy/cv2 CPU code in the reference;
// the file:line each follows is cited at the kernel.
#include "aux_kernels.h"
#include "conv_common.h"
#include "bbox.cuh"
#include "launch.h"
#include "ptx.cuh"
#include "storage.cuh"
#include <cfloat>

namespace se3tn {

// =============================================================================================
// K0: crop window + nearest resize + depth offset/clip + (x-mean)/std  -> padded NHWC4
// =============================================================================================
// bbox:   reference Utils.py:302-316 (compute_bbox): 4 corners of an object_width-mm square at the
//         object depth, projected in float64, np.round (half-to-even == rint) to int32.
// crop:   reference Utils.py:320-359 (crop_bbox): window copy with zero padding outside the frame,
//         then cv2.resize(INTER_NEAREST): src = min(floor(dst * (1/(dsize/ssize))), ssize-1).
// depth:  reference data_augmentation.py:134-144: invalid = d<=100 || d>=2000 (raw mm), then
//         float32(double(d) -/+ z*1000), invalid -> 2000.  (numpy>=2 semantics, see oracle header.)
// norm:   reference data_augmentation.py:154-164: (x - mean[c]) / std[c]; float32 arithmetic when
//         mean/std are float32 arrays (what train.py:121-125 saves), float64 otherwise.
// pack:   reference data_augmentation.py:179-189 builds CHW float32; here the result goes straight
//         into the stem conv's zero-padded NHWC4 layout (and optionally to NCHW for the drop-in API).

__device__ __forceinline__ float norm_f32(float x, float m, float s) { return __fdiv_rn(__fsub_rn(x, m), s); }
__device__ __forceinline__ float norm_f64(float x, double m, double s) { return static_cast<float>(__ddiv_rn(__dsub_rn(static_cast<double>(x), m), s)); }

__device__ __forceinline__ float depth_offset(unsigned d, double z1000, bool gl) {
    if (d <= 100u || d >= 2000u) return 2000.f;
    return static_cast<float>(gl ? __dadd_rn(static_cast<double>(d), z1000) : __dsub_rn(static_cast<double>(d), z1000));
}

// One CTA = one quarter (44 rows) of one track's 176x176 window.  Everything that depends only on the pixel VALUE is tabulated once
// per CTA with the same IEEE operations the per-pixel code would use (bit-identical results):
//   * (v - mean) / std of an 8-bit colour value: 6 channels x 256 entries;
//   * the whole depth chain  u16 mm -> clip -> float32(double(d) -+ z*1000) -> (x - mean) / std : a function of d alone for a given
//     track, non-constant only for 100 < d < 2000 -> 2 x 1899 entries (A and B use different statistics);
//   * cv2's nearest-neighbour source index floor(dst * (1 / (176 / size))) for the 176 columns and this CTA's 44 rows.
// The per-pixel work is then byte loads, table look-ups, the bf16 / tf32 packing and two 16-byte stores: ~3x fewer instructions
// than dividing per pixel (ncu, round 2: the kernel was issue-bound at 274 instructions per pixel, DRAM at 7 %).
constexpr int kPreRowsMax = 88;                   // most rows one CTA handles (rows per CTA is a launch parameter: 88, 22 or 11)
constexpr int kDepthLo = 101, kDepthN = 1899;     // valid raw depths 101..1999

// THREADS = 256 (strips of 11 / 22 rows) or 1024 (half an image per CTA: the per-CTA tables are built twice per track instead of eight times)
template <int THREADS>
__global__ void __launch_bounds__(THREADS, THREADS == 256 ? 4 : 1)
preprocess_kernel(PreprocessArgs a, int rows_per_cta)
{
    ptx::grid_dep_launch();
    const int n = blockIdx.y;
    const int row0 = blockIdx.x * rows_per_cta;
    const double* pose = a.poses + n * 16;
    __shared__ float s_lut[6][256];
    __shared__ float s_dlut[2][kDepthN];
    __shared__ float s_dinv[2];                    // normalised value of an invalid depth (2000)
    __shared__ int s_sx[kImg], s_sy[kPreRowsMax];        // int: a window may be up to 2e9 px wide (bbox_window), far past 16 bits
    __shared__ int s_win[4];
    const int wi = a.weight_ids ? min(max(a.weight_ids[n], 0), a.stats_rows - 1) : 0;   // ids without statistics are rejected on the host where it can see them; never index past the table
    if (threadIdx.x < 256) {
        const float v = static_cast<float>(threadIdx.x);
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            const int mc = c < 3 ? c : c + 1;                   // A: mean[0..2], B: mean[4..6]
            s_lut[c][threadIdx.x] = a.stats_f64 ? norm_f64(v, a.mean64[wi * 8 + mc], a.std64[wi * 8 + mc])
                                                : norm_f32(v, a.mean32[wi * 8 + mc], a.std32[wi * 8 + mc]);
        }
    }
    ptx::grid_dep_wait();                                       // poses come from the previous step's pose update
    const double z = pose[11];
    const bool gl = z < 0;
    const double z1000 = __dmul_rn(z, 1000.0);
    for (int i = threadIdx.x; i < 2 * kDepthN + 2; i += blockDim.x) {
        const int which = i >= kDepthN + 1;                     // 0: A statistics (channel 3), 1: B statistics (channel 7)
        const int j = which ? i - (kDepthN + 1) : i;            // j == kDepthN: the invalid-depth value
        const float zf = (j == kDepthN) ? 2000.f : depth_offset(static_cast<unsigned>(kDepthLo + j), z1000, gl);
        const int mc = which ? 7 : 3;
        const float r = a.stats_f64 ? norm_f64(zf, a.mean64[wi * 8 + mc], a.std64[wi * 8 + mc]) : norm_f32(zf, a.mean32[wi * 8 + mc], a.std32[wi * 8 + mc]);
        if (j == kDepthN) s_dinv[which] = r; else s_dlut[which][j] = r;
    }
    if (!a.b_precropped) {
        if (threadIdx.x == 0) {
            int top, left, ch, cw;
            bbox_window(pose, a.fx, a.fy, a.cx, a.cy, a.object_width[n], 1000.0, 1000.0, 1000.0, top, left, ch, cw);
            s_win[0] = top; s_win[1] = left; s_win[2] = ch; s_win[3] = cw;
        }
        __syncthreads();
        const int ch = s_win[2], cw = s_win[3];
        // cv2 resizeNN index: floor(dst * ifx), ifx = 1/(dsize/ssize) in double, clamped to ssize-1
        const double ifx = (cw > 0) ? 1.0 / (static_cast<double>(kImg) / cw) : 0.0;
        const double ify = (ch > 0) ? 1.0 / (static_cast<double>(kImg) / ch) : 0.0;
        if (threadIdx.x < kImg) { int sx = static_cast<int>(floor(threadIdx.x * ifx)); if (sx > cw - 1) sx = cw - 1; s_sx[threadIdx.x] = sx; }
        constexpr int kSyFirst = THREADS == 256 ? 192 : 256;     // threads that fill the row table (the column table takes 0..175)
        if (threadIdx.x >= kSyFirst && threadIdx.x < kSyFirst + rows_per_cta) {
            const int y = row0 + threadIdx.x - kSyFirst;
            int sy = static_cast<int>(floor(y * ify)); if (sy > ch - 1) sy = ch - 1; s_sy[threadIdx.x - kSyFirst] = sy;
        }
    }
    __syncthreads();
    const int top = s_win[0], left = s_win[1], ch = s_win[2], cw = s_win[3];
    const size_t img0 = static_cast<size_t>(n) * kImg * kImg;
    auto depth_norm = [&](unsigned d, int which) -> float {
        const unsigned j = d - kDepthLo;
        return j < static_cast<unsigned>(kDepthN) ? s_dlut[which][j] : s_dinv[which];
    };
    // consecutive threads take consecutive pixels: every load / store instruction of a warp touches 32 consecutive pixels
    // (the 16-byte stem stores are 512 contiguous bytes per instruction); four pixels per thread and iteration so that four
    // sets of byte loads are in flight at once (the loop is latency-bound otherwise)
    const int npix = rows_per_cta * kImg;
    for (int lp0 = threadIdx.x; lp0 < npix; lp0 += 4 * blockDim.x) {
        unsigned rA[4], gA[4], bA[4], dA[4], rB[4], gB[4], bB[4], dB[4];
        int pixs[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int lp = lp0 + u * blockDim.x;
            rA[u] = gA[u] = bA[u] = dA[u] = rB[u] = gB[u] = bB[u] = dB[u] = 0; pixs[u] = -1;
            if (lp >= npix) continue;
            const int ly = lp / kImg, x = lp - ly * kImg;
            const int pix = (row0 + ly) * kImg + x;
            pixs[u] = pix;
            const size_t ao = img0 + pix;
            // ---- B: observed frame crop ------------------------------------------------------------------
            if (a.b_precropped) {
                // frame_rgb / frame_depth already hold n 176x176 crops (TrackDataset.processData's inputs)
                const uint8_t* pr = a.frame_rgb + ao * 3;
                rB[u] = pr[0]; gB[u] = pr[1]; bB[u] = pr[2];
                dB[u] = a.frame_depth[ao];
            } else if (ch > 0 && cw > 0) {
                const int fy_ = top + s_sy[ly], fx_ = left + s_sx[x];
                if (fy_ >= 0 && fy_ < a.H && fx_ >= 0 && fx_ < a.W) {
                    const size_t fo = static_cast<size_t>(fy_) * a.W + fx_;
                    const uint8_t* pr = a.frame_rgb + fo * 3;
                    rB[u] = pr[0]; gB[u] = pr[1]; bB[u] = pr[2];
                    dB[u] = a.frame_depth[fo];
                }
            }
            // ---- A: rendered previous view --------------------------------------------------------------
            const uint8_t* pa = a.rgbA + ao * 3;
            rA[u] = pa[0]; gA[u] = pa[1]; bA[u] = pa[2]; dA[u] = a.depthA[ao];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int pix = pixs[u];
            if (pix < 0) continue;
            const int y = pix / kImg, x = pix - y * kImg;
            const size_t ao = img0 + pix;
            if (a.crop_rgb) { uint8_t* o = a.crop_rgb + ao * 3; o[0] = static_cast<uint8_t>(rB[u]); o[1] = static_cast<uint8_t>(gB[u]); o[2] = static_cast<uint8_t>(bB[u]); }
            if (a.crop_depth) a.crop_depth[ao] = static_cast<uint16_t>(dB[u]);
            const float4 vA = make_float4(s_lut[0][rA[u]], s_lut[1][gA[u]], s_lut[2][bA[u]], depth_norm(dA[u], 0));
            const float4 vB = make_float4(s_lut[3][rB[u]], s_lut[4][gB[u]], s_lut[5][bB[u]], depth_norm(dB[u], 1));
            if (a.nchwA) {
                float* oa = a.nchwA + static_cast<size_t>(n) * 4 * kImg * kImg + pix;
                float* ob = a.nchwB + static_cast<size_t>(n) * 4 * kImg * kImg + pix;
                oa[0] = vA.x; oa[kImg * kImg] = vA.y; oa[2 * kImg * kImg] = vA.z; oa[3 * kImg * kImg] = vA.w;
                ob[0] = vB.x; ob[kImg * kImg] = vB.y; ob[2 * kImg * kImg] = vB.z; ob[3 * kImg * kImg] = vB.w;
            }
            if (a.stemA) {
                const size_t so = (static_cast<size_t>(n) * kStemH + (y + 3)) * kStemW + (x + 3);
                reinterpret_cast<float4*>(a.stemA)[so] = encode_stem_pixel(vA, a.precision);
                reinterpret_cast<float4*>(a.stemB)[so] = encode_stem_pixel(vB, a.precision);
            }
        }
    }
}


cudaError_t launch_preprocess(const PreprocessArgs& a, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    // rows per CTA: big strips amortise the per-CTA tables, small ones fill the machine when there are few tracks
    int rows = n >= 64 ? 88 : (n >= 32 ? 22 : 11);
    dim3 grid(kImg / rows, n);
    if (rows == 88) return launch_kernel(preprocess_kernel<1024>, grid, dim3(1024), 0, s, true, a, rows);
    return launch_kernel(preprocess_kernel<256>, grid, dim3(256), 0, s, true, a, rows);
}

// =============================================================================================
// Stand-alone compute_bbox / crop_bbox (reference Utils.py:302-316, 320-359) for the drop-in
// Utils API: the same arithmetic as inside preprocess_kernel, with the bbox made visible.
// =============================================================================================
__global__ void bbox_kernel(const double* __restrict__ poses, double fx, double fy, double cx, double cy,
                            const double* __restrict__ widths, double sx, double sy, double sz,
                            int* __restrict__ out /* (n,4,2) rows (x-,y-),(x-,y+),(x+,y-),(x+,y+), cols (v,u) */, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* pose = poses + i * 16;
    const double ox = __dmul_rn(pose[3], sx), oy = __dmul_rn(pose[7], sy), oz = __dmul_rn(pose[11], sz);
    const double half = widths[i] / 2;
    const double lim = 2.0e9;
    auto proj = [&](double v, double f, double c) {
        const double p = rint(__dadd_rn(__ddiv_rn(__dmul_rn(v, f), oz), c));
        return static_cast<int>(fmax(-lim, fmin(lim, p == p ? p : 0.0)));
    };
    const int u0 = proj(ox - half, fx, cx), u1 = proj(ox + half, fx, cx);
    const int v0 = proj(oy - half, fy, cy), v1 = proj(oy + half, fy, cy);
    int* o = out + i * 8;
    o[0] = v0; o[1] = u0; o[2] = v1; o[3] = u0; o[4] = v0; o[5] = u1; o[6] = v1; o[7] = u1;
}

cudaError_t launch_bbox(const double* poses, const double* K4, const double* widths, const double* scale3,
                        int* out, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    bbox_kernel<<<(n + 127) / 128, 128, 0, s>>>(poses, K4[0], K4[1], K4[2], K4[3], widths, scale3[0], scale3[1], scale3[2], out, n);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
crop_kernel(const uint8_t* __restrict__ frame_rgb, const uint16_t* __restrict__ frame_depth, int H, int W,
            const int* __restrict__ bbox, int out_h, int out_w, uint8_t* __restrict__ crop_rgb, uint16_t* __restrict__ crop_depth)
{
    const int n = blockIdx.y;
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= out_h * out_w) return;
    const int y = pix / out_w, x = pix - y * out_w;
    const int* bb = bbox + n * 8;
    const int top = min(min(bb[0], bb[2]), min(bb[4], bb[6])), bottom = max(max(bb[0], bb[2]), max(bb[4], bb[6]));
    const int left = min(min(bb[1], bb[3]), min(bb[5], bb[7])), right = max(max(bb[1], bb[3]), max(bb[5], bb[7]));
    const int ch = bottom - top, cw = right - left;
    unsigned r = 0, g = 0, b = 0, d = 0;
    if (ch > 0 && cw > 0) {
        const double ifx = 1.0 / (static_cast<double>(out_w) / cw);
        const double ify = 1.0 / (static_cast<double>(out_h) / ch);
        int sx = static_cast<int>(floor(x * ifx)); if (sx > cw - 1) sx = cw - 1;
        int sy = static_cast<int>(floor(y * ify)); if (sy > ch - 1) sy = ch - 1;
        const int fy_ = top + sy, fx_ = left + sx;
        if (fy_ >= 0 && fy_ < H && fx_ >= 0 && fx_ < W) {
            const size_t fo = static_cast<size_t>(fy_) * W + fx_;
            r = frame_rgb[fo * 3]; g = frame_rgb[fo * 3 + 1]; b = frame_rgb[fo * 3 + 2];
            d = frame_depth[fo];
        }
    }
    const size_t o = static_cast<size_t>(n) * out_h * out_w + pix;
    crop_rgb[o * 3] = r; crop_rgb[o * 3 + 1] = g; crop_rgb[o * 3 + 2] = b;
    crop_depth[o] = static_cast<uint16_t>(d);
}

cudaError_t launch_crop(const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const int* bbox, int n,
                        int out_h, int out_w, uint8_t* crop_rgb, uint16_t* crop_depth, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    dim3 grid((out_h * out_w + 255) / 256, n);
    crop_kernel<<<grid, 256, 0, s>>>(frame_rgb, frame_depth, H, W, bbox, out_h, out_w, crop_rgb, crop_depth);
    return cudaGetLastError();
}

// crop_bbox with its segmentation plane (reference Utils.py:320-359 with seg, produce_train_pair_data.py:125-139): rgb and depth
// exactly as crop_kernel cuts them, and the seg plane through the same window and nearest mapping -- zero outside the image,
// never masked (Utils.py:346-349).  One CTA per sample.  class_ids null: crop_seg receives the label values.  class_ids given:
// crop_seg receives (seg == class id) as 0 / 1, what the generator writes to disk, and count[i] the number of such pixels,
// reduced in the CTA (np.sum(segB == class_id), produce_train_pair_data.py:128).
constexpr int kCropSegThreads = 1024;
__global__ void __launch_bounds__(kCropSegThreads)
crop_seg_kernel(const uint8_t* __restrict__ frame_rgb, const uint16_t* __restrict__ frame_depth, const uint8_t* __restrict__ seg,
                int H, int W, const int* __restrict__ bbox, const int* __restrict__ class_ids, int out_h, int out_w,
                uint8_t* __restrict__ crop_rgb, uint16_t* __restrict__ crop_depth, uint8_t* __restrict__ crop_seg, int* __restrict__ count)
{
    ptx::grid_dep_wait();                                   // the bbox comes from bbox_kernel (a step may chain them)
    const int n = blockIdx.x;
    const int* bb = bbox + n * 8;
    const int top = min(min(bb[0], bb[2]), min(bb[4], bb[6])), bottom = max(max(bb[0], bb[2]), max(bb[4], bb[6]));
    const int left = min(min(bb[1], bb[3]), min(bb[5], bb[7])), right = max(max(bb[1], bb[3]), max(bb[5], bb[7]));
    const int ch = bottom - top, cw = right - left;
    const int cid = class_ids ? class_ids[n] : 0;
    const double ifx = cw > 0 ? 1.0 / (static_cast<double>(out_w) / cw) : 0.0;
    const double ify = ch > 0 ? 1.0 / (static_cast<double>(out_h) / ch) : 0.0;
    int hits = 0;
    for (int pix = threadIdx.x; pix < out_h * out_w; pix += blockDim.x) {
        const int y = pix / out_w, x = pix - y * out_w;
        unsigned r = 0, g = 0, b = 0, d = 0, sv = 0;
        if (ch > 0 && cw > 0) {
            int sx = static_cast<int>(floor(x * ifx)); if (sx > cw - 1) sx = cw - 1;
            int sy = static_cast<int>(floor(y * ify)); if (sy > ch - 1) sy = ch - 1;
            const int fy_ = top + sy, fx_ = left + sx;
            if (fy_ >= 0 && fy_ < H && fx_ >= 0 && fx_ < W) {
                const size_t fo = static_cast<size_t>(fy_) * W + fx_;
                r = frame_rgb[fo * 3]; g = frame_rgb[fo * 3 + 1]; b = frame_rgb[fo * 3 + 2];
                d = frame_depth[fo]; sv = seg[fo];
            }
        }
        if (class_ids) {                                    // zero outside the image compares as label 0, as in the reference
            sv = static_cast<int>(sv) == cid ? 1u : 0u;
            hits += static_cast<int>(sv);
        }
        const size_t o = static_cast<size_t>(n) * out_h * out_w + pix;
        crop_rgb[o * 3] = r; crop_rgb[o * 3 + 1] = g; crop_rgb[o * 3 + 2] = b;
        crop_depth[o] = static_cast<uint16_t>(d);
        crop_seg[o] = static_cast<uint8_t>(sv);
    }
    if (!count) return;
    __shared__ int s_hits[kCropSegThreads / 32];
    for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    if ((threadIdx.x & 31) == 0) s_hits[threadIdx.x >> 5] = hits;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kCropSegThreads / 32; ++w) t += s_hits[w];
        count[n] = t;
    }
}

cudaError_t launch_crop_seg(const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W, const int* bbox,
                            const int* class_ids, int n, int out_h, int out_w, uint8_t* crop_rgb, uint16_t* crop_depth,
                            uint8_t* crop_seg, int* count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    return launch_kernel(crop_seg_kernel, dim3(n), dim3(kCropSegThreads), 0, s, false, frame_rgb, frame_depth, seg, H, W, bbox,
                         class_ids, out_h, out_w, crop_rgb, crop_depth, crop_seg, count);
}

// =============================================================================================
// se3tn_append_pairs: the kept rows of a pair step to the tails of their validation queues
// =============================================================================================
// Grid (kAppendSlices, n): CTA (x, i) copies slice x of row i's four planes (five with a.segB) in 16-byte words (consecutive
// threads, consecutive words) and, in slice 0, its two poses.  Row i's slot is its queue's tail plus the kept rows of that queue
// before it, counted by the whole CTA.  Every CTA reads the tail before it counts itself done on a.done; the CTA that counts last
// has seen every other one read, so it alone adds each queue's kept rows to its tail, then clears the counter for the next launch.
constexpr int kAppendThreads = 256, kAppendSlices = 8;
constexpr int kRgbWords = kImg * kImg * 3 / 16, kDepthWords = kImg * kImg * 2 / 16, kSegWords = kImg * kImg / 16, kPoseWords = 16 * 8 / 16;
static_assert(kImg * kImg % 16 == 0, "a crop plane is a whole number of 16-byte words");

__device__ __forceinline__ void copy_words(const void* src, void* dst, int words) {
    const uint4* s = static_cast<const uint4*>(src);
    uint4* d = static_cast<uint4*>(dst);
    for (int v = blockIdx.x * kAppendThreads + threadIdx.x; v < words; v += kAppendSlices * kAppendThreads) d[v] = __ldg(s + v);
}

__global__ void __launch_bounds__(kAppendThreads) append_pairs_kernel(const AppendArgs a)
{
    const int i = blockIdx.y;
    const int q = a.queue_ids[i];
    int before = 0;
    for (int j0 = 0; j0 < i; j0 += kAppendThreads) {
        const int j = j0 + threadIdx.x;
        before += __syncthreads_count(j < i && a.queue_ids[j] == q && a.count[j] >= a.min_count);
    }
    __shared__ int s_tail;
    __shared__ bool s_last;
    if (threadIdx.x == 0) s_tail = a.tails[q];
    __syncthreads();
    const int slot = s_tail + before;
    if (a.count[i] >= a.min_count && slot < a.cap) {
        const size_t src = static_cast<size_t>(i), dst = static_cast<size_t>(q) * a.cap + slot;
        copy_words(a.rgbA + src * kRgbWords * 16, a.q_rgbA + dst * kRgbWords * 16, kRgbWords);
        copy_words(a.rgbB + src * kRgbWords * 16, a.q_rgbB + dst * kRgbWords * 16, kRgbWords);
        copy_words(a.depthA + src * kDepthWords * 8, a.q_depthA + dst * kDepthWords * 8, kDepthWords);
        copy_words(a.depthB + src * kDepthWords * 8, a.q_depthB + dst * kDepthWords * 8, kDepthWords);
        if (a.segB) copy_words(a.segB + src * kSegWords * 16, a.q_segB + dst * kSegWords * 16, kSegWords);
        if (blockIdx.x == 0 && threadIdx.x < 2 * kPoseWords) {
            const bool b = threadIdx.x >= kPoseWords;
            const int w = threadIdx.x - (b ? kPoseWords : 0);
            const uint4* s = reinterpret_cast<const uint4*>((b ? a.B_in_cam : a.A_in_cam) + src * 16);
            reinterpret_cast<uint4*>((b ? a.q_B : a.q_A) + dst * 16)[w] = __ldg(s + w);
        }
    }
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(a.done, 1u) == gridDim.x * gridDim.y - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int r = threadIdx.x; r < a.num_queues; r += kAppendThreads) {
        int kept = 0;
        for (int j = 0; j < a.n; ++j) kept += a.queue_ids[j] == r && a.count[j] >= a.min_count;
        if (kept) a.tails[r] += kept;
    }
    if (threadIdx.x == 0) *a.done = 0u;
}

cudaError_t launch_append_pairs(const AppendArgs& a, cudaStream_t s) {
    if (a.n <= 0) return cudaSuccess;
    append_pairs_kernel<<<dim3(kAppendSlices, a.n), kAppendThreads, 0, s>>>(a);
    return cudaGetLastError();
}

// =============================================================================================
// NCHW float32 (N,4,176,176) -> zero-padded NHWC4 stem input (for Se3TrackNet.forward(A, B))
// =============================================================================================
__global__ void __launch_bounds__(256)
nchw_to_stem_kernel(const float* __restrict__ src, float* __restrict__ dst, int precision)
{
    const int n = blockIdx.y;
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= kImg * kImg) return;
    const int y = pix / kImg, x = pix - y * kImg;
    const float* s = src + static_cast<size_t>(n) * 4 * kImg * kImg + pix;
    float4 v = make_float4(s[0], s[kImg * kImg], s[2 * kImg * kImg], s[3 * kImg * kImg]);
    v = encode_stem_pixel(v, precision);
    reinterpret_cast<float4*>(dst)[(static_cast<size_t>(n) * kStemH + (y + 3)) * kStemW + (x + 3)] = v;
}

cudaError_t launch_nchw_to_stem(const float* src, float* dst, int n, int precision, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    dim3 grid((kImg * kImg + 255) / 256, n);
    nchw_to_stem_kernel<<<grid, 256, 0, s>>>(src, dst, precision);
    return cudaGetLastError();
}

// =============================================================================================
// MaxPool2d(3, 2, 1) on NHWC (reference se3_tracknet.py:58,62,85,89).  Padding behaves as -inf
// (the SELU output it follows can be negative).
// =============================================================================================
__global__ void __launch_bounds__(256)
maxpool_kernel(const float4* __restrict__ in, float4* __restrict__ out, int n_img, int Hin, int Win, int C4)
{
    const int Ho = Hin / 2, Wo = Win / 2;
    const long long total = static_cast<long long>(n_img) * Ho * Wo * C4;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = static_cast<int>(i % C4);
    long long r = i / C4;
    const int ox = static_cast<int>(r % Wo); r /= Wo;
    const int oy = static_cast<int>(r % Ho);
    const int n = static_cast<int>(r / Ho);
    float4 m = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
        const int y = 2 * oy + dy;
        if (y < 0 || y >= Hin) continue;
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int x = 2 * ox + dx;
            if (x < 0 || x >= Win) continue;
            const float4 v = __ldg(&in[((static_cast<size_t>(n) * Hin + y) * Win + x) * C4 + c]);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    out[i] = m;
}

cudaError_t launch_maxpool(const float* in, float* out, int n_img, int Hin, int Win, int C, cudaStream_t s) {
    const long long total = static_cast<long long>(n_img) * (Hin / 2) * (Win / 2) * (C / 4);
    if (total <= 0) return cudaSuccess;
    maxpool_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), n_img, Hin, Win, C / 4);
    return cudaGetLastError();
}

// =============================================================================================
// K4 head of the fp32 FFMA mode: AdaptiveAvgPool2d(1) + Linear(512,3) + Tanh for both heads
// (reference se3_tracknet.py:100-102, 107-109).  x: fp32 NHWC (N, 11*11, 1024): channels [0,512) are
// the translation head, [512,1024) the rotation head.
// =============================================================================================
__global__ void __launch_bounds__(512)
head_kernel(const float4* __restrict__ x, const float* __restrict__ fcw /*[6][512]*/, const float* __restrict__ fcb /*[6]*/,
            float* __restrict__ out_trans, float* __restrict__ out_rot, int npix)
{
    // grid (n, 2): blockIdx.y = head (0 trans: channels 0..511, 1 rot: 512..1023).  512 threads =
    // 4 pixel groups x 128 threads, each thread 4 channels.
    ptx::grid_dep_launch();
    __shared__ float4 part4[4][128];
    __shared__ float red[4][3];
    const int n = blockIdx.x, head = blockIdx.y, t = threadIdx.x;
    const int cq = t & 127, pg = t >> 7;
    const int c = head * 512 + cq * 4;                 // first of this thread's 4 channels
    ptx::grid_dep_wait();
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* xp = x + static_cast<size_t>(n) * npix * 256 + (c >> 2);
    for (int p = pg; p < npix; p += 4) {
        const float4 v = __ldg(xp + static_cast<size_t>(p) * 256);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    part4[pg][cq] = s;
    __syncthreads();
    if (t < 128) {
        const float4 a0 = part4[0][t], a1 = part4[1][t], a2 = part4[2][t], a3 = part4[3][t];
        const float inv = 1.0f / static_cast<float>(npix);
        const float mx = ((a0.x + a1.x) + (a2.x + a3.x)) * inv, my = ((a0.y + a1.y) + (a2.y + a3.y)) * inv;
        const float mz = ((a0.z + a1.z) + (a2.z + a3.z)) * inv, mw = ((a0.w + a1.w) + (a2.w + a3.w)) * inv;
        float part[3];
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(fcw + (head * 3 + o) * 512 + t * 4));
            part[o] = mx * w.x + my * w.y + mz * w.z + mw * w.w;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1)
#pragma unroll
            for (int o = 0; o < 3; ++o) part[o] += __shfl_xor_sync(0xffffffffu, part[o], off);
        if ((t & 31) == 0) { red[t >> 5][0] = part[0]; red[t >> 5][1] = part[1]; red[t >> 5][2] = part[2]; }
    }
    __syncthreads();
    if (t < 3) {
        const float v = red[0][t] + red[1][t] + red[2][t] + red[3][t] + fcb[head * 3 + t];
        (head == 0 ? out_trans : out_rot)[n * 3 + t] = tanhf(v);
    }
}

// =============================================================================================
// K6 pose update (reference datasets.py:159-175): t' = t + float32(trans*tn);
// R' = float32(Rodrigues(float32(rot*rn))) . R, all remaining arithmetic in float64 (F9/F10).
// Rodrigues follows OpenCV's cvRodrigues2 vector->matrix branch:
//   theta = |r|; theta < DBL_EPSILON -> I; else R = cos*I + (1-cos)*rr^T + sin*[r]x, r <- r/theta.
// =============================================================================================
__device__ __forceinline__ void rodrigues_exp_f32in(float rx32, float ry32, float rz32, double R[9], bool round_f32)
{
    double rx = rx32, ry = ry32, rz = rz32;
    const double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < DBL_EPSILON) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1.0 - c, it = 1.0 / theta;
    rx *= it; ry *= it; rz *= it;
    // same association as cv::Matx: c*I + c1*(r r^T) + s*[r]x, outer products formed first
    const double xx = rx * rx, xy = rx * ry, xz = rx * rz, yy = ry * ry, yz = ry * rz, zz = rz * rz;
    R[0] = c + c1 * xx;      R[1] = c1 * xy - s * rz; R[2] = c1 * xz + s * ry;
    R[3] = c1 * xy + s * rz; R[4] = c + c1 * yy;      R[5] = c1 * yz - s * rx;
    R[6] = c1 * xz - s * ry; R[7] = c1 * yz + s * rx; R[8] = c + c1 * zz;
    if (round_f32)
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = static_cast<double>(static_cast<float>(R[i]));
}

// one track: A (row-major 4x4) and the network's 3+3 output -> B
__device__ __forceinline__ void pose_update_one(const double* A, const float tr[3], const float ro[3], float tn, float rn,
                                                double* B /* may alias A */)
{
    // float32 * python-float stays float32 in numpy
    const float t0 = __fmul_rn(tr[0], tn), t1 = __fmul_rn(tr[1], tn), t2 = __fmul_rn(tr[2], tn);
    const float r0 = __fmul_rn(ro[0], rn), r1 = __fmul_rn(ro[1], rn), r2 = __fmul_rn(ro[2], rn);
    double R[9];
    rodrigues_exp_f32in(r0, r1, r2, R, true);
    double out[16];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            out[r * 4 + c] = __dadd_rn(__dadd_rn(__dmul_rn(R[r * 3 + 0], A[0 * 4 + c]), __dmul_rn(R[r * 3 + 1], A[1 * 4 + c])),
                                       __dmul_rn(R[r * 3 + 2], A[2 * 4 + c]));
    out[3] = static_cast<double>(t0) + A[3];
    out[7] = static_cast<double>(t1) + A[7];
    out[11] = static_cast<double>(t2) + A[11];
    out[12] = 0; out[13] = 0; out[14] = 0; out[15] = 1;        // B_in_cam starts as np.eye(4)
#pragma unroll
    for (int k = 0; k < 16; ++k) B[k] = out[k];
}

// K5 label of one pair (defined with so3_log_kernel below); the outputs may be global or shared memory
__device__ __noinline__ void so3_label(const double* A, const double* B, double tn, double rn, double* trans_label, double* rot_label);

// One squared error of the reference's loss: nn.MSELoss on pred.float() and target.float() (se3_tracknet.py:114-121) forms
// (pred - float32(label))^2 in fp32 before it averages.
__device__ __forceinline__ float loss_term(float pred, double label) {
    const float d = __fsub_rn(pred, __double2float_rn(label));
    return __fmul_rn(d, d);
}

// Head on the fused average pool (conv_wgmma.cu writes pool_part[image][kPoolSlices][1024] column sums): mean -> Linear -> tanh for
// BOTH heads of one image per CTA (threads 0-127 translation, 128-255 rotation), and -- when poses_in is given -- the pose update of that
// track by thread 0 (K4 + K6 in one launch: the update is a 650-instruction fp64 chain per track, pure latency as its own kernel).
// loss.poses_a given: the pair's label (thread 0, alongside the others' FC work) and its six loss terms (LossArgs).
// `zero_words` (nullable): scheduler / dependency counters of the step that just finished, cleared for the next one by block 0.
__global__ void __launch_bounds__(256)
head_pooled_kernel(const float4* __restrict__ part, const float* __restrict__ fcw, const float* __restrict__ fcb,
                   float* __restrict__ out_trans, float* __restrict__ out_rot, int npix,
                   const int* __restrict__ img_wid, const float* const* __restrict__ fc_table,
                   const double* poses_in, double* poses_out /* may alias */, float tn, float rn, LossArgs loss,
                   unsigned* __restrict__ zero_words, int n_zero)
{
    ptx::grid_dep_launch();
    __shared__ float red[8][3];
    __shared__ float six[6];
    __shared__ double label[6];
    const int n = blockIdx.x, head = threadIdx.x >> 7, t = threadIdx.x & 127;
    ptx::grid_dep_wait();
    if (zero_words && blockIdx.x == 0) for (int i = threadIdx.x; i < n_zero; i += blockDim.x) zero_words[i] = 0u;
    if (loss.poses_a && threadIdx.x == 0) so3_label(loss.poses_a + n * 16, loss.poses_b + n * 16, loss.tn, loss.rn, label, label + 3);
    if (img_wid) { fcw = fc_table[img_wid[n]]; fcb = fcw + 6 * 512; }
    static_assert(se3tn::kPoolSlices == 8, "pairwise sum below");
    const float4* pp = part + static_cast<size_t>(n) * se3tn::kPoolSlices * 256 + head * 128 + t;
    float4 a[se3tn::kPoolSlices];
#pragma unroll
    for (int i = 0; i < se3tn::kPoolSlices; ++i) a[i] = pp[i * 256];
    const float inv = 1.0f / static_cast<float>(npix);
    auto sum8 = [&](float a0, float a1, float a2, float a3, float a4, float a5, float a6, float a7) {
        return (((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7))) * inv;
    };
    const float mx = sum8(a[0].x, a[1].x, a[2].x, a[3].x, a[4].x, a[5].x, a[6].x, a[7].x);
    const float my = sum8(a[0].y, a[1].y, a[2].y, a[3].y, a[4].y, a[5].y, a[6].y, a[7].y);
    const float mz = sum8(a[0].z, a[1].z, a[2].z, a[3].z, a[4].z, a[5].z, a[6].z, a[7].z);
    const float mw = sum8(a[0].w, a[1].w, a[2].w, a[3].w, a[4].w, a[5].w, a[6].w, a[7].w);
    float acc[3];
#pragma unroll
    for (int o = 0; o < 3; ++o) {
        const float4 w = __ldg(reinterpret_cast<const float4*>(fcw + (head * 3 + o) * 512 + t * 4));
        acc[o] = mx * w.x + my * w.y + mz * w.z + mw * w.w;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int o = 0; o < 3; ++o) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], off);
    if ((t & 31) == 0) { red[threadIdx.x >> 5][0] = acc[0]; red[threadIdx.x >> 5][1] = acc[1]; red[threadIdx.x >> 5][2] = acc[2]; }
    __syncthreads();
    if (threadIdx.x < 6) {
        const int h = threadIdx.x / 3, o = threadIdx.x - 3 * h;
        const float v = tanhf(red[4 * h + 0][o] + red[4 * h + 1][o] + red[4 * h + 2][o] + red[4 * h + 3][o] + fcb[h * 3 + o]);
        (h == 0 ? out_trans : out_rot)[n * 3 + o] = v;
        six[threadIdx.x] = v;
        if (loss.poses_a) {                                      // label[] was written by thread 0 before the barrier above
            loss.sq[n * 6 + threadIdx.x] = loss_term(v, label[threadIdx.x]);
            if (loss.labels) loss.labels[n * 6 + threadIdx.x] = label[threadIdx.x];
        }
    }
    if (!poses_in) return;
    __syncthreads();
    if (threadIdx.x == 0) pose_update_one(poses_in + n * 16, six, six + 3, tn, rn, poses_out + n * 16);
}
cudaError_t launch_head_pooled(const float* part, const float* fcw, const float* fcb, float* out_trans, float* out_rot,
                               int n_img, int npix, const int* img_wid, const float* const* fc_table,
                               const double* poses_in, double* poses_out, float tn, float rn, const LossArgs& loss,
                               unsigned* zero_words, int n_zero, cudaStream_t s) {
    if (n_img <= 0) return cudaSuccess;
    if (loss.poses_a && (!loss.poses_b || !loss.sq)) return cudaErrorInvalidValue;
    const float4* p4 = reinterpret_cast<const float4*>(part);
    return launch_kernel(head_pooled_kernel, dim3(n_img), dim3(256), 0, s, true, p4, fcw, fcb, out_trans, out_rot, npix, img_wid, fc_table,
                         poses_in, poses_out, tn, rn, loss, zero_words, n_zero);
}

// =============================================================================================
// The reduction of the loss terms (reference se3_tracknet.py:114-121: one nn.MSELoss per head).  Thread t adds the terms of pairs
// t, t + 256, ... in index order, each pair's three as (x + y) + z, and a shared-memory tree adds the 256 partial sums: the order
// depends on n alone, never on scheduling.  Both launches below use it, so the validation step and se3tn_pair_loss agree bit for
// bit on equal terms.
// =============================================================================================
constexpr int kLossThreads = 256;

template <class Terms>   // terms(i, float t[6]) yields pair i's six terms
__device__ __forceinline__ void reduce_loss_terms(int n, Terms terms, float* sums)
{
    __shared__ float s_tr[kLossThreads], s_ro[kLossThreads];
    float a = 0.f, b = 0.f;
    for (int i = threadIdx.x; i < n; i += kLossThreads) {
        float q[6];
        terms(i, q);
        a = __fadd_rn(a, __fadd_rn(__fadd_rn(q[0], q[1]), q[2]));
        b = __fadd_rn(b, __fadd_rn(__fadd_rn(q[3], q[4]), q[5]));
    }
    s_tr[threadIdx.x] = a; s_ro[threadIdx.x] = b;
    __syncthreads();
#pragma unroll
    for (int w = kLossThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) {
            s_tr[threadIdx.x] = __fadd_rn(s_tr[threadIdx.x], s_tr[threadIdx.x + w]);
            s_ro[threadIdx.x] = __fadd_rn(s_ro[threadIdx.x], s_ro[threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { sums[0] = s_tr[0]; sums[1] = s_ro[0]; }
}

__global__ void __launch_bounds__(kLossThreads) loss_reduce_kernel(const float* __restrict__ sq, int n, float* __restrict__ sums)
{
    reduce_loss_terms(n, [&](int i, float q[6]) {
#pragma unroll
        for (int k = 0; k < 6; ++k) q[k] = sq[i * 6 + k];
    }, sums);
}

cudaError_t launch_loss_reduce(const float* sq, int n, float* sums, cudaStream_t s) {
    if (n <= 0) return cudaErrorInvalidValue;
    loss_reduce_kernel<<<1, kLossThreads, 0, s>>>(sq, n, sums);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(kLossThreads)
pair_loss_kernel(const float* __restrict__ trans, const float* __restrict__ rot, const double* __restrict__ trans_label,
                 const double* __restrict__ rot_label, LossArgs loss, int n, float* __restrict__ sums)
{
    reduce_loss_terms(n, [&](int i, float q[6]) {
        double lab[6];
        if (trans_label) {
#pragma unroll
            for (int k = 0; k < 3; ++k) { lab[k] = trans_label[i * 3 + k]; lab[3 + k] = rot_label[i * 3 + k]; }
        } else {
            so3_label(loss.poses_a + i * 16, loss.poses_b + i * 16, loss.tn, loss.rn, lab, lab + 3);
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            q[k] = loss_term(k < 3 ? trans[i * 3 + k] : rot[i * 3 + k - 3], lab[k]);
            if (loss.sq) loss.sq[i * 6 + k] = q[k];
            if (loss.labels) loss.labels[i * 6 + k] = lab[k];
        }
    }, sums);
}

cudaError_t launch_pair_loss(const float* trans, const float* rot, const double* trans_label, const double* rot_label,
                             const LossArgs& loss, int n, float* sums, cudaStream_t s) {
    if (n <= 0 || !trans || !rot || !sums || (!trans_label != !rot_label) || (!trans_label && (!loss.poses_a || !loss.poses_b)))
        return cudaErrorInvalidValue;
    pair_loss_kernel<<<1, kLossThreads, 0, s>>>(trans, rot, trans_label, rot_label, loss, n, sums);
    return cudaGetLastError();
}

cudaError_t launch_head(const float* x, const float* fcw, const float* fcb, float* out_trans, float* out_rot,
                        int n_img, int npix, cudaStream_t s) {
    if (n_img <= 0) return cudaSuccess;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    return launch_kernel(head_kernel, dim3(n_img, 2), dim3(512), 0, s, true, x4, fcw, fcb, out_trans, out_rot, npix);
}

// =============================================================================================
// NHWC -> NCHW (the 'feature' entry of the reference's output dict, se3_tracknet.py:96)
// =============================================================================================
// in: the storage format of PREC (storage.cuh), C % 4 == 0.  One CTA transposes 32 pixels x 32 channels.
template <int PREC>
__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int HW, int C, const float* __restrict__ fp8_scale)
{
    using R = Raw<PREC, 4>;
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    {
        const int j = threadIdx.x >> 3, g = threadIdx.x & 7;    // pixel p0 + j, channels c0 + 4g .. + 3
        const int p = p0 + j, c = c0 + 4 * g;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (p < HW && c < C) {
            const uint8_t* src = in + Storage<PREC>::addr(static_cast<size_t>(n) * HW + p, C, c);
            R r;
#pragma unroll
            for (int q = 0; q < R::kPieces; ++q) r.set(q, *R::at(src, q));
            Storage<PREC>::decode(r, v);
            if constexpr (PREC == SE3TN_PREC_FP8) {
                const float sc = *fp8_scale;           // a power of two: exact
#pragma unroll
                for (int e = 0; e < 4; ++e) v[e] *= sc;
            }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) tile[j][4 * g + e] = v[e];
    }
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;    // 32 x 8
    for (int j = ty; j < 32; j += 8) {
        const int c = c0 + j, p = p0 + tx;
        if (p < HW && c < C) out[(static_cast<size_t>(n) * C + c) * HW + p] = tile[tx][j];
    }
}

cudaError_t launch_nhwc_to_nchw(const void* in, float* out, int n_img, int HW, int C, int precision, cudaStream_t s,
                                const float* fp8_scale) {
    if (n_img <= 0) return cudaSuccess;
    if (C % 4) return cudaErrorInvalidValue;
    dim3 grid((HW + 31) / 32, (C + 31) / 32, n_img);
    const uint8_t* src = static_cast<const uint8_t*>(in);
    switch (precision) {
        case SE3TN_PREC_FP32:            // plain fp32 words decode like tf32 ones
        case SE3TN_PREC_TF32:   nhwc_to_nchw_kernel<SE3TN_PREC_TF32><<<grid, 256, 0, s>>>(src, out, HW, C, nullptr); break;
        case SE3TN_PREC_BF16X3: nhwc_to_nchw_kernel<SE3TN_PREC_BF16X3><<<grid, 256, 0, s>>>(src, out, HW, C, nullptr); break;
        case SE3TN_PREC_BF16:   nhwc_to_nchw_kernel<SE3TN_PREC_BF16><<<grid, 256, 0, s>>>(src, out, HW, C, nullptr); break;
        case SE3TN_PREC_FP16:   nhwc_to_nchw_kernel<SE3TN_PREC_FP16><<<grid, 256, 0, s>>>(src, out, HW, C, nullptr); break;
        case SE3TN_PREC_FP8:
            if (!fp8_scale) return cudaErrorInvalidValue;
            nhwc_to_nchw_kernel<SE3TN_PREC_FP8><<<grid, 256, 0, s>>>(src, out, HW, C, fp8_scale); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// =============================================================================================
// Weight preparation for the tensor-core modes (conv_wgmma.cu): the fp32 K-major matrices in the storage formats of
// storage.cuh, a weight row being a "pixel" of ktot channels.
// =============================================================================================
template <int PREC>
__global__ void encode_weights_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, int rows, int ktot)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // one thread per 4 K words of a row
    if (i >= rows * (ktot / 4)) return;
    const int row = i / (ktot / 4), k = (i - row * (ktot / 4)) * 4;
    const float* w = src + static_cast<size_t>(row) * ktot + k;
    const float v[4] = {w[0], w[1], w[2], w[3]};
    Storage<PREC>::encode(v).store(dst + Storage<PREC>::addr(row, ktot, k));
}
cudaError_t launch_encode_weights(int precision, const float* src, void* dst, int rows, int ktot, cudaStream_t s) {
    if (rows <= 0 || ktot <= 0 || ktot % 32) return cudaErrorInvalidValue;
    const int blocks = (rows * (ktot / 4) + 255) / 256;
    uint8_t* d = static_cast<uint8_t*>(dst);
    switch (precision) {
        case SE3TN_PREC_TF32:   encode_weights_kernel<SE3TN_PREC_TF32><<<blocks, 256, 0, s>>>(src, d, rows, ktot); break;
        case SE3TN_PREC_BF16X3: encode_weights_kernel<SE3TN_PREC_BF16X3><<<blocks, 256, 0, s>>>(src, d, rows, ktot); break;
        case SE3TN_PREC_BF16:   encode_weights_kernel<SE3TN_PREC_BF16><<<blocks, 256, 0, s>>>(src, d, rows, ktot); break;
        case SE3TN_PREC_FP16:   encode_weights_kernel<SE3TN_PREC_FP16><<<blocks, 256, 0, s>>>(src, d, rows, ktot); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// SE3TN_PREC_FP8 weights: one CTA per row.  s_w = 2^ceil(log2(max|w| / 448)) (pow2_scale), codes e4m3(w / s_w).
__device__ __forceinline__ float pow2_scale_dev(float amax) {
    if (!(amax > 0.f)) return 1.f;
    int ex;
    const float m = frexpf(amax, &ex);            // amax = m 2^ex, m in [0.5, 1); 448 = 0.875 2^9
    return ldexpf(1.f, ex - 9 + (m > 0.875f ? 1 : 0));
}
__global__ void __launch_bounds__(256)
encode_weights_fp8_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, float* __restrict__ row_scale, int ktot)
{
    __shared__ float red[8];
    const int row = blockIdx.x;
    const float* w = src + static_cast<size_t>(row) * ktot;
    float m = 0.f;
    for (int k = threadIdx.x; k < ktot; k += 256) m = fmaxf(m, fabsf(w[k]));
#pragma unroll
    for (int off = 16; off; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    const float sw = pow2_scale_dev(m), inv = 1.f / sw;
    if (threadIdx.x == 0) row_scale[row] = sw;
    using S = Storage<SE3TN_PREC_FP8>;
    for (int k = 4 * threadIdx.x; k < ktot; k += 4 * 256) {
        const float v[4] = {w[k] * inv, w[k + 1] * inv, w[k + 2] * inv, w[k + 3] * inv};
        S::encode(v).store(dst + S::addr(row, ktot, k));
    }
}
cudaError_t launch_encode_weights_fp8(const float* src, void* dst, float* row_scale, int rows, int ktot, cudaStream_t s) {
    if (rows <= 0 || ktot <= 0 || ktot % 128) return cudaErrorInvalidValue;
    encode_weights_fp8_kernel<<<rows, 256, 0, s>>>(src, static_cast<uint8_t*>(dst), row_scale, ktot);
    return cudaGetLastError();
}

// max|x| of bf16x3 tensors as stored: one grid row per tensor, atomicMax on the fp32 bits (non-negative floats order as
// their bits; NaN's bits exceed +inf's, so a NaN shows as a non-finite maximum)
__global__ void __launch_bounds__(256) amax_bf16x3_kernel(AmaxArgs a, unsigned* __restrict__ amax_bits)
{
    const AmaxArgs::Tensor t = a.t[blockIdx.y];
    const int groups = t.nc / 4;
    const size_t total = static_cast<size_t>(a.n) * t.pixels * groups;
    using S = Storage<SE3TN_PREC_BF16X3>;
    using R = Raw<SE3TN_PREC_BF16X3, 4>;
    float m = 0.f;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t pix = i / groups;
        const int c = t.c0 + 4 * static_cast<int>(i - pix * groups);
        const uint8_t* p = t.buf + S::addr(pix, t.C, c);
        R r;
#pragma unroll
        for (int q = 0; q < R::kPieces; ++q) r.set(q, *R::at(p, q));
        float v[4];
        S::decode(r, v);
#pragma unroll
        for (int e = 0; e < 4; ++e) m = (fabsf(v[e]) > m || v[e] != v[e]) ? fabsf(v[e]) : m;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, m, off);
        m = (o > m || o != o) ? o : m;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(amax_bits + blockIdx.y, __float_as_uint(m));
}
cudaError_t launch_amax_bf16x3(const AmaxArgs& a, unsigned* amax_bits, cudaStream_t s) {
    if (a.n_tensors <= 0 || a.n_tensors > AmaxArgs::kMax || a.n <= 0) return cudaErrorInvalidValue;
    for (int i = 0; i < a.n_tensors; ++i) if (a.t[i].nc % 4 || a.t[i].c0 % 4) return cudaErrorInvalidValue;
    amax_bf16x3_kernel<<<dim3(132, a.n_tensors), 256, 0, s>>>(a, amax_bits);
    return cudaGetLastError();
}

// STACK layouts for the resident-weight kernels (conv_wgmma.cu): the bf16x3 split as 128 rows, rows 0-63 the hi parts, rows 64-127
// the lo parts, each row plain bf16.
// 64-channel 3x3 layers: src [64][9*64] (K-major, tap*64 + c) -> dst [128][9*32 words]; a tap's 128 bytes = 64 bf16 = both chunks.
__global__ void split_stack_weights_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // one thread per 4 K words of a row
    if (i >= 64 * 144) return;
    const int co = i / 144, k = (i - co * 144) * 4;
    const float* w = src + co * 576 + k;
    const float v[4] = {w[0], w[1], w[2], w[3]};
    const auto x = Storage<SE3TN_PREC_BF16X3>::encode(v);
    using B = Storage<SE3TN_PREC_BF16>;
    *reinterpret_cast<uint2*>(dst + B::addr(co, 576, k)) = x.get(0);
    *reinterpret_cast<uint2*>(dst + B::addr(64 + co, 576, k)) = x.get(1);
}
// stem: src [64][7*32] -> dst [128][7*32 words]; pixel slot p of filter row r: rows 0-63 [h0..h3 h0..h3], rows 64-127 [l0..l3 0 0 0 0]
// (against the stem input's [4 x hi | 4 x lo] pixels, storage.cuh stem_input_prec)
__global__ void split_stem_stack_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // one thread per (co, r, p): 4 channels
    if (i >= 64 * 7 * 8) return;
    const int p = i & 7, r = (i >> 3) % 7, co = i / 56;
    const float* w = src + co * 224 + r * 32 + p * 4;
    const float v[4] = {w[0], w[1], w[2], w[3]};
    const auto x = Storage<SE3TN_PREC_BF16X3>::encode(v);
    const uint2 h = x.get(0), l = x.get(1);
    *reinterpret_cast<uint4*>(dst + (static_cast<size_t>(co) * 224 + r * 32 + p * 4) * 4) = make_uint4(h.x, h.y, h.x, h.y);
    *reinterpret_cast<uint4*>(dst + (static_cast<size_t>(64 + co) * 224 + r * 32 + p * 4) * 4) = make_uint4(l.x, l.y, 0u, 0u);
}
// Resident 64-channel layers (conv_wgmma.cu, register-fragment epilogue): accumulator column 8j + 2m + e of every 32-column block
// must carry output channel 8m + 2j + e, so the weight ROWS are stored in that order.
__global__ void permute_rows64_kernel(const float* __restrict__ src, float* __restrict__ dst, int ktot)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * ktot) return;
    const int col = i / ktot, k = i - col * ktot;
    const int ch = (col & 32) | (((col >> 1) & 3) << 3) | (((col >> 3) & 3) << 1) | (col & 1);
    dst[i] = src[ch * ktot + k];
}
cudaError_t launch_permute_rows64(const float* src, float* dst, int ktot, cudaStream_t s) {
    permute_rows64_kernel<<<(64 * ktot + 255) / 256, 256, 0, s>>>(src, dst, ktot);
    return cudaGetLastError();
}
cudaError_t launch_split_stack_weights(const float* src, void* dst, bool stem, cudaStream_t s) {
    if (stem) split_stem_stack_kernel<<<(64 * 7 * 8 + 127) / 128, 128, 0, s>>>(src, static_cast<uint8_t*>(dst));
    else split_stack_weights_kernel<<<(64 * 144 + 255) / 256, 256, 0, s>>>(src, static_cast<uint8_t*>(dst));
    return cudaGetLastError();
}

// stand-alone K6 (se3tn_pose_update; the batched path runs it inside head_pooled_kernel)
__global__ void pose_update_kernel(const double* poses_in, const float* __restrict__ trans,
                                   const float* __restrict__ rot, float tn, float rn,
                                   double* poses_out /* may alias poses_in */, int n)
{
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float tr[3] = {trans[i * 3 + 0], trans[i * 3 + 1], trans[i * 3 + 2]};
    const float ro[3] = {rot[i * 3 + 0], rot[i * 3 + 1], rot[i * 3 + 2]};
    pose_update_one(poses_in + i * 16, tr, ro, tn, rn, poses_out + i * 16);
}

cudaError_t launch_pose_update(const double* poses_in, const float* trans, const float* rot, float tn, float rn,
                               double* poses_out, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    return launch_kernel(pose_update_kernel, dim3((n + 31) / 32), dim3(32), 0, s, true, poses_in, trans, rot, tn, rn, poses_out, n);
}

// =============================================================================================
// K5 so(3) log label (reference datasets.py:141-150): trans = (tB - tA)/tn;
// rot = Rodrigues^-1(normalize_cols(R_B R_A^T))/rn  (Utils.py:363-367 + cvRodrigues2 matrix->vector
// branch: R <- U V^T from the SVD, then the antisymmetric-part formula with its small-angle cases).
// The SVD's U V^T is the orthogonal polar factor of R; it is computed here with the Newton
// iteration X <- (X + X^-T)/2, which converges quadratically to the same matrix.
// =============================================================================================
__device__ __forceinline__ void inv_transpose3(const double* m, double* o) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
    const double id = 1.0 / det;
    o[0] = c00 * id; o[1] = c01 * id; o[2] = c02 * id;
    o[3] = (m[2] * m[7] - m[1] * m[8]) * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[1] * m[6] - m[0] * m[7]) * id;
    o[6] = (m[1] * m[5] - m[2] * m[4]) * id; o[7] = (m[2] * m[3] - m[0] * m[5]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// One pair.  so3_log_kernel, the validation head and pair_loss_kernel all call this one (not inlined) function, so their labels are
// the same bits.
__device__ __noinline__ void so3_label(const double* A, const double* B, double tn, double rn, double* trans_label, double* rot_label)
{
    trans_label[0] = (B[3] - A[3]) / tn;
    trans_label[1] = (B[7] - A[7]) / tn;
    trans_label[2] = (B[11] - A[11]) / tn;
    double R[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)     // R_B . R_A^T
            R[r * 3 + c] = B[r * 4 + 0] * A[c * 4 + 0] + B[r * 4 + 1] * A[c * 4 + 1] + B[r * 4 + 2] * A[c * 4 + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) {       // column normalise
        const double nr = sqrt(R[c] * R[c] + R[3 + c] * R[3 + c] + R[6 + c] * R[6 + c]);
        R[c] /= nr; R[3 + c] /= nr; R[6 + c] /= nr;
    }
    for (int it = 0; it < 12; ++it) {   // polar factor
        double T[9]; inv_transpose3(R, T);
        double diff = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) { const double v = 0.5 * (R[k] + T[k]); diff = fmax(diff, fabs(v - R[k])); R[k] = v; }
        if (diff < 1e-16) break;
    }
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : (c < -1. ? -1. : c);
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) { rx = ry = rz = 0; }
        else {
            double t;
            t = (R[0] + 1) * 0.5; rx = sqrt(fmax(t, 0.));
            t = (R[4] + 1) * 0.5; ry = sqrt(fmax(t, 0.)) * (R[1] < 0 ? -1. : 1.);
            t = (R[8] + 1) * 0.5; rz = sqrt(fmax(t, 0.)) * (R[2] < 0 ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((R[5] > 0) != (ry * rz > 0))) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            rx *= theta; ry *= theta; rz *= theta;
        }
    } else {
        const double vth = theta / (2 * s);
        rx *= vth; ry *= vth; rz *= vth;
    }
    rot_label[0] = rx / rn; rot_label[1] = ry / rn; rot_label[2] = rz / rn;
}

__global__ void so3_log_kernel(const double* __restrict__ poses_a, const double* __restrict__ poses_b,
                               double tn, double rn, double* __restrict__ trans_label, double* __restrict__ rot_label, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    so3_label(poses_a + i * 16, poses_b + i * 16, tn, rn, trans_label + i * 3, rot_label + i * 3);
}

cudaError_t launch_so3_log(const double* poses_a, const double* poses_b, double tn, double rn,
                           double* trans_label, double* rot_label, int n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    so3_log_kernel<<<(n + 127) / 128, 128, 0, s>>>(poses_a, poses_b, tn, rn, trans_label, rot_label, n);
    return cudaGetLastError();
}

}  // namespace se3tn
