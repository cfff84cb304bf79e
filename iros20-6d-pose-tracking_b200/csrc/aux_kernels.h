// Launch wrappers for the non-GEMM kernels of the hot path (see aux_kernels.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace se3tn {

constexpr int kImg = 176;                 // crop resolution (reference dataset_info.yml:15)
constexpr int kStemH = kImg + 6;          // 3-pixel zero halo for the 7x7 stem
constexpr int kStemW = kImg + 8;          // 3 left + 176 + 5 right: the stem K-slice reads 8 pixels from x = 2*ox
constexpr size_t kStemImgFloats = static_cast<size_t>(kStemH) * kStemW * 4;

struct PreprocessArgs {
    const uint8_t* frame_rgb;      // H x W x 3
    const uint16_t* frame_depth;   // H x W (mm)
    int H, W;
    double fx, fy, cx, cy;
    const double* poses;           // N x 16 row-major 4x4
    const double* object_width;    // N (mm)
    const uint8_t* rgbA;           // N x 176 x 176 x 3 (renderer output)
    const uint16_t* depthA;        // N x 176 x 176
    const int* weight_ids;         // N or null (all 0): selects the mean/std row
    const float* mean32; const float* std32;      // [sets][8] when !stats_f64
    const double* mean64; const double* std64;    // [sets][8] when stats_f64
    int stats_f64;
    int stats_rows;                // rows of the mean/std tables (weight ids are clamped to it)
    int precision;                 // SE3TN_PREC_*: selects the stem-input format of stemA / stemB (storage.cuh)
    int b_precropped;              // frame_rgb/frame_depth are n ready-made 176x176 crops (processData inputs)
    float* stemA; float* stemB;    // N x 182 x 184 x 4 (nullable)
    float* nchwA; float* nchwB;    // N x 4 x 176 x 176 (nullable)
    uint8_t* crop_rgb;             // N x 176 x 176 x 3 (nullable)
    uint16_t* crop_depth;          // N x 176 x 176 (nullable)
};

// The training loss of a validation step (reference se3_tracknet.py:114-121 on the labels of datasets.py:141-150), fused into
// head_pooled_kernel: poses_a non-null turns it on.  For pair i it forms the label exactly as so3_log_kernel does and the six
// squared errors (pred - float(label))^2 in fp32, trans then rot.
struct LossArgs {
    const double* poses_a = nullptr;   // (n,16) A_in_cam
    const double* poses_b = nullptr;   // (n,16) B_in_cam
    double tn = 0.0, rn = 0.0;         // trans / rot normalizer
    float* sq = nullptr;               // (n,6) squared errors (required when poses_a is set)
    double* labels = nullptr;          // (n,6) labels, nullable
};

cudaError_t launch_preprocess(const PreprocessArgs& a, int n, cudaStream_t s);
cudaError_t launch_bbox(const double* poses, const double* K4, const double* widths, const double* scale3,
                        int* out, int n, cudaStream_t s);
cudaError_t launch_crop(const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const int* bbox, int n,
                        int out_h, int out_w, uint8_t* crop_rgb, uint16_t* crop_depth, cudaStream_t s);
// crop_bbox with the seg plane (uint8 (H,W) labels): class_ids null -> crop_seg holds the labels; class_ids (n) given -> crop_seg
// holds (label == class id) as 0 / 1 and count (n, nullable) the number of ones.  One CTA per sample.
cudaError_t launch_crop_seg(const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W, const int* bbox,
                            const int* class_ids, int n, int out_h, int out_w, uint8_t* crop_rgb, uint16_t* crop_depth,
                            uint8_t* crop_seg, int* count, cudaStream_t s);
// se3tn_append_pairs: rows of a pair step with count >= min_count copied to their queue's tail (see include/se3tn.h)
struct AppendArgs {
    const uint8_t* rgbA; const uint16_t* depthA; const uint8_t* rgbB; const uint16_t* depthB;   // (n, 176, 176[, 3])
    const int* count; const double* A_in_cam; const double* B_in_cam; const int* queue_ids;     // (n), (n,16), (n,16), (n)
    int n, num_queues, cap, min_count;
    int* tails;                    // (num_queues), advanced by the CTA that finishes last
    unsigned* done;                // context-owned CTA counter, zero between launches
    uint8_t* q_rgbA; uint16_t* q_depthA; uint8_t* q_rgbB; uint16_t* q_depthB; double* q_A; double* q_B;   // (num_queues * cap, ...)
    const uint8_t* segB; uint8_t* q_segB;   // optional fifth plane, (n, 176, 176) -> (num_queues * cap, 176, 176); null: not copied
};
cudaError_t launch_append_pairs(const AppendArgs& a, cudaStream_t s);
cudaError_t launch_nchw_to_stem(const float* src, float* dst, int n, int precision, cudaStream_t s);
cudaError_t launch_maxpool(const float* in, float* out, int n_img, int Hin, int Win, int C, cudaStream_t s);
// poses_in non-null: also the pose update of every track (K6 fused into K4); loss.poses_a non-null: also the loss terms of every pair;
// zero_words: n_zero 32-bit counters cleared for the next step
cudaError_t launch_head_pooled(const float* part /*[n][kPoolSlices][1024]*/, const float* fcw, const float* fcb, float* out_trans, float* out_rot,
                               int n_img, int npix, const int* img_wid, const float* const* fc_table,
                               const double* poses_in, double* poses_out, float tn, float rn, const LossArgs& loss,
                               unsigned* zero_words, int n_zero, cudaStream_t s);
// sums[0] / sums[1]: the sums of the n x 3 translation / rotation terms of sq (n,6), in the fixed order of reduce_loss_terms
cudaError_t launch_loss_reduce(const float* sq, int n, float* sums, cudaStream_t s);
// The loss of n predictions on their own: labels from trans_label / rot_label (n,3) when given, else from loss.poses_a / poses_b;
// the terms go to loss.sq / loss.labels when those are non-null, and their sums to `sums`, as launch_loss_reduce adds them.
cudaError_t launch_pair_loss(const float* trans, const float* rot, const double* trans_label, const double* rot_label,
                             const LossArgs& loss, int n, float* sums, cudaStream_t s);
cudaError_t launch_head(const float* x, const float* fcw, const float* fcb, float* out_trans, float* out_rot,
                        int n_img, int npix, cudaStream_t s);
// `in` points at the first image, in the activation format of `precision` (SE3TN_PREC_*); SE3TN_PREC_FP8: fp8_scale (device)
// is the tensor's scale
cudaError_t launch_nhwc_to_nchw(const void* in, float* out, int n_img, int HW, int C, int precision, cudaStream_t s,
                                const float* fp8_scale = nullptr);
// fp32 weight matrix [rows][ktot] -> the weight format of a tensor-core precision (storage.cuh)
cudaError_t launch_encode_weights(int precision, const float* src, void* dst, int rows, int ktot, cudaStream_t s);
// SE3TN_PREC_FP8 weights: e4m3 codes of w / s_w[row] (K-major, ktot bytes per row) and the per-row power-of-two scales
// s_w[row] = 2^ceil(log2(max_k |w[row][k]| / 448)), 1 for an all-zero row
cudaError_t launch_encode_weights_fp8(const float* src, void* dst, float* row_scale, int rows, int ktot, cudaStream_t s);
// max|x| over images [0, n) of up to kMax bf16x3-format NHWC tensors (channels [c0, c0 + nc) of C): amax_bits[i] receives
// tensor i's maximum as fp32 bits through atomicMax (the caller zeroes them first)
struct AmaxArgs {
    static constexpr int kMax = 8;
    struct Tensor { const uint8_t* buf; int pixels, C, c0, nc; } t[kMax];
    int n_tensors, n;
};
cudaError_t launch_amax_bf16x3(const AmaxArgs& a, unsigned* amax_bits, cudaStream_t s);
cudaError_t launch_permute_rows64(const float* src /*[64][ktot]*/, float* dst, int ktot, cudaStream_t s);
cudaError_t launch_split_stack_weights(const float* src, void* dst /*[128][9*32 | 7*32 words]*/, bool stem, cudaStream_t s);
cudaError_t launch_pose_update(const double* poses_in, const float* trans, const float* rot, float tn, float rn,
                               double* poses_out, int n, cudaStream_t s);
cudaError_t launch_so3_log(const double* poses_a, const double* poses_b, double tn, double rn,
                           double* trans_label, double* rot_label, int n, cudaStream_t s);

}  // namespace se3tn
