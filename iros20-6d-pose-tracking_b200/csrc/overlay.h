// Track overlays of the sequence drivers' result videos (see overlay.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
namespace se3tn {
// 32-bit words of one track's H x W dot mask.
size_t overlay_mask_words(int H, int W);
// Track i's model points [offsets[s], offsets[s+1]) of pts, s = track_set[i] (device arrays; max_m: the largest such set), moved
// by poses[i] and projected with K = {fx, fy, cx, cy}, drawn over the RGB frame in BGR with the label mask (label_h rows of W from
// row label_y0, or NULL) under (label_over == 0) or over the dots, and halved -> out_bgr (n, H/2, W/2, 3).  masks: n dot masks of
// overlay_mask_words(H, W) words, cleared here.  H and W even.
cudaError_t launch_draw_tracks(const uint8_t* frame_rgb, int H, int W, const double* K, const double* poses, int n, const double* pts,
                               const int* offsets, const int* track_set, int max_m, const uint8_t* label, int label_y0, int label_h,
                               int label_over, uint32_t* masks, uint8_t* out_bgr, cudaStream_t s);
}
