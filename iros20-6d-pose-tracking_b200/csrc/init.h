// Start poses from a segmentation mask or a 2D box and a depth frame: render-and-compare over a rotation grid (see init.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
constexpr int kInitCols = 8;             // score row: status, candidate, model, maskc, overlap, pairs, inlier, delta_mm (include/se3tn.h)
constexpr int kInitStats = 6;            // mask statistics (int64): status, mask, depth_px, sum_u, sum_v, z_med
constexpr int kInitAcc = 4;              // per-object accumulators of the mask pass: mask, depth_px, sum_u, sum_v
constexpr int kInitBins = 65536;         // one bin per uint16 depth value
constexpr int kInitMaxKeep = 32;
constexpr int kInitMaxDepths = 8;        // se3tn_init_boxes' depth candidates D per object

struct MaskArgs {
    const uint16_t* depth; const uint8_t* seg; int H, W;
    const int32_t* labels; int n;        // [n] device, 1..255 (null with boxes)
    const int32_t* boxes;                // null: the pixels of object i are seg == labels[i]; else [n][4] device (x0, y0, x1, y1)
                                         // half-open, inside the frame, and the pixels are the box's
    int D;                               // depth candidates per object, 1..kInitMaxDepths (1 with a mask)
    long long box_px_max;                // with boxes: the largest box's pixel count (sizes the box pass)
    unsigned long long* acc;             // [n][kInitAcc], zeroed by launch_mask_stats
    unsigned* hist;                      // [n][kInitBins] depth histogram of the object's pixels with depth, zeroed by launch_mask_stats
    int min_pixels;
    double fx, fy, cx, cy;
    long long* stats;                    // [n][kInitStats]
    double* t0;                          // [n][D][3] metres
};
// memsets + 2 launches (the pass over the frame or the boxes, then one CTA per object for the depths and t0)
cudaError_t launch_mask_stats(const MaskArgs& a, cudaStream_t s);

struct GridArgs {
    int n, V, R, D;
    const double* t0;                    // [n][D][3]
    const double* width_in;              // [n] mm
    const int32_t* ids_in;               // [n] or null (mesh 0)
    double* poses;                       // [n D V R][16] object i's candidate c = d V R + v R + r is row i D V R + c
    double* width;                       // [n D V R]
    int32_t* ids;                        // [n D V R], or null when ids_in is
};
cudaError_t launch_grid(const GridArgs& a, cudaStream_t s);

struct ScoreArgs {
    const double* poses;                 // [rows][16] indexed by the global row
    const double* object_width;          // [rows]
    double fx, fy, cx, cy;
    const uint16_t* frame_depth; const uint8_t* seg; int H, W;
    const uint16_t* rendered;            // [chunk rows][176][176] mm, chunk row r is global row row0 + r
    const int32_t* labels;               // [n] (null with boxes)
    const int32_t* boxes;                // null: M = (seg == labels[i]); else [n][4] device: M = the frame pixel lies in object i's box
    const long long* stats;              // [n][kInitStats]
    int row0, per_object;                // object of global row g: g / per_object
    const int32_t* cand_rows;            // null: the candidate is g % per_object; else [rows][kInitCols], the candidate in column 1
    int tau;                             // mm
    int fixed_delta;                     // 1: delta = 0 (a refined pose is scored where it is)
    int32_t* rows;                       // [rows][kInitCols] indexed by the global row
};
// one 4-CTA cluster per chunk row, launched with programmatic dependent launch behind the render that draws `rendered`
cudaError_t launch_score(const ScoreArgs& a, int chunk_rows, cudaStream_t s);

struct KeepArgs {
    int n, per_object, K;
    const int32_t* rows;                 // [n per_object][kInitCols]
    const double* poses;                 // [n per_object][16]
    const double* width_in; const int32_t* ids_in;   // [n]; ids may be null
    int32_t* kept_rows; double* kept_poses; double* kept_width; int32_t* kept_ids;   // [n K] ...; kept_ids null when ids_in is
};
// one CTA per object: its K best rows in rank order, each grid pose moved along its ray by the row's delta
cudaError_t launch_keep(const KeepArgs& a, cudaStream_t s);

struct ChooseArgs {
    int n, K;
    const int32_t* rows;                 // [n K][kInitCols]
    const double* poses;                 // [n K][16]
    const long long* stats;              // [n][kInitStats]
    double* poses_out; int32_t* rows_out;   // [n][16], [n][kInitCols]; NaN pose when the object's status != 0
};
cudaError_t launch_choose(const ChooseArgs& a, cudaStream_t s);
}  // namespace se3tn
