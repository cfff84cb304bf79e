// Re-initialisation of lost tracks: the loss rule over the fit rows, and the accept rule for their starts (see reinit.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
// event codes per track and step (include/se3tn.h, se3tn_lost_tracks / se3tn_accept_starts)
constexpr int kReinitNone = 0, kReinitBelow = 1, kReinitRestarted = 2, kReinitNoStart = 3, kReinitRejected = 4;

struct LostArgs {
    const int32_t* fit_rows;             // [n][kFitCols]
    int n, below_permille, after;
    int32_t* streak;                     // [n] in / out
    int32_t* event;                      // [n]
    int32_t* lost;                       // [n + 1]: the count, then the lost tracks in ascending order
};
// one CTA
cudaError_t launch_lost(const LostArgs& a, cudaStream_t s);

struct AcceptArgs {
    const int32_t* lost_idx; int m;      // [m] the tracks the starts belong to
    const double* starts;                // [m][16]
    const int32_t* init_rows;            // [m][kInitCols]
    const int32_t* start_fit;            // [m][kFitCols]
    double* poses;                       // [n][16] in place
    int32_t* fit_rows;                   // [n][kFitCols] in place
    int32_t* streak;                     // [n]
    int32_t* event;                      // [n]
};
cudaError_t launch_accept(const AcceptArgs& a, cudaStream_t s);
}  // namespace se3tn
