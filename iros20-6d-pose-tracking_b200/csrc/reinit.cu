// Re-initialisation of lost tracks (include/se3tn.h, se3tn_lost_tracks / se3tn_accept_starts; oracle/reinit_ref.py).
//
// lost_kernel applies the loss rule to every track's fit row.  Track i is below when 1000 inlier < below_permille model,
// compared as int64 (model = 0 is below); its streak becomes streak + 1 when below, else 0, and it is lost when the streak
// reaches `after`.  Event 1 for a track below, 0 otherwise.  The lost tracks are compacted in ascending order by a block-wide
// exclusive scan over tiles of kLostThreads tracks, so the list is the same whatever order the threads run in.
//
// accept_kernel applies the accept rule to the starts of the m lost tracks, one thread per start: a start whose init status
// is not 0 is event 3 and changes nothing; a start whose fit row ranks strictly above the track's (fit_better, the hypothesis
// choice's order) replaces the track's pose and fit row, event 2; otherwise event 4.  Every one of the m streaks goes back
// to 0.  Tracks that are not in the list are not touched.
#include "reinit.h"
#include "fit.h"
#include "fit_rank.cuh"
#include "init.h"
#include "launch.h"
#include <cub/block/block_scan.cuh>

namespace se3tn {
namespace {
constexpr int kLostThreads = 1024, kAcceptThreads = 128;

__global__ void __launch_bounds__(kLostThreads) lost_kernel(const LostArgs a)
{
    using Scan = cub::BlockScan<int, kLostThreads>;
    __shared__ typename Scan::TempStorage tmp;
    int base = 0;                                        // lost tracks of the tiles before this one
    for (int t0 = 0; t0 < a.n; t0 += kLostThreads) {
        const int i = t0 + threadIdx.x;
        int lost = 0;
        if (i < a.n) {
            const long long model = a.fit_rows[kFitCols * static_cast<size_t>(i)];
            const long long inlier = a.fit_rows[kFitCols * static_cast<size_t>(i) + 2];
            const bool below = model == 0 || 1000LL * inlier < static_cast<long long>(a.below_permille) * model;
            const int streak = below ? a.streak[i] + 1 : 0;
            a.streak[i] = streak;
            a.event[i] = below ? kReinitBelow : kReinitNone;
            lost = below && streak >= a.after;
        }
        int at, total;
        Scan(tmp).ExclusiveSum(lost, at, total);
        if (lost) a.lost[1 + base + at] = i;
        base += total;
        __syncthreads();                                 // tmp is reused by the next tile's scan
    }
    if (threadIdx.x == 0) a.lost[0] = base;
}

__global__ void __launch_bounds__(kAcceptThreads) accept_kernel(const AcceptArgs a)
{
    const int k = blockIdx.x * kAcceptThreads + threadIdx.x;
    if (k >= a.m) return;
    const size_t i = static_cast<size_t>(a.lost_idx[k]);
    const int32_t* start_row = a.start_fit + kFitCols * static_cast<size_t>(k);
    int32_t* row = a.fit_rows + kFitCols * i;
    int event = kReinitNoStart;
    if (a.init_rows[kInitCols * static_cast<size_t>(k)] == 0) {
        event = kReinitRejected;
        if (fit_better(start_row, row)) {
            event = kReinitRestarted;
            for (int c = 0; c < 16; ++c) a.poses[16 * i + c] = a.starts[16 * static_cast<size_t>(k) + c];
            for (int c = 0; c < kFitCols; ++c) row[c] = start_row[c];
        }
    }
    a.event[i] = event;
    a.streak[i] = 0;
}
}  // namespace

cudaError_t launch_lost(const LostArgs& a, cudaStream_t s) {
    if (a.n < 0 || (a.n > 0 && (!a.fit_rows || !a.streak || !a.event)) || !a.lost) return cudaErrorInvalidValue;
    return launch_kernel(lost_kernel, dim3(1), dim3(kLostThreads), 0, s, false, a);
}

cudaError_t launch_accept(const AcceptArgs& a, cudaStream_t s) {
    if (a.m <= 0) return cudaSuccess;
    if (!a.lost_idx || !a.starts || !a.init_rows || !a.start_fit || !a.poses || !a.fit_rows || !a.streak || !a.event)
        return cudaErrorInvalidValue;
    return launch_kernel(accept_kernel, dim3((a.m + kAcceptThreads - 1) / kAcceptThreads), dim3(kAcceptThreads), 0, s, false, a);
}

}  // namespace se3tn
