// Multi-hypothesis tracking (see hypotheses.cu): the expansion of n tracks into n x S start poses, and the choice of one
// hypothesis per track from the fit check's rows.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
constexpr int kHypDraws = 8;          // draws columns: U_theta, U_phi of the translation, of the rotation axis, m_T (m), m_R (deg), tries_T, tries_R
constexpr int kHypMaxTries = 64;      // truncated-normal redraws per magnitude before it is clamped to +-max

struct HypArgs {
    const double* poses_in;           // [n][16]: the tracks' previous poses
    const int64_t* keys;              // [n]: each track's draw key (read only when S > 1)
    int n, S;
    uint64_t seed;
    double max_t, max_r_deg;          // metres, degrees
    const int32_t* wid_in;            // [n] or NULL
    const double* width_in;           // [n] or NULL
    double* poses;                    // [n][S][16] out
    int32_t* wid;                     // [n][S] out, NULL when wid_in is NULL
    double* width;                    // [n][S] out, NULL when width_in is NULL
    double* draws;                    // [n][S][kHypDraws] out or NULL
};
// One thread per hypothesis row.  A plain launch: it reads poses_in, which the launch before it may have written.
cudaError_t launch_hypotheses(const HypArgs& a, cudaStream_t s);

struct SelectArgs {
    int n, S;
    const int32_t* rows;              // [n][S][6]: the fit check of every hypothesis (fit.h kFitCols)
    const double* poses;              // [n][S][16]: every hypothesis after the last round
    const float* trans; const float* rot;   // [n][S][3]: their last round's network outputs
    double* poses_out;                // [n][16]
    float* trans_out; float* rot_out; // [n][3] or NULL
    int32_t* choice;                  // [n]
    int32_t* fit_out;                 // [n][6]: the chosen rows
};
// One thread per track.  A plain launch: it starts once the fit kernel before it has completed.
cudaError_t launch_select(const SelectArgs& a, cudaStream_t s);
}  // namespace se3tn
