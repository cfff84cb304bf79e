// ADD / ADD-S / VOCap on the GPU (see metrics.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
namespace se3tn {
cudaError_t launch_add_adi(const double* model, int m, const double* pred, const double* gt, int n,
                           double* out_add, double* out_adi, cudaStream_t s);
cudaError_t vocap(const double* errs, int n, double* out_host, cudaStream_t s);   // synchronises the stream
// ADD / ADD-S of n poses, pose p against points [offsets[s], offsets[s+1]) of the (M,3) table pts, s = pose_set[p] (device arrays).
cudaError_t launch_add_adi_sets(const double* pts, const int* offsets, const int* pose_set, const double* pred, const double* gt,
                                int n, double* out_add, double* out_adi, cudaStream_t s);
// Translation error (mm), rotation angle (degrees), ADD and ADD-S of n rows into out (n,4), as launch_add_adi_sets scores them;
// keep (nullable) uint8 per row: a 0 row gets NaN values and out_set -1 (out_set nullable: each scored row's set id).
cudaError_t launch_pose_errors_sets(const double* pts, const int* offsets, const int* pose_set, const double* pred, const double* gt,
                                    const uint8_t* keep, int n, double* out, int* out_set, cudaStream_t s);
// Device scratch vocap_sets needs for n errors in n_sets sets.
cudaError_t vocap_sets_scratch_bytes(int n, int n_sets, size_t* bytes);
// VOCap of each set's errors and of all n (errs, err_set device; n > 0) -> out_host[0..n_sets], and *bad_host != 0 when an id is
// outside [0, n_sets).  Synchronises the stream.
cudaError_t vocap_sets(const double* errs, const int* err_set, int n, int n_sets, uint8_t* scratch, double* out_host, int* bad_host,
                       cudaStream_t s);
}
