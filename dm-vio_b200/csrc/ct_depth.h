// the BA handle's side of dmv_ct_set_ref_from_ba, shared by ct_depth.cu and ba_api.cu
#pragma once
#include "../../include/dmvio_b200.h"
#include <cstdint>
#include <cuda_runtime.h>
namespace dmv {
// What dmv_ct_set_ref_from_ba reads from a BA handle (filled by dmv_ba_ref_source, ba_api.cu): the committed linearisation's outputs of the
// residuals into the window's newest frame, one entry per point in dmv_ba_set_points order, and that frame's level-0 plane.
struct CDFromBA {
  int device, w, h, npts;
  const uint8_t* st;        // [npts] state_NewState (0 = IN; 255 = no residual, e.g. dropped by dmv_ba_drop_residuals)
  const float *cu, *cv, *cid; // [npts] centerProjectedTo
  const float* hdi;         // [npts] EFPoint::HdiF of the last solveSystemF
  const float4* img;        // newest frame's level-0 [I, dx, dy, 0] plane
  cudaStream_t stream;      // the BA handle's stream
  // FullSystem::removeOutliers' reorder (remove_outliers.h): n_moves (from, to) pairs of point indices; point `from` (which keeps residuals)
  // takes position `to` (a point without residuals) in the fold order, its own position stays empty.  moves_host: filled by the BA handle;
  // moves: the same pairs on the device (filled by the caller)
  int n_moves;
  const int* moves_host;
  const int* moves;
};
}  // namespace dmv
