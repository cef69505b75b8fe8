// device-side makeCoarseDepthL0 (ct_depth.cu): per-level working planes and output lists
#pragma once
#include "../../include/dmvio_b200.h"
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>
namespace dmv {
struct CDLevels {
  int levels, cap;
  int w[DMV_MAX_PYR_LEVELS], h[DMV_MAX_PYR_LEVELS];
  float *idepth[DMV_MAX_PYR_LEVELS], *ws[DMV_MAX_PYR_LEVELS], *ws2[DMV_MAX_PYR_LEVELS];
  const float4* img[DMV_MAX_PYR_LEVELS];                       // the reference frame's planes (I, dx, dy, 0)
  float *pc_u[DMV_MAX_PYR_LEVELS], *pc_v[DMV_MAX_PYR_LEVELS], *pc_id[DMV_MAX_PYR_LEVELS], *pc_col[DMV_MAX_PYR_LEVELS];
  int *rowcnt, *rowoff, *totals;                               // scratch rows; totals[l] = pc_n[l] (device-visible pinned host memory)
};
void cd_launch(const CDLevels& L, int n_unique, const int* d_pix, const float* d_idw, const float* d_wsum, cudaStream_t s);

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
// scratch of the device fold: radix-sort keys / ordinals (double-buffered) and CUB's temporary storage, for up to cap points
struct CDSortScratch {
  unsigned *key[2];
  int *ord[2];
  void* temp;
  size_t temp_bytes;
  int* bad;                 // lowest point index whose projection leaves the image (>= npts: none)
  int* moves;               // device copy of CDFromBA::moves_host (2 * cap ints)
  int* h_moves;             // its pinned staging
};
size_t cd_sort_temp_bytes(int cap);
// the same lists as cd_launch fed with the host fold of the IN residuals, built without leaving the device.  *kernels = the kernels it
// launches itself (the radix sort's own launches are not counted); returns the first error of the sort or a launch.
cudaError_t cd_launch_from_ba(const CDLevels& L, const CDFromBA& B, const CDSortScratch& S, cudaStream_t s, int* kernels);
}  // namespace dmv
