// argument block of ip_trace_kernel (ip_trace.cu), shared with the C ABI in ct_kernels.cu
#pragma once
#include "../../include/dmvio_b200.h"
#include <cuda_runtime.h>
namespace dmv {
struct IPTraceArgs {
  int n, w, h;
  float KRKi[9], Kt[3], aff[2];   // one host frame (tab == nullptr)
  const float* tab;               // several host frames in one launch: [set][14] = KRKi 9 | Kt 3 | aff 2, and set_of[point]
  const int* set_of;
  dmv_ip_settings s;
  const float *u, *v, *color, *weights, *gradH, *energyTH;
  float *idepth_min, *idepth_max, *quality;
  int* status;
  float *uv, *interval;
  const float4* img;
};
struct IPInitArgs {
  int n, w;
  const int* n_dev;   // non-null: the point count is read there (written by an earlier kernel on the stream); n bounds it and sizes the grid
  float outlierTHSumComponent, outlierTH, overallEnergyTHWeight;
  const int *u, *v;
  float *color, *weights, *gradH, *energyTH;
  int* ok;
  const float4* img;
};
struct IPActArgs {   // ip_activate_kernel: FullSystem::optimizeImmaturePoint per point
  int n, nf, w, h, minObs, GNIts;
  float fxl, fyl, cxl, cyl, fxli, fyli, huberTH, minIdepthH_act;
  const float4* img[DMV_MAX_FRAMES];
  const float* RT;    // [h*nf+t][12]
  const float* aff;   // [h*nf+t][2]
  const int* host;
  const float *u, *v, *color, *weights, *energyTH, *idepth_min, *idepth_max;
  int* status;
  float* idepth;
  int* res_state;     // [n][nf]
};
void launch_ip_activate(const IPActArgs& A, cudaStream_t s);
void launch_ip_trace(const IPTraceArgs& A, cudaStream_t s);
void launch_ip_init(const IPInitArgs& A, cudaStream_t s);
}  // namespace dmv
