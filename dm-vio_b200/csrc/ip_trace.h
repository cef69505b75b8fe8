// ip_init_kernel (ip_trace.cu), which pixel selection (ps_select.cu) also runs on its candidates
#pragma once
#include "../../include/dmvio_b200.h"
#include <cuda_runtime.h>
namespace dmv {
struct IPInitArgs {
  int n, w;
  const int* n_dev;   // non-null: the point count is read there (written by an earlier kernel on the stream); n bounds it and sizes the grid
  float outlierTHSumComponent, outlierTH, overallEnergyTHWeight;
  const int *u, *v;
  float *color, *weights, *gradH, *energyTH;
  int* ok;
  const float4* img;
};
void launch_ip_init(const IPInitArgs& A, cudaStream_t s);
}  // namespace dmv
