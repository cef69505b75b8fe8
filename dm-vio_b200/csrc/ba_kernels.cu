// Small sm_90a kernels of the bundle-adjustment path next to ba_fused_kernel (ba_fused.cu):
//   ba_resub_kernel     stand-alone EnergyFunctional::resubstituteFPt + point part of doStepFromBackup (the hot loop uses the fused prologue)
//   l2_flush_kernel     larger-than-L2 scrub used by the bench between timed iterations
#include "ba_common.cuh"

namespace dmv {

// ---------------------------------------------------------------------------------------------------------------
// stand-alone EnergyFunctional::resubstituteFPt (EnergyFunctional.cpp:L295-321) + point part of doStepFromBackup
// sums[0..2] += sum step^2, sum |idepth_backup|, npts   (caller zeroes sums)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) ba_resub_kernel(const __grid_constant__ BAWinDev W, const __grid_constant__ BAIter it, int apply,
                                                       double* __restrict__ sums) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  float step2 = 0.f, nid = 0.f;
  if (p < W.npts) {
    int h = 0;
    while (h < W.nf - 1 && p >= W.host_start[h + 1]) h++;
    const float step = resub_point(W, it, p, h);
    W.step[p] = step;
    const float idb = W.idepth_backup[p];
    step2 = step * step;
    nid = fabsf(idb);
    if (apply) {
      const float v = idb + step;
      W.idepth_out[p] = v;  // DM-VIO: idepth_zero follows (FullSystemOptimize.cpp:L268); the host aliases the pointers
    }
  }
  __shared__ float s2[128], sn[128];
  s2[threadIdx.x] = step2; sn[threadIdx.x] = nid;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) { s2[threadIdx.x] += s2[threadIdx.x + s]; sn[threadIdx.x] += sn[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    atomicAdd(sums, (double)s2[0]);
    atomicAdd(sums + 1, (double)sn[0]);
    atomicAdd(sums + 2, (double)min(128, W.npts - (int)blockIdx.x * 128));
  }
}

// larger-than-L2 scrub used by the bench between timed iterations
__global__ void l2_flush_kernel(float4* buf, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) { float4 v = buf[i]; v.x += 1.f; buf[i] = v; }
}

// ---------------------------------------------------------------------------------------------------------------
// launch helpers (called from ba_api.cu)
// ---------------------------------------------------------------------------------------------------------------
void launch_resub_kernel(const BAWinDev& W, const BAIter& it, int apply, double* sums, cudaStream_t s) {
  ba_resub_kernel<<<(W.npts + 127) / 128, 128, 0, s>>>(W, it, apply, sums);
}
void launch_l2_flush(float4* buf, size_t n, cudaStream_t s) { l2_flush_kernel<<<132 * 8, 256, 0, s>>>(buf, n); }

}  // namespace dmv
