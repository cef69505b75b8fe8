// sm_90a image-plane kernels of FrameHessian::makeImages (HessianBlocks.cpp:L128-191), shared by the BA, coarse-tracker and initialiser
// uploads (launchers declared in common_host.h):
//   repack_aos3_kernel   host-built AoS3 [I, dx, dy] -> float4 texels
//   make_dI_kernel       level-0 [I, dx, dy, 0] from intensities (L169-179)
//   pyr_down_kernel      level l+1 intensity = 2x2 box mean of level l (L159-166)
#include <cuda_runtime.h>

namespace dmv {

__global__ void repack_aos3_kernel(const float* __restrict__ src, float4* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = make_float4(src[3 * i], src[3 * i + 1], src[3 * i + 2], 0.f);
}

__global__ void make_dI_kernel(const float* __restrict__ img, float4* __restrict__ dst, int w, int h) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= w * h) return;
  float dx = 0.f, dy = 0.f;
  if (idx >= w && idx < w * (h - 1)) {  // the reference's flat loop: row ends wrap into the neighbouring rows
    dx = 0.5f * (img[idx + 1] - img[idx - 1]);
    dy = 0.5f * (img[idx + w] - img[idx - w]);
    if (!isfinite(dx)) dx = 0.f;
    if (!isfinite(dy)) dy = 0.f;
  }
  dst[idx] = make_float4(img[idx], dx, dy, 0.f);
}

__global__ void pyr_down_kernel(const float4* __restrict__ src, float* __restrict__ dst, int wl, int hl, int wlm1) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= wl || y >= hl) return;
  const float4* p = src + (size_t)2 * y * wlm1 + 2 * x;
  dst[(size_t)y * wl + x] = 0.25f * (p[0].x + p[1].x + p[wlm1].x + p[wlm1 + 1].x);
}

void launch_repack(const float* src, float4* dst, int n, cudaStream_t s) { repack_aos3_kernel<<<(n + 255) / 256, 256, 0, s>>>(src, dst, n); }
void launch_make_dI(const float* img, float4* dst, int w, int h, cudaStream_t s) { make_dI_kernel<<<(w * h + 255) / 256, 256, 0, s>>>(img, dst, w, h); }
void launch_pyr_down(const float4* src, float* dst, int wl, int hl, int wlm1, cudaStream_t s) {
  pyr_down_kernel<<<dim3((wl + 127) / 128, hl), 128, 0, s>>>(src, dst, wl, hl, wlm1);
}

}  // namespace dmv
