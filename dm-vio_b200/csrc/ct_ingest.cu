// sm_90a raw-frame ingest: the per-frame part of Undistort::undistort<T> (util/Undistort.cpp:L385-482) with
// PhotometricUndistorter::processFrame (L213-252), one output pixel per thread, writing the level-0 intensity plane that
// grad_kernel / pyr_down_kernel (ct_kernels.cu) turn into the pyramid.
//
// The reference maps the whole raw image photometrically and then resamples it.  The map is pointwise, so each thread maps only
// the four raw taps it reads: same values, no intermediate image.  Bit-identical to the reference's scalar SSE2 code: this
// translation unit is compiled with -fmad=false (see the Makefile) and keeps the reference's operation order.
#include "ct_ingest.h"

namespace dmv {

// PM: 0 = factor * raw (no calibration, exposure <= 0 or mode 0; L222-230), 1 = G[raw] (L233-236), 2 = G[raw] * vignetteMapInv (L238-242)
template <typename T, int PM, bool REMAP>
__global__ void __launch_bounds__(256) ingest_kernel(const T* __restrict__ raw, const float2* __restrict__ remap, const float* __restrict__ G,
                                                     const float* __restrict__ vigInv, float factor, float* __restrict__ out, int npx, int wOrg) {
  __shared__ float sG[256];
  if (PM != 0 && sizeof(T) == 1) {  // the 8-bit LUT from shared memory; the 65536-entry one does not fit and is read through L2
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sG[i] = G[i];
    __syncthreads();
  }
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= npx) return;
  auto tap = [&](int j) -> float {
    const int r = raw[j];
    if (PM == 0) return factor * (float)r;
    const float g = sizeof(T) == 1 ? sG[r] : __ldg(G + r);
    return PM == 2 ? g * __ldg(vigInv + j) : g;
  };
  if (!REMAP) {  // passthrough (L474-477)
    out[idx] = tap(idx);
    return;
  }
  const float2 m = remap[idx];
  float xx = m.x, yy = m.y;
  if (xx < 0) {
    out[idx] = 0.f;
    return;
  }
  // L449-463: integer and rational parts, then the bilinear sum in the reference's order
  const int xxi = (int)xx, yyi = (int)yy;
  xx -= xxi;
  yy -= yyi;
  const float xxyy = xx * yy;
  const int j = xxi + yyi * wOrg;
  out[idx] = xxyy * tap(j + 1 + wOrg) + (yy - xxyy) * tap(j + wOrg) + (xx - xxyy) * tap(j + 1) + (1 - xx - yy + xxyy) * tap(j);
}

template <typename T, int PM>
static void launch_pm(const IngestTables& t, const T* raw, float factor, float* out, cudaStream_t s) {
  const unsigned grid = (unsigned)((t.npx + 255) / 256);
  if (t.remap)
    ingest_kernel<T, PM, true><<<grid, 256, 0, s>>>(raw, t.remap, t.G, t.vigInv, factor, out, t.npx, t.wOrg);
  else
    ingest_kernel<T, PM, false><<<grid, 256, 0, s>>>(raw, t.remap, t.G, t.vigInv, factor, out, t.npx, t.wOrg);
}

template <typename T>
static void launch_t(const IngestTables& t, const T* raw, bool use_G, float factor, float* out, cudaStream_t s) {
  if (!use_G) launch_pm<T, 0>(t, raw, factor, out, s);
  else if (t.mode == 2) launch_pm<T, 2>(t, raw, factor, out, s);
  else launch_pm<T, 1>(t, raw, factor, out, s);
}

void ingest_launch(const IngestTables& t, const void* raw, int bpp, bool use_G, float factor, float* out, cudaStream_t s) {
  if (bpp == 1) launch_t(t, static_cast<const unsigned char*>(raw), use_G, factor, out, s);
  else launch_t(t, static_cast<const unsigned short*>(raw), use_G, factor, out, s);
}

}  // namespace dmv
