// sm_90a raw-frame ingest: the per-frame part of Undistort::undistort<T> (util/Undistort.cpp:L385-482) with
// PhotometricUndistorter::processFrame (L213-252), one output pixel per thread, writing the level-0 intensity plane that
// ct_build_pyramid turns into the pyramid; and the entry points dmv_ct_set_undistort / dmv_ct_upload_raw_image.
//
// The reference maps the whole raw image photometrically and then resamples it.  The map is pointwise, so each thread maps only
// the four raw taps it reads: same values, no intermediate image.  Bit-identical to the reference's scalar SSE2 code: this
// translation unit is compiled with -fmad=false (see the Makefile) and keeps the reference's operation order.
#include "ct_handle.h"
#include <cstring>
#include <vector>

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
static void launch_pm(const dmv_ct* c, const T* raw, float factor) {
  const int npx = c->w[0] * c->h[0];
  const unsigned grid = (unsigned)((npx + 255) / 256);
  if (c->d_remap)
    ingest_kernel<T, PM, true><<<grid, 256, 0, c->stream>>>(raw, c->d_remap, c->d_G, c->d_vigInv, factor, c->d_gray[0], npx, c->wOrg);
  else
    ingest_kernel<T, PM, false><<<grid, 256, 0, c->stream>>>(raw, c->d_remap, c->d_G, c->d_vigInv, factor, c->d_gray[0], npx, c->wOrg);
}

template <typename T>
static void launch_t(const dmv_ct* c, const T* raw, bool use_G, float factor) {
  if (!use_G) launch_pm<T, 0>(c, raw, factor);
  else if (c->pmode == 2) launch_pm<T, 2>(c, raw, factor);
  else launch_pm<T, 1>(c, raw, factor);
}

}  // namespace dmv

using namespace dmv;

int dmv_ct_set_undistort(dmv_ct* c, const dmv_undistort_config* u) {
  if (!c || !u) return set_error(DMV_ERR_INVALID, "null argument");
  const int w = c->w[0], h = c->h[0];
  if (u->wOrg < 2 || u->hOrg < 2 || (size_t)u->wOrg * u->hOrg > ((size_t)1 << 28)) return set_error(DMV_ERR_INVALID, "bad raw size %d x %d", u->wOrg, u->hOrg);
  if (!u->remapX != !u->remapY) return set_error(DMV_ERR_INVALID, "remapX and remapY must both be given or both be NULL");
  if (!u->remapX && (u->wOrg != w || u->hOrg != h)) return set_error(DMV_ERR_INVALID, "passthrough needs the raw size to equal level 0 (%d x %d)", w, h);
  if (u->photometric_mode < 0 || u->photometric_mode > 2) return set_error(DMV_ERR_INVALID, "photometric_mode must be 0, 1 or 2");
  if (u->G && (u->nG < 256 || u->nG > 65536)) return set_error(DMV_ERR_INVALID, "nG = %d: the response map has 256 to 65536 entries", u->nG);
  if (u->G && u->photometric_mode == 2 && !u->vignetteInv) return set_error(DMV_ERR_INVALID, "photometric_mode 2 needs vignetteInv");
  const size_t npx = (size_t)w * h, nraw = (size_t)u->wOrg * u->hOrg;
  std::vector<float2> remap;
  if (u->remapX) {  // every sample the kernel reads must lie inside the raw image (the reference's constructor guarantees it, L920-941)
    remap.resize(npx);
    const float xmax = (float)(u->wOrg - 1), ymax = (float)(u->hOrg - 1);
    for (size_t i = 0; i < npx; i++) {
      const float x = u->remapX[i], y = u->remapY[i];
      if (!(x < 0) && !(x >= 0 && x < xmax && y >= 0 && y < ymax))
        return set_error(DMV_ERR_INVALID, "remap entry %zu = (%g, %g) lies outside [0, %d) x [0, %d)", i, x, y, u->wOrg - 1, u->hOrg - 1);
      remap[i] = make_float2(x, y);
    }
  }
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));  // kernels in flight may read the old tables or the staging buffer
  c->staging_busy = false;
  c->have_undistort = false;
  c->d_remap = {}; c->d_G = {}; c->d_vigInv = {}; c->d_raw = {};
  CK(c->h_scratch.reserve((nraw * 2 + sizeof(float) - 1) / sizeof(float)));
  CK(c->d_raw.alloc(nraw * 2));
  if (u->remapX) {
    CK(c->d_remap.alloc(npx));
    CK(cudaMemcpy(c->d_remap, remap.data(), npx * sizeof(float2), cudaMemcpyHostToDevice));
  }
  if (u->G) {
    CK(c->d_G.alloc(u->nG));
    CK(cudaMemcpy(c->d_G, u->G, (size_t)u->nG * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (u->G && u->vignetteInv) {
    CK(c->d_vigInv.alloc(nraw));
    CK(cudaMemcpy(c->d_vigInv, u->vignetteInv, nraw * sizeof(float), cudaMemcpyHostToDevice));
  }
  c->wOrg = u->wOrg; c->hOrg = u->hOrg; c->nG = u->G ? u->nG : 0; c->pmode = u->photometric_mode;
  c->have_undistort = true;
  return DMV_OK;
}

int dmv_ct_upload_raw_image(dmv_ct* c, const void* raw, int bpp, float exposure, float factor) {
  if (!c || !raw) return set_error(DMV_ERR_INVALID, "null argument");
  if (bpp != 1 && bpp != 2) return set_error(DMV_ERR_INVALID, "bytes_per_px must be 1 or 2");
  if (!c->have_undistort) return set_error(DMV_ERR_INVALID, "dmv_ct_set_undistort first");
  // PhotometricUndistorter::processFrame L222: the calibrated branch needs a valid calibration, exposure_time > 0 and mode != 0
  const bool use_G = c->d_G && exposure > 0 && c->pmode != 0;
  if (use_G && c->nG < (bpp == 1 ? 256 : 65536)) return set_error(DMV_ERR_INVALID, "a %d-entry response map does not cover %d-bit pixels", c->nG, 8 * bpp);
  CK(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->wOrg * c->hOrg * bpp;
  CK(ct_wait_staging(c));
  std::memcpy(c->h_scratch, raw, bytes);
  CK(cudaMemcpyAsync(c->d_raw, c->h_scratch, bytes, cudaMemcpyHostToDevice, c->stream));
  // the level-0 intensity plane d_gray[0] from the raw frame
  if (bpp == 1) launch_t(c, c->d_raw.get(), use_G, factor);
  else launch_t(c, reinterpret_cast<const unsigned short*>(c->d_raw.get()), use_G, factor);
  c->launches++;
  const int rc = ct_build_pyramid(c, 0);
  if (rc != DMV_OK) return rc;
  c->staging_busy = true;  // asynchronous like dmv_ct_upload_new_image
  return DMV_OK;
}
