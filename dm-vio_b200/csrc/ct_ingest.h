// raw-frame ingest (ct_ingest.cu): Undistort::undistort<T> + PhotometricUndistorter::processFrame on the device
#pragma once
#include <cuda_runtime.h>
namespace dmv {
struct IngestTables {
  int npx, wOrg;              // output pixels (level 0), raw row length
  const float2* remap;        // (remapX, remapY) per output pixel; nullptr = passthrough
  const float* G;             // response map (device), used when use_G
  const float* vigInv;        // vignetteMapInv (device, wOrg*hOrg), used when use_G and mode 2
  int mode;                   // setting_photometricCalibration
};
// writes the level-0 intensity plane `out` from the raw frame (bpp 1 or 2 bytes per pixel); use_G = the reference's calibrated branch
// (valid && exposure > 0 && mode != 0), otherwise factor * raw
void ingest_launch(const IngestTables& t, const void* raw, int bpp, bool use_G, float factor, float* out, cudaStream_t s);
}  // namespace dmv
