// CoarseTracker's raw-frame ingest (Undistort::undistort<T> on the device) and its C glue.  Kept apart from coarse_tracker.cpp and
// host_capi.cpp: the CPU build of the host adapters over an oracle stand-in of the C ABI (oracle/Makefile, libhost_on_oracle.so) links
// those two files and has no ingest path.
#include "coarse_tracker.h"
#include "host_capi.h"

namespace dmvio_b200 {

bool CoarseTracker::setUndistort(const dmv_undistort_config& cfg) {
  if (!ct_ || dmv_ct_set_undistort(ct_, &cfg) != DMV_OK) { err_ = dmv_last_error(); return false; }
  return true;
}
bool CoarseTracker::uploadRawImage(const void* raw, int bytes_per_px, float exposure, float factor, float ab_exposure) {
  newFrame_ab_exposure_ = ab_exposure;
  if (!ct_ || dmv_ct_upload_raw_image(ct_, raw, bytes_per_px, exposure, factor) != DMV_OK) { err_ = dmv_last_error(); return false; }
  return true;
}
bool CoarseTracker::downloadFrame(int level, float* dIp_aos3) {
  if (!ct_ || dmv_ct_download_frame(ct_, level, dIp_aos3) != DMV_OK) { err_ = dmv_last_error(); return false; }
  return true;
}

}  // namespace dmvio_b200

using dmvio_b200::CoarseTracker;

int dmvh_ct_set_undistort(void* p, int wOrg, int hOrg, const float* remapX, const float* remapY, const float* G, int nG, const float* vignetteInv,
                          int photometric_mode) {
  const dmv_undistort_config cfg = {wOrg, hOrg, remapX, remapY, G, nG, vignetteInv, photometric_mode};
  return static_cast<CoarseTracker*>(p)->setUndistort(cfg) ? 0 : -1;
}
int dmvh_ct_upload_raw_image(void* p, const void* raw, int bytes_per_px, float exposure, float factor, float ab_exposure) {
  return static_cast<CoarseTracker*>(p)->uploadRawImage(raw, bytes_per_px, exposure, factor, ab_exposure) ? 0 : -1;
}
int dmvh_ct_download_frame(void* p, int level, float* dIp_aos3) { return static_cast<CoarseTracker*>(p)->downloadFrame(level, dIp_aos3) ? 0 : -1; }
