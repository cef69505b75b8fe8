// TEST INFRASTRUCTURE ONLY — C harness around the REFERENCE's own Undistort (src/dso/util/Undistort.cpp, compiled from where it lies by
// oracle/ref_build.sh).  The test writes the calibration and response files; the vignette image comes from memory through the
// two IOWrap readers defined here (the reference reads it with OpenCV).  Exposes Undistort::undistort<T> and the tables it built, so the
// restatement (orc_undistort.cpp) and the device path can be fed the very same remap, G and vignetteMapInv.
#include <Eigen/Core>
#include <cstring>
#include <string>
#include <vector>
#include "util/NumType.h"
#include "util/MinimalImage.h"
#include "util/ImageAndExposure.h"
#include "util/settings.h"
#define private public
#define protected public
#include "util/Undistort.h"
#undef private
#undef protected

namespace {
std::vector<unsigned char> g_vig8;
std::vector<unsigned short> g_vig16;
int g_vw = 0, g_vh = 0;
}  // namespace

namespace dso {
namespace IOWrap {
MinimalImageB* readImageBW_8U(std::string) {
  if (g_vig8.empty()) return nullptr;
  MinimalImageB* m = new MinimalImageB(g_vw, g_vh);
  std::memcpy(m->data, g_vig8.data(), g_vig8.size());
  return m;
}
MinimalImage<unsigned short>* readImageBW_16U(std::string) {
  if (g_vig16.empty()) return nullptr;
  auto* m = new MinimalImage<unsigned short>(g_vw, g_vh);
  std::memcpy(m->data, g_vig16.data(), g_vig16.size() * 2);
  return m;
}
}  // namespace IOWrap
}  // namespace dso

using namespace dso;

extern "C" {
// Undistort::getUndistorterForFile(calib, gamma, "vignette") with setting_photometricCalibration = mode during construction (it shapes G,
// Undistort.cpp:L112-115).  vignette: vw*vh pixels of vbpp bytes, or NULL (no vignette: the calibration is invalid, as in the reference).
void* refu_create(const char* calib, const char* gamma, const void* vignette, int vbpp, int vw, int vh, int mode) {
  g_vig8.clear(); g_vig16.clear();
  g_vw = vw; g_vh = vh;
  if (vignette && vbpp == 1) g_vig8.assign((const unsigned char*)vignette, (const unsigned char*)vignette + (size_t)vw * vh);
  if (vignette && vbpp == 2) g_vig16.assign((const unsigned short*)vignette, (const unsigned short*)vignette + (size_t)vw * vh);
  setting_photometricCalibration = mode;
  return Undistort::getUndistorterForFile(calib, gamma, "vignette");
}
void refu_destroy(void* p) {
  Undistort* u = static_cast<Undistort*>(p);
  delete u->photometricUndist;
  delete u;
}
// out4 = (w, h, wOrg, hOrg); returns passthrough; valid_GDepth = (photometric valid, GDepth)
int refu_info(void* p, int* out4, int* valid_GDepth) {
  Undistort* u = static_cast<Undistort*>(p);
  out4[0] = u->w; out4[1] = u->h; out4[2] = u->wOrg; out4[3] = u->hOrg;
  valid_GDepth[0] = u->photometricUndist->valid ? 1 : 0;
  valid_GDepth[1] = u->photometricUndist->GDepth;
  return u->passthrough ? 1 : 0;
}
// remapX / remapY (w*h), G (65536: the whole array the reference indexes), vignetteMapInv (wOrg*hOrg, if valid); any may be NULL
void refu_tables(void* p, float* remapX, float* remapY, float* G, float* vigInv) {
  Undistort* u = static_cast<Undistort*>(p);
  const size_t n = (size_t)u->w * u->h, no = (size_t)u->wOrg * u->hOrg;
  if (remapX) std::memcpy(remapX, u->remapX, n * 4);
  if (remapY) std::memcpy(remapY, u->remapY, n * 4);
  if (G) std::memcpy(G, u->photometricUndist->G, 65536 * 4);
  if (vigInv && u->photometricUndist->vignetteMapInv) std::memcpy(vigInv, u->photometricUndist->vignetteMapInv, no * 4);
}
// Undistort::undistort<T>(raw, exposure, 0, factor) with setting_photometricCalibration = mode; out = w*h floats
void refu_undistort(void* p, const void* raw, int bpp, float exposure, float factor, int mode, float* out) {
  Undistort* u = static_cast<Undistort*>(p);
  setting_photometricCalibration = mode;
  ImageAndExposure* r;
  if (bpp == 1) {
    MinimalImageB img(u->wOrg, u->hOrg, (unsigned char*)raw);
    r = u->undistort<unsigned char>(&img, exposure, 0.0, factor);
  } else {
    MinimalImage<unsigned short> img(u->wOrg, u->hOrg, (unsigned short*)raw);
    r = u->undistort<unsigned short>(&img, exposure, 0.0, factor);
  }
  std::memcpy(out, r->image, sizeof(float) * u->w * u->h);
  delete r;
}
}
