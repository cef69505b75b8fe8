// TEST INFRASTRUCTURE ONLY — C entry points that drive the REFERENCE's own compiled PixelSelector (FullSystem/PixelSelector2.cpp), its
// FrameHessian::makeImages and its ImmaturePoint constructor, for tests/test_ref_pin_select.py and tests/golden/make_golden_select.py.
// Built by ref_build_select.sh into a library of its own, linked with the reference objects ref_build.sh compiles and ref_harness.o.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "FullSystem/HessianBlocks.h"
#include "FullSystem/ImmaturePoint.h"
#include "FullSystem/PixelSelector2.h"
#include "util/globalCalib.h"
#include "util/settings.h"

using namespace dso;

namespace {
struct RefSelFrame {
  CalibHessian* Hc;
  FrameHessian* fh;
};
}  // namespace

extern "C" {

// the reference's process-global selection settings (util/settings.cpp:L144, L167-170)
void ref_sel_settings(float minGradHistCut, float minGradHistAdd, float gradDownweightPerLevel, int selectDirectionDistribution, int gammaWeightsPixelSelect) {
  setting_minGradHistCut = minGradHistCut;
  setting_minGradHistAdd = minGradHistAdd;
  setting_gradDownweightPerLevel = gradDownweightPerLevel;
  setting_selectDirectionDistribution = selectDirectionDistribution != 0;
  setting_gammaWeightsPixelSelect = gammaWeightsPixelSelect;
}

// a keyframe as FullSystem builds it: setGlobalCalib, CalibHessian::B as given (NULL: its constructor's identity), FrameHessian::makeImages.
// makeImages never writes rows 0 and h_l-1 of absSquaredGrad[l] (HessianBlocks.cpp:L169), and select reads the last row of level 2 for
// pixels on row h-4; they are cleared here so that runs do not depend on what the allocator returns.
void* ref_sel_frame_create(int w, int h, const double K[4], const float* color, const float* B) {
  Eigen::Matrix3f Km;
  Km.setZero();
  Km(0, 0) = (float)K[0]; Km(1, 1) = (float)K[1]; Km(0, 2) = (float)K[2]; Km(1, 2) = (float)K[3]; Km(2, 2) = 1.f;
  setGlobalCalib(w, h, Km);
  RefSelFrame* F = new RefSelFrame();
  F->Hc = new CalibHessian();
  if (B) std::memcpy(F->Hc->B, B, sizeof(float) * 256);
  F->fh = new FrameHessian();
  for (int l = 0; l < PYR_LEVELS; l++) { F->fh->dIp[l] = 0; F->fh->absSquaredGrad[l] = 0; }
  F->fh->makeImages(const_cast<float*>(color), F->Hc);
  for (int l = 0; l < pyrLevelsUsed; l++) {
    std::memset(F->fh->absSquaredGrad[l], 0, sizeof(float) * wG[l]);
    std::memset(F->fh->absSquaredGrad[l] + (size_t)wG[l] * (hG[l] - 1), 0, sizeof(float) * wG[l]);
  }
  return F;
}
void ref_sel_frame_destroy(void* p) {
  RefSelFrame* F = static_cast<RefSelFrame*>(p);
  delete F->fh;
  delete F->Hc;
  delete F;
}
// levels 0-2 of the frame as [I, dx, dy]
void ref_sel_frame_dI(void* p, int level, float* out) {
  RefSelFrame* F = static_cast<RefSelFrame*>(p);
  for (int i = 0; i < wG[level] * hG[level]; i++)
    for (int k = 0; k < 3; k++) out[3 * i + k] = F->fh->dIp[level][i][k];
}

void* ref_sel_create(int w, int h) { return new PixelSelector(w, h); }
void ref_sel_destroy(void* ps) { delete static_cast<PixelSelector*>(ps); }
int ref_sel_get_potential(void* ps) { return static_cast<PixelSelector*>(ps)->currentPotential; }
void ref_sel_set_potential(void* ps, int p) { static_cast<PixelSelector*>(ps)->currentPotential = p; }
int ref_sel_make_maps(void* ps, void* frame, float* map_out, float density, int recursionsLeft, float thFactor) {
  return static_cast<PixelSelector*>(ps)->makeMaps(static_cast<RefSelFrame*>(frame)->fh, map_out, density, recursionsLeft, false, thFactor);
}

// FullSystem::makeNewTraces' loop (FullSystem.cpp:L1652-1663) with the reference's ImmaturePoint constructor; returns the points kept
int ref_sel_new_traces(void* frame, const float* map, int32_t* u, int32_t* v, float* type, float* color8, float* weights8, float* gradH4, float* energyTH) {
  RefSelFrame* F = static_cast<RefSelFrame*>(frame);
  int n = 0;
  for (int y = patternPadding + 1; y < hG[0] - patternPadding - 2; y++)
    for (int x = patternPadding + 1; x < wG[0] - patternPadding - 2; x++) {
      int i = x + y * wG[0];
      if (map[i] == 0) continue;
      ImmaturePoint* impt = new ImmaturePoint(x, y, F->fh, map[i], F->Hc);
      if (std::isfinite(impt->energyTH)) {
        u[n] = x; v[n] = y; type[n] = map[i];
        std::memcpy(color8 + 8 * n, impt->color, 32); std::memcpy(weights8 + 8 * n, impt->weights, 32);
        gradH4[4 * n] = impt->gradH(0, 0); gradH4[4 * n + 1] = impt->gradH(0, 1); gradH4[4 * n + 2] = impt->gradH(1, 0); gradH4[4 * n + 3] = impt->gradH(1, 1);
        energyTH[n] = impt->energyTH;
        n++;
      }
      delete impt;
    }
  return n;
}

}  // extern "C"
