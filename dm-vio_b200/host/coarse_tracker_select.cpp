// CoarseTracker::makeNewTraces (FullSystem::makeNewTraces on the device) and its C glue.  Kept apart from coarse_tracker.cpp and
// host_capi.cpp: the CPU build of the host adapters over an oracle stand-in of the C ABI (oracle/Makefile, libhost_on_oracle.so) links those
// two files and has no pixel-selection path.
#include "coarse_tracker.h"
#include "host_capi.h"

namespace dmvio_b200 {

bool CoarseTracker::makeNewTraces(int& currentPotential, float density, int recursionsLeft, float thFactor, const float* B, const dmv_ps_settings* settings,
                                  int cap, int* n, int* numPointsTotal, int32_t* u, int32_t* v, float* type, float* color8, float* weights8, float* gradH4,
                                  float* energyTH, float* map) {
  dmv_new_traces_args a = {density, recursionsLeft, thFactor, B, settings, &currentPotential, cap, n, numPointsTotal, u, v, type, color8, weights8, gradH4,
                           energyTH, map};
  if (!ct_ || dmv_ct_make_new_traces(ct_, &a) != DMV_OK) { err_ = dmv_last_error(); return false; }
  return true;
}

}  // namespace dmvio_b200

using dmvio_b200::CoarseTracker;

int dmvh_ct_make_new_traces(void* p, int* potential, float density, int recursionsLeft, float thFactor, const float* B, const float* settings5, int cap,
                            int* n, int* numPointsTotal, int32_t* u, int32_t* v, float* type, float* color8, float* weights8, float* gradH4,
                            float* energyTH, float* map) {
  dmv_ps_settings s;
  if (settings5) {
    s.minGradHistCut = settings5[0]; s.minGradHistAdd = settings5[1]; s.gradDownweightPerLevel = settings5[2];
    s.selectDirectionDistribution = (int)settings5[3]; s.gammaWeightsPixelSelect = (int)settings5[4];
  }
  return static_cast<CoarseTracker*>(p)->makeNewTraces(*potential, density, recursionsLeft, thFactor, B, settings5 ? &s : nullptr, cap, n, numPointsTotal,
                                                       u, v, type, color8, weights8, gradH4, energyTH, map)
             ? 0
             : -1;
}
