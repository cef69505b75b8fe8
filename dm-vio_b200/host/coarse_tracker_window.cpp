// CoarseTracker's keyframe hand-off straight from the BA window on the device (dmv_ct_set_ref_from_ba) and its C glue.  Kept apart from
// coarse_tracker.cpp and host_capi.cpp, like coarse_tracker_ingest.cpp: the CPU build of the host adapters over an oracle stand-in of the
// C ABI (oracle/Makefile, libhost_on_oracle.so) links those two files and has no device hand-off.
#include "coarse_tracker.h"
#include "host_capi.h"
#include <cstdio>

namespace dmvio_b200 {

bool CoarseTracker::setCoarseTrackingRefFromWindow(const WindowBA& W, AffLight ref_aff, float ref_exposure) {
  lastRef_aff_g2l_ = ref_aff;
  lastRef_ab_exposure_ = ref_exposure;
  if (!ct_ || !W.ok()) { err_ = "setCoarseTrackingRefFromWindow: invalid tracker or window"; return false; }
  // The device takes a point exactly when its residual into the newest frame survived the tail (linearizeAll(true) deletes every residual that
  // did not end IN).  The reference takes it when ph->lastResiduals[0] is that residual and IN.  Both agree whenever lastResiduals follows
  // makeKeyFrame (FullSystem.cpp:L1386-1387, FullSystemOptPoint.cpp:L187-193); check it here on the host instead of assuming it.
  const int newest = (int)W.frameHessians.size() - 1;
  if (newest < 1) { err_ = "setCoarseTrackingRefFromWindow: the window has fewer than two frames"; return false; }
  const int tid = W.frameHessians[newest].frameID;
  std::vector<char> has(W.points.size(), 0);
  for (const PointFrameResidual& r : W.activeResiduals)
    if (r.target == newest && r.point >= 0 && r.point < (int)has.size()) has[r.point] = 1;
  for (size_t p = 0; p < W.points.size(); p++) {
    const PointHessian& ph = W.points[p];
    const bool last_in = ph.lastResiduals_target[0] == tid && ph.lastResiduals_state[0] == 0;
    if (last_in != (has[p] != 0)) {
      char m[256];
      std::snprintf(m, sizeof(m), "setCoarseTrackingRefFromWindow: point %zu: lastResiduals[0] %s, but the window %s a residual into the newest frame",
                    p, last_in ? "is IN there" : "is not IN there", has[p] ? "holds" : "holds no");
      err_ = m;
      return false;
    }
  }
  int32_t cnt[DMV_MAX_PYR_LEVELS] = {0};
  if (dmv_ct_set_ref_from_ba(ct_, W.handle(), cnt) != DMV_OK) { err_ = dmv_last_error(); return false; }
  for (int l = 0; l < levels_; l++) { pc_n[l] = cnt[l]; pc_u[l].clear(); pc_v[l].clear(); pc_idepth[l].clear(); pc_color[l].clear(); }
  return true;
}

}  // namespace dmvio_b200

using dmvio_b200::CoarseTracker;
using dmvio_b200::WindowBA;

int dmvh_ct_set_ref_from_window(void* p, void* win, double ref_a, double ref_b, float ref_exposure) {
  dmvio_b200::AffLight a;
  a.a = ref_a; a.b = ref_b;
  return static_cast<CoarseTracker*>(p)->setCoarseTrackingRefFromWindow(*static_cast<WindowBA*>(win), a, ref_exposure) ? 0 : -1;
}
const char* dmvh_ct_error(void* p) { return static_cast<CoarseTracker*>(p)->error().c_str(); }
void* dmvh_window_ba_handle(void* win) { return static_cast<WindowBA*>(win)->handle(); }
int dmvh_window_coarse_ref_inputs(void* win, float* Ku, float* Kv, float* nid, float* HdiF, int32_t* point, int cap) {
  return static_cast<WindowBA*>(win)->coarseTrackingRefInputs(Ku, Kv, nid, HdiF, point, cap);
}
void dmvh_window_get_last_residuals(void* win, int32_t* target2, int32_t* state2) {
  const WindowBA* W = static_cast<WindowBA*>(win);
  for (size_t i = 0; i < W->points.size(); i++)
    for (int k = 0; k < 2; k++) { target2[2 * i + k] = W->points[i].lastResiduals_target[k]; state2[2 * i + k] = W->points[i].lastResiduals_state[k]; }
}
