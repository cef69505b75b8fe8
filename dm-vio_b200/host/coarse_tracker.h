// Host-side C++ mirror of the reference's CoarseTracker surface (src/dso/FullSystem/CoarseTracker.{h,cpp}) on top of
// the C ABI: makeK, setCoarseTrackingRef (makeCoarseDepthL0), trackNewestCoarse with its LM loop and 8x8 solve on the host,
// calcRes + calcGSSSE fused in one CUDA launch per evaluation.
#pragma once
#include "window_ba.h"

namespace dmvio_b200 {

class CoarseTracker {
 public:
  CoarseTracker(int w, int h, int levels, int max_points, int device = 0);
  ~CoarseTracker();
  CoarseTracker(const CoarseTracker&) = delete;
  CoarseTracker& operator=(const CoarseTracker&) = delete;
  bool ok() const { return ct_ != nullptr; }
  const std::string& error() const { return err_; }

  Settings s;
  int levels() const { return levels_; }
  int levelPixels(int l) const { return w_[l] * h_[l]; }

  // CoarseTracker.cpp:L105-134
  void makeK(const CalibHessian& HCalib);
  // CoarseTracker.cpp:L524-538 + makeCoarseDepthL0 (L138-295).  Inputs are what the reference reads from the window:
  // per IN residual targeting the reference frame: centerProjectedTo (Ku, Kv, new_idepth) and the point's HdiF;
  // refdIp[l] = lastRef->dIp[l] (w_l*h_l*3 floats).
  void setCoarseTrackingRef(int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, const float* const* refdIp,
                            AffLight lastRef_aff_g2l, float lastRef_ab_exposure);
  // Same, entirely on the device (dmv_ct_make_coarse_depth): the reference keyframe's raw image is uploaded (pyramid built on the device),
  // splat / pooling / dilation / compaction run there and the pc_* lists never leave the GPU.  Bit-identical lists.
  bool setCoarseTrackingRefOnDevice(int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, const float* ref_image_wh,
                                    AffLight lastRef_aff_g2l, float lastRef_ab_exposure);
  // Same, fed straight from the window on the device (coarse_tracker_window.cpp, dmv_ct_set_ref_from_ba): FullSystem::makeKeyFrame's
  // removeOutliers + setCoarseTrackingRef(frameHessians) (FullSystem.cpp:L1438-1458) after finishOptimize and before the window is
  // re-uploaded (the fold follows removeOutliers' point order).  The reference keyframe is the window's newest frame; its IN residuals, the last solve's HdiF and its level-0 plane never leave the GPU.  Unsharded
  // windows only.  Refuses (false, error()) a window whose lastResiduals bookkeeping disagrees with the residuals it holds into the newest frame.
  bool setCoarseTrackingRefFromWindow(const WindowBA& W, AffLight lastRef_aff_g2l, float lastRef_ab_exposure);
  // newFrame: raw image (pyramid built on the device) and its exposure
  bool setNewFrame(const float* image_wh, float ab_exposure);
  bool setNewFramePyramid(const float* const* dIp, float ab_exposure);
  // Raw frames (coarse_tracker_ingest.cpp): the per-frame part of Undistort::undistort<T> runs on the device (dmv_ct_set_undistort /
  // dmv_ct_upload_raw_image).  setUndistort once per sequence with the host-built tables; uploadRawImage replaces setNewFrame with the
  // camera's frame; downloadFrame reads dIp[level] back (keyframes: pixel selection, initialisation).
  bool setUndistort(const dmv_undistort_config& cfg);
  bool uploadRawImage(const void* raw, int bytes_per_px, float exposure, float factor, float ab_exposure);
  bool downloadFrame(int level, float* dIp_aos3);
  // FullSystem::makeNewTraces on the resident keyframe (coarse_tracker_select.cpp, dmv_ct_make_new_traces): PixelSelector::makeMaps with the
  // caller's currentPotential (in/out; FullSystem's one selector outlives the tracker swap), then the ImmaturePoint constructor per selected
  // pixel.  Outputs as dmv_new_traces_args; false (error()) on overflow with *n = the count needed.
  bool makeNewTraces(int& currentPotential, float density, int recursionsLeft, float thFactor, const float* B, const dmv_ps_settings* settings, int cap,
                     int* n, int* numPointsTotal, int32_t* u, int32_t* v, float* type, float* color8, float* weights8, float* gradH4, float* energyTH,
                     float* map);
  // CoarseTracker.cpp:L539-770 (visual-only branch L639-683)
  bool trackNewestCoarse(SE3& lastToNew_out, AffLight& aff_g2l_out, int coarsestLvl, const double minResForAbort[5]);

  // true (default): the whole LM loop runs on the device in one persistent launch (dmv_ct_track); false: the loop below on the host,
  // one fused calcRes+calcGSSSE launch per evaluation (dmv_ct_calc_res_gs)
  bool useDeviceLM = true;
  // Downstream consumer of the 8x8 system (SURVEY §8b): the slot of dmvio::IMUIntegration::computeCoarseUpdate (IMU/IMUIntegration.hpp:L106-107,
  // called from CoarseTracker.cpp:L616-637 when setting_useIMU): gets H (8x8 row-major), b, extrapFac, lambda; returns the new refToNew and writes
  // the affine increments and the increment norm.  When set, trackNewestCoarse runs its LM loop on the host (one fused calcRes + calcGSSSE launch
  // per evaluation) and calls this instead of the 8x8 LDL^T; acceptCoarseUpdate is called on every accepted step (L700).
  std::function<SE3(const double H[64], const double b[8], float extrapFac, float lambda, double& incA, double& incB, double& incNorm)> computeCoarseUpdate;
  std::function<void()> acceptCoarseUpdate;
  double lastResiduals[5];
  double lastFlowIndicators[3];
  int pc_n[DMV_MAX_PYR_LEVELS];
  int iterations = 0;       // LM iterations of the last trackNewestCoarse
  long long evaluations = 0;  // fused calcRes+GS launches of the last trackNewestCoarse
  double pointEvaluations = 0;  // reference points evaluated, summed over the evaluations (device LM loop only; measurement)
  // reference point cloud of a level (for tests)
  std::vector<float> pc_u[DMV_MAX_PYR_LEVELS], pc_v[DMV_MAX_PYR_LEVELS], pc_idepth[DMV_MAX_PYR_LEVELS], pc_color[DMV_MAX_PYR_LEVELS];

 private:
  // one fused evaluation: Vec6 of calcRes (L508-516) and, if wanted, H/b of calcGSSSE (L341-355)
  bool eval(int lvl, const SE3& refToNew, AffLight aff_g2l, float cutoffTH, bool wantGS, double res6[6], double H[64], double b[8]);
  dmv_ct* ct_ = nullptr;
  int w_[DMV_MAX_PYR_LEVELS], h_[DMV_MAX_PYR_LEVELS], levels_;
  float fx_[DMV_MAX_PYR_LEVELS], fy_[DMV_MAX_PYR_LEVELS], cx_[DMV_MAX_PYR_LEVELS], cy_[DMV_MAX_PYR_LEVELS];
  AffLight lastRef_aff_g2l_;
  float lastRef_ab_exposure_ = 1, newFrame_ab_exposure_ = 1;
  std::string err_;
};

}  // namespace dmvio_b200
