// Host-side C++ mirror of FullSystem::optimize / EnergyFunctional on top of the C ABI — see window_ba.h.
#include "window_ba.h"
#include "marg_frame.h"
#include "nullspace.h"
#include "../csrc/inv3.h"
#include "../csrc/remove_outliers.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>

namespace dmvio_b200 {

void AffLight::fromToVecExposure(float exposureF, float exposureT, AffLight g2F, AffLight g2T, double out[2]) {
  if (exposureF == 0 || exposureT == 0) exposureT = exposureF = 1;  // util/NumType.h:L174-186
  const double a = std::exp(g2T.a - g2F.a) * exposureT / exposureF;
  out[0] = a;
  out[1] = g2T.b - a * g2F.b;
}

void CalibHessian::setValue(const double v[4]) {  // HessianBlocks.h:L356-371
  for (int i = 0; i < 4; i++) value[i] = v[i];
  value_scaled[0] = SCALE_F * value[0]; value_scaled[1] = SCALE_F * value[1];
  value_scaled[2] = SCALE_C * value[2]; value_scaled[3] = SCALE_C * value[3];
  for (int i = 0; i < 4; i++) value_scaledf[i] = (float)value_scaled[i];
  value_scaledi[0] = 1.0f / value_scaledf[0];
  value_scaledi[1] = 1.0f / value_scaledf[1];
  value_scaledi[2] = -value_scaledf[2] / value_scaledf[0];
  value_scaledi[3] = -value_scaledf[3] / value_scaledf[1];
  for (int i = 0; i < 4; i++) value_minus_value_zero[i] = value[i] - value_zero[i];
}
void CalibHessian::setValueScaled(const double vs[4]) {  // HessianBlocks.h:L373-387
  const double v[4] = {vs[0] / SCALE_F, vs[1] / SCALE_F, vs[2] / SCALE_C, vs[3] / SCALE_C};
  setValue(v);
  for (int i = 0; i < 4; i++) { value_scaled[i] = vs[i]; value_scaledf[i] = (float)vs[i]; }
  value_scaledi[0] = 1.0f / value_scaledf[0];
  value_scaledi[1] = 1.0f / value_scaledf[1];
  value_scaledi[2] = -value_scaledf[2] / value_scaledf[0];
  value_scaledi[3] = -value_scaledf[3] / value_scaledf[1];
}

void FrameHessian::setState(const double s[10]) {  // HessianBlocks.h:L172-186
  for (int i = 0; i < 10; i++) state[i] = s[i];
  for (int i = 0; i < 3; i++) state_scaled[i] = SCALE_XI_TRANS * s[i];
  for (int i = 3; i < 6; i++) state_scaled[i] = SCALE_XI_ROT * s[i];
  state_scaled[6] = SCALE_A * s[6]; state_scaled[7] = SCALE_B * s[7];
  state_scaled[8] = SCALE_A * s[8]; state_scaled[9] = SCALE_B * s[9];
  PRE_worldToCam = SE3::exp(state_scaled) * worldToCam_evalPT;
  PRE_camToWorld = PRE_worldToCam.inverse();
}

WindowBA::WindowBA(int w, int h, int max_frames, int max_points, int device) : w_(w), h_(h), max_frames_(max_frames), max_points_(max_points) {
  dmv_ba_config cfg = {w, h, max_frames, max_points, device, 0};
  if (dmv_ba_create(&cfg, &ba_) != DMV_OK) { err_ = dmv_last_error(); ba_ = nullptr; }
  for (int i = 0; i < 4; i++) { Hcalib.value_zero[i] = 0; Hcalib.step[i] = 0; Hcalib.value_backup[i] = 0; }
}
WindowBA::~WindowBA() { if (ba_) dmv_ba_destroy(ba_); }

bool WindowBA::fail(const char* what) {
  err_ = std::string(what) + ": " + dmv_last_error();
  return false;
}

int WindowBA::insertFrame(const float* image, const SE3& evalPT, const double state[10], const double state_zero[10], float ab_exposure, int frameID) {
  if (!ba_ || nf() >= max_frames_) return -1;
  FrameHessian f;
  f.worldToCam_evalPT = evalPT;
  for (int i = 0; i < 10; i++) { f.state_zero[i] = state_zero[i]; f.step[i] = 0; f.state_backup[i] = state[i]; }
  f.ab_exposure = ab_exposure;
  f.frameID = frameID;
  f.slot = 0;  // first image slot not used by a frame of the window: frames stay resident on the device while window indices shift
  for (bool used = true; used; f.slot += used ? 1 : 0) {
    used = false;
    for (const FrameHessian& g : frameHessians) used = used || g.slot == f.slot;
  }
  f.setState(state);
  if (image && dmv_ba_upload_image(ba_, f.slot, image) != DMV_OK) { fail("dmv_ba_upload_image"); return -1; }
  growHM(HM, bM, nf());  // EnergyFunctional::insertFrame (EnergyFunctional.cpp:L453-496): 8 zero rows / columns for the new keyframe
  frameHessians.push_back(f);
  return nf() - 1;
}
int WindowBA::insertFrameDI(const float* dI, const SE3& evalPT, const double state[10], const double state_zero[10], float ab_exposure, int frameID) {
  const int idx = insertFrame(nullptr, evalPT, state, state_zero, ab_exposure, frameID);
  if (idx < 0) return idx;
  if (dmv_ba_upload_frame(ba_, frameHessians[idx].slot, dI) != DMV_OK) { fail("dmv_ba_upload_frame"); return -1; }
  return idx;
}

// EnergyFunctional::marginalizeFrame as far as the GPU side is concerned (EnergyFunctional.cpp:L511-676): the frame leaves the window,
// its image slot becomes free, later frames shift down by one index.  (The marginalisation prior HM/bM is host data owned by the caller.)
void WindowBA::dropFrame(int idx) {
  if (idx < 0 || idx >= nf()) return;
  frameHessians.erase(frameHessians.begin() + idx);
  HM.clear(); bM.clear();
}

bool WindowBA::marginalizeFrame(int idx) {
  err_.clear();  // per-call status: an earlier, already reported failure must not fail this call
  const int n = nf();
  if (idx < 0 || idx >= n) return false;
  for (const PointHessian& p : points)
    if (p.host == idx) { err_ = "marginalizeFrame: the frame still hosts points (flagPointsForRemoval + marginalizePointsF first)"; return false; }
  // EnergyFunctional.cpp:L569-631 on the host prior; EFFrame::prior / delta_prior as takeData left them (EnergyFunctionalStructs.cpp:L52-64)
  if ((int)HM.size() != (8 * n + CPARS) * (8 * n + CPARS)) { HM.assign((size_t)(8 * n + CPARS) * (8 * n + CPARS), 0.0); bM.assign(8 * n + CPARS, 0.0); }
  {
    const FrameHessian& f = frameHessians[idx];
    double pr[10], prior8[8], dprior8[8];
    framePrior(f, pr);
    for (int i = 0; i < 8; i++) { prior8[i] = pr[i]; dprior8[i] = f.state[i]; }  // getPriorZero() == 0
    marginalizeFrameHM(HM, bM, n, idx, prior8, dprior8);
  }
  // FullSystemMarginalize.cpp:L168-198: drop all observations of existing points in that frame (lastResiduals entries cleared); the frame
  // leaves, later frames shift down by one index (EnergyFunctional.cpp:L642-649)
  const int goneID = frameHessians[idx].frameID;
  for (PointHessian& p : points)
    for (int k = 0; k < 2; k++) if (p.lastResiduals_target[k] == goneID) p.lastResiduals_target[k] = -1;
  std::vector<PointFrameResidual> rkeep;
  rkeep.reserve(activeResiduals.size());
  for (const PointFrameResidual& r : activeResiduals)
    if (r.target != idx) { rkeep.push_back(r); if (rkeep.back().target > idx) rkeep.back().target--; }
  {  // the residual states and the optimised depths live on the device: pull them before the re-upload
    const int nr = (int)activeResiduals.size(), np = (int)points.size();
    std::vector<int32_t> ns(nr);
    std::vector<float> ne(nr);
    if (nr > 0 && fetchResidualOutputs(ns.data(), ne.data(), nullptr, nullptr)) {
      int w = 0;
      for (int i = 0; i < nr; i++)
        if (activeResiduals[i].target != idx) { rkeep[w].state_state = ns[i]; rkeep[w].state_energy = ne[i]; w++; }
    }
    if (np > 0) {
      std::vector<float> id(np);
      getIdepths(id.data());
      for (int i = 0; i < np; i++) { points[i].idepth = id[i]; points[i].idepth_zero = id[i]; points[i].idepth_backup = id[i]; }
    }
  }
  activeResiduals.swap(rkeep);
  for (PointHessian& p : points) if (p.host > idx) p.host--;
  frameHessians.erase(frameHessians.begin() + idx);
  if (!makeIDX()) return false;
  setAdjointsF();
  setPrecalcValues();
  return err_.empty();
}

void WindowBA::insertPoints(int n, const int* host, const float* u, const float* v, const float* idepth, const float* idepth_zero,
                            const float* color8, const float* weights8, const unsigned char* hasDepthPrior, const int* carry_from) {
  // The list replaces the window's point set (ordered by host frame, EnergyFunctional::allPoints).  Per-point statistics the reference keeps
  // on the PointHessian object (numGoodResiduals, maxRelBaseline, lastResiduals: HessianBlocks.h:L440-447) are RESET for every entry unless
  // carry_from[i] >= 0 names the point's index in the PREVIOUS list: newly activated points are hosted by older keyframes, so they land in
  // the middle of the list and every later point changes index.
  const std::vector<PointHessian> old(points);
  points.assign(n, PointHessian());
  for (int i = 0; i < n; i++) {
    PointHessian& p = points[i];
    if (carry_from && carry_from[i] >= 0 && carry_from[i] < (int)old.size()) {
      const PointHessian& q = old[carry_from[i]];
      p.numGoodResiduals = q.numGoodResiduals; p.maxRelBaseline = q.maxRelBaseline;
      for (int k = 0; k < 2; k++) { p.lastResiduals_target[k] = q.lastResiduals_target[k]; p.lastResiduals_state[k] = q.lastResiduals_state[k]; }
    }
    p.host = host[i]; p.u = u[i]; p.v = v[i]; p.idepth = idepth[i]; p.idepth_zero = idepth_zero ? idepth_zero[i] : idepth[i];
    p.idepth_backup = p.idepth; p.step = 0;
    for (int k = 0; k < 8; k++) { p.color[k] = color8[8 * i + k]; p.weights[k] = weights8[8 * i + k]; }
    p.hasDepthPrior = hasDepthPrior && hasDepthPrior[i];
    p.priorF = p.hasDepthPrior ? s.setting_idepthFixPrior * SCALE_IDEPTH * SCALE_IDEPTH : 0;  // EFPoint::takeData
  }
}
void WindowBA::insertResiduals(int n, const int* point, const int* target) {
  activeResiduals.resize(n);
  for (int i = 0; i < n; i++) { activeResiduals[i] = PointFrameResidual(); activeResiduals[i].point = point[i]; activeResiduals[i].target = target[i]; }
}

bool WindowBA::makeIDX() {
  err_.clear();  // per-call status: an earlier, already reported failure must not fail this call
  if (!ba_) return false;
  const int n = nf(), np = (int)points.size();
  std::vector<int> slots(n);
  for (int f = 0; f < n; f++) slots[f] = frameHessians[f].slot;
  if (dmv_ba_set_window(ba_, n, slots.data()) != DMV_OK) return fail("dmv_ba_set_window");
  dmv_ba_params prm;
  prm.huberTH = s.setting_huberTH; prm.outlierTHSumComponent = s.setting_outlierTHSumComponent;
  prm.affineOptModeA = s.setting_affineOptModeA; prm.affineOptModeB = s.setting_affineOptModeB;
  dmv_ba_set_params(ba_, &prm);
  // the share of every rank (round robin over the point index keeps the per-host-frame load even; one rank = everything)
  pts_of_rank_.assign(nranks_, std::vector<int>());
  local_of_point_.assign(np, 0);
  for (int i = 0; i < np; i++) { std::vector<int>& l = pts_of_rank_[i % nranks_]; local_of_point_[i] = (int)l.size(); l.push_back(i); }
  rebuildResidualMaps();
  const std::vector<int>& mine = pts_of_rank_[rank_];
  const std::vector<int>& mres = res_of_rank_[rank_];
  const int lp = (int)mine.size(), lr = (int)mres.size();
  std::vector<int32_t> host(lp);
  std::vector<float> u(lp), v(lp), id(lp), idz(lp), col((size_t)lp * 8), wgt((size_t)lp * 8), prior(lp);
  for (int i = 0; i < lp; i++) {
    const PointHessian& p = points[mine[i]];
    host[i] = p.host; u[i] = p.u; v[i] = p.v; id[i] = p.idepth; idz[i] = p.idepth_zero; prior[i] = p.priorF;
    for (int k = 0; k < 8; k++) { col[(size_t)8 * i + k] = p.color[k]; wgt[(size_t)8 * i + k] = p.weights[k]; }
  }
  if (dmv_ba_set_points(ba_, lp, host.data(), u.data(), v.data(), id.data(), idz.data(), col.data(), wgt.data(), prior.data()) != DMV_OK)
    return fail("dmv_ba_set_points");
  std::vector<int32_t> rp(lr), rt(lr), rs(lr);
  std::vector<float> re(lr);
  for (int i = 0; i < lr; i++) {
    const PointFrameResidual& r = activeResiduals[mres[i]];
    rp[i] = local_of_point_[r.point]; rt[i] = r.target; rs[i] = r.state_state; re[i] = r.state_energy;
  }
  if (dmv_ba_set_residuals(ba_, lr, rp.data(), rt.data(), rs.data(), re.data()) != DMV_OK) return fail("dmv_ba_set_residuals");
  const int N = 8 * n + CPARS;
  if ((int)HM.size() != N * N) { HM.assign((size_t)N * N, 0.0); bM.assign(N, 0.0); }
  have_pending_x_ = false;
  solved_since_makeIDX_ = false;
  return true;
}

void WindowBA::framePrior(const FrameHessian& f, double p[10]) const {  // HessianBlocks.h:L262-298 (getPrior)
  for (int i = 0; i < 10; i++) p[i] = 0;
  if (f.frameID == 0) {
    for (int i = 0; i < 3; i++) p[i] = s.setting_initialTransPrior;
    for (int i = 3; i < 6; i++) p[i] = s.setting_initialRotPrior;
    p[6] = s.setting_initialAffAPrior; p[7] = s.setting_initialAffBPrior;
  } else {
    p[6] = (s.setting_affineOptModeA < 0) ? s.setting_initialAffAPrior : s.setting_affineOptModeA;
    p[7] = (s.setting_affineOptModeB < 0) ? s.setting_initialAffBPrior : s.setting_affineOptModeB;
  }
  p[8] = s.setting_initialAffAPrior; p[9] = s.setting_initialAffBPrior;
  if (f.addCamPrior) {
    for (int i = 0; i < 3; i++) p[i] = s.setting_initialTransPrior;
    for (int i = 3; i < 6; i++) p[i] = s.setting_initialRotPrior;
  }
}

void WindowBA::setAdjointsF() {  // EnergyFunctional.cpp:L48-108
  const int n = nf();
  adHost.assign((size_t)n * n * 64, 0.0);
  adTarget.assign((size_t)n * n * 64, 0.0);
  for (int h = 0; h < n; h++)
    for (int t = 0; t < n; t++) {
      const FrameHessian& host = frameHessians[h];
      const FrameHessian& target = frameHessians[t];
      const SE3 hostToTarget = target.worldToCam_evalPT * host.worldToCam_evalPT.inverse();
      double Adj[36];
      hostToTarget.Adj(Adj);
      double* AH = &adHost[(size_t)(h + t * n) * 64];
      double* AT = &adTarget[(size_t)(h + t * n) * 64];
      for (int i = 0; i < 8; i++) { AH[i * 8 + i] = 1; AT[i * 8 + i] = 1; }
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) AH[i * 8 + j] = -Adj[j * 6 + i];
      double aff[2];
      AffLight::fromToVecExposure(host.ab_exposure, target.ab_exposure, host.aff_g2l_0(), target.aff_g2l_0(), aff);
      const float a0 = (float)aff[0];
      AT[6 * 8 + 6] = -a0; AH[6 * 8 + 6] = a0; AT[7 * 8 + 7] = -1; AH[7 * 8 + 7] = a0;
      const double sc[8] = {SCALE_XI_TRANS, SCALE_XI_TRANS, SCALE_XI_TRANS, SCALE_XI_ROT, SCALE_XI_ROT, SCALE_XI_ROT, SCALE_A, SCALE_B};
      for (int r = 0; r < 8; r++)
        for (int c = 0; c < 8; c++) { AH[r * 8 + c] *= sc[r]; AT[r * 8 + c] *= sc[r]; }
    }
  for (FrameHessian& f : frameHessians) {  // EFFrame::takeData
    double p[10];
    framePrior(f, p);
    for (int i = 0; i < 8; i++) f.prior[i] = p[i];
  }
  if (ba_ && dmv_ba_set_adjoints(ba_, adHost.data(), adTarget.data()) != DMV_OK) fail("dmv_ba_set_adjoints");
}

void WindowBA::setPrecalcValues() {  // FullSystem.cpp:L1670-1680 -> FrameFramePrecalc::set (HessianBlocks.cpp:L193-223) + setDeltaF
  const int n = nf();
  precalc.assign((size_t)n * n * DMV_PRECALC_FLOATS, 0.f);
  const float fx = Hcalib.value_scaledf[0], fy = Hcalib.value_scaledf[1], cx = Hcalib.value_scaledf[2], cy = Hcalib.value_scaledf[3];
  const float K[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1};
  float Ki[9];
  dmv::inv3_cofactor(K, Ki);  // K.inverse() with the reference's rounding (FrameFramePrecalc::set, HessianBlocks.cpp:L217)
  for (int h = 0; h < n; h++)
    for (int t = 0; t < n; t++) {
      const FrameHessian& host = frameHessians[h];
      const FrameHessian& target = frameHessians[t];
      float* q = &precalc[(size_t)(h * n + t) * DMV_PRECALC_FLOATS];
      const SE3 l0 = target.worldToCam_evalPT * host.worldToCam_evalPT.inverse();
      const SE3 l = target.PRE_worldToCam * host.PRE_camToWorld;
      float R[9], tt[3];
      for (int i = 0; i < 9; i++) { R[i] = (float)l.R[i]; q[12 + i] = (float)l0.R[i]; }
      for (int i = 0; i < 3; i++) { tt[i] = (float)l.t[i]; q[21 + i] = (float)l0.t[i]; }
      float KR[9];
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) KR[i * 3 + j] = K[i * 3] * R[j] + K[i * 3 + 1] * R[3 + j] + K[i * 3 + 2] * R[6 + j];
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) q[i * 3 + j] = KR[i * 3] * Ki[j] + KR[i * 3 + 1] * Ki[3 + j] + KR[i * 3 + 2] * Ki[6 + j];
      for (int i = 0; i < 3; i++) q[9 + i] = K[i * 3] * tt[0] + K[i * 3 + 1] * tt[1] + K[i * 3 + 2] * tt[2];
      double aff[2];
      AffLight::fromToVecExposure(host.ab_exposure, target.ab_exposure, host.aff_g2l(), target.aff_g2l(), aff);
      q[24] = (float)aff[0]; q[25] = (float)aff[1];
      q[26] = (float)host.aff_g2l_0().b;
    }
  for (FrameHessian& f : frameHessians)  // EnergyFunctional::setDeltaF (EnergyFunctional.cpp:L188-192)
    for (int i = 0; i < 8; i++) { f.delta[i] = f.state[i] - f.state_zero[i]; f.delta_prior[i] = f.state[i]; }
}

std::vector<float> WindowBA::adHTdeltaF() const {  // EnergyFunctional.cpp:L175-187
  const int n = nf();
  std::vector<float> out((size_t)n * n * 8, 0.f);
  for (int h = 0; h < n; h++)
    for (int t = 0; t < n; t++) {
      const int idx = h + t * n;
      const FrameHessian &fh = frameHessians[h], &ft = frameHessians[t];
      for (int c = 0; c < 8; c++) {
        float sacc = 0, tacc = 0;
        for (int k = 0; k < 8; k++) sacc += (float)(fh.state[k] - fh.state_zero[k]) * (float)adHost[(size_t)idx * 64 + k * 8 + c];
        for (int k = 0; k < 8; k++) tacc += (float)(ft.state[k] - ft.state_zero[k]) * (float)adTarget[(size_t)idx * 64 + k * 8 + c];
        out[(size_t)idx * 8 + c] = sacc + tacc;
      }
    }
  return out;
}

int WindowBA::marginalizePointsF(const std::vector<int>& toMargIn, const std::vector<int>& toDrop) {
  err_.clear();  // per-call status: an earlier, already reported failure must not fail this call
  if (!ba_) return -1;
  const int n = nf(), N = 8 * n + CPARS, np = (int)points.size();
  // FullSystem.cpp:L840-850: a candidate is marginalised only if its inverse depth is well constrained, otherwise dropped
  // PointHessian::idepth_hessian is written by AccumulatedSCHessian::addPoint only (AccumulatedSCHessian.cpp:L42-50), i.e. during the LAST
  // solveSystemF — not by the tail's linearizeAll(true): use the HdiF cached there (no solve yet: idepth_hessian = 0, candidates are dropped)
  std::vector<float> HdiF(np, 0.f);
  if (np > 0 && solved_since_makeIDX_ && !fetchPointFloats(1, HdiF.data())) { fail("dmv_ba_get_solve_HdiF"); return -1; }
  {  // the residual states live on the device (applyRes_Reductor commits there): pull them for the re-upload below
    const int nr = (int)activeResiduals.size();
    std::vector<int32_t> ns(nr);
    std::vector<float> ne(nr);
    if (nr > 0 && fetchResidualOutputs(ns.data(), ne.data(), nullptr, nullptr))
      for (int i = 0; i < nr; i++) { activeResiduals[i].state_state = ns[i]; activeResiduals[i].state_energy = ne[i]; }
  }
  std::vector<int32_t> toMarg;
  std::vector<char> erase(np, 0);
  for (int i : toDrop) if (i >= 0 && i < np) erase[i] = 1;
  for (int i : toMargIn) {
    if (i < 0 || i >= np) continue;
    erase[i] = 1;
    const float idepth_hessian = HdiF[i] > 0 ? 1.0f / HdiF[i] : 0.f;  // AccumulatedSCHessian.cpp:L42-50
    if (idepth_hessian > s.setting_minIdepthH_marg) toMarg.push_back(i);
  }
  int added = 0;
  if (!toMarg.empty()) {
    const std::vector<float> ad = adHTdeltaF();
    std::vector<double> M((size_t)N * N), Mb(N), Msc((size_t)N * N), Mbsc(N);
    dmv_ba_marg_args a;
    // sharded: every rank marginalises ITS flagged points (possibly none); M / Msc come back summed over the ranks
    std::vector<int32_t> toMargLocal;
    for (int32_t i : toMarg) if (i % nranks_ == rank_) toMargLocal.push_back(local_of_point_[i]);
    a.n = (int32_t)toMargLocal.size(); a.point = toMargLocal.data(); a.adHTdeltaF = ad.data();
    for (int i = 0; i < 4; i++) a.cDeltaF[i] = (float)Hcalib.value_minus_value_zero[i];
    a.idepthFixPriorMargFac = s.setting_idepthFixPriorMargFac;
    a.M = M.data(); a.Mb = Mb.data(); a.Msc = Msc.data(); a.Mbsc = Mbsc.data();
    int32_t nres = 0;
    a.resInM = &nres; a.ngoodRes = nullptr; a.res_toZeroF = nullptr; a.isLinearized = nullptr;
    if (dmv_ba_marginalize_points(ba_, &a) != DMV_OK) { fail("dmv_ba_marginalize_points"); return -1; }
    if ((int)HM.size() != N * N) { HM.assign((size_t)N * N, 0.0); bM.assign(N, 0.0); }
    for (size_t i = 0; i < (size_t)N * N; i++) HM[i] += (double)s.setting_margWeightFac * (M[i] - Msc[i]);   // EnergyFunctional.cpp:L729-730
    for (int i = 0; i < N; i++) bM[i] += (double)s.setting_margWeightFac * (Mb[i] - Mbsc[i]);
    added = nres;
    resInM += nres;
  }
  // EnergyFunctional::removePoint for every listed point: erase it and its residuals, renumber, upload the smaller window
  std::vector<int> newIndex(np, -1);
  std::vector<PointHessian> keep;
  keep.reserve(np);
  for (int i = 0; i < np; i++)
    if (!erase[i]) { newIndex[i] = (int)keep.size(); keep.push_back(points[i]); }
  // the device keeps the optimised depths: pull them before the re-upload
  if (np > 0) {
    std::vector<float> id(np);
    getIdepths(id.data());
    for (int i = 0; i < np; i++)
      if (newIndex[i] >= 0) { keep[newIndex[i]].idepth = id[i]; keep[newIndex[i]].idepth_zero = id[i]; keep[newIndex[i]].idepth_backup = id[i]; }
  }
  std::vector<PointFrameResidual> rkeep;
  rkeep.reserve(activeResiduals.size());
  for (const PointFrameResidual& r : activeResiduals)
    if (newIndex[r.point] >= 0) { rkeep.push_back(r); rkeep.back().point = newIndex[r.point]; }
  points.swap(keep);
  activeResiduals.swap(rkeep);
  if (!makeIDX()) return -1;
  setAdjointsF();  // makeIDX re-binds the window on the device: the adjoints go with it (FullSystem::makeKeyFrame calls ef->setAdjointsF next)
  return err_.empty() ? added : -1;
}

void WindowBA::fillState(dmv_ba_state* st, float* th) const {
  for (int i = 0; i < 4; i++) { st->calib[i] = Hcalib.value_scaledf[i]; st->calib[4 + i] = Hcalib.value_scaledi[i]; }
  for (int f = 0; f < nf(); f++) th[f] = frameHessians[f].frameEnergyTH;
  st->precalc = precalc.data();
  st->frameEnergyTH = th;
  st->idepth = nullptr;
  st->idepth_zero = nullptr;
}

double WindowBA::linearizeAll(bool fixLinearization) {
  // FullSystemOptimize.cpp:L150-218.  One C-ABI call: a pending resubstitute + point step (from the last solveSystemF /
  // doStepFromBackup) rides along, fused on the device.
  (void)fixLinearization;  // the applyRes / bookkeeping half of fixLinearization is syncResidualStates() + applyRes_Reductor()
  dmv_ba_state st;
  float th[DMV_MAX_FRAMES];
  fillState(&st, th);
  dmv_ba_lin_result r;
  const double* x = have_pending_x_ ? pending_x_.data() : nullptr;
  if (dmv_ba_gn_step(ba_, x, &st, &r, step_sums_) != DMV_OK) { fail("dmv_ba_gn_step"); return NAN; }
  have_pending_x_ = false;
  if (fixLinearization) applyRes_Reductor();  // linearizeAll_Reductor applies inside the map (L64); the energies read below are the same
  setNewFrameEnergyTH();
  if (!fixLinearization) return r.energy;
  // ---- FullSystemOptimize.cpp:L66-84 (per active residual: maxRelBaseline, numGoodResiduals; the others are collected) and L186-215
  syncResidualStates();
  const int n = nf(), np = (int)points.size(), nr = (int)activeResiduals.size();
  std::vector<float> id(np);
  if (np > 0) getIdepths(id.data());
  std::vector<int32_t> toRemove;
  for (int i = 0; i < nr; i++) {
    PointFrameResidual& res = activeResiduals[i];
    PointHessian& p = points[res.point];
    if (res.state_state != 1) { res.state_state = res.state_NewState; res.state_energy = res.state_NewEnergy; }  // applyRes; OOB is final (Residuals.cpp:L306-328)
    if (res.state_state == 0) {  // isActive(): state_NewState == IN
      // every residual is "new" in the reference (PointFrameResidual::isNew is never cleared)
      const float* q = &precalc[(size_t)(p.host * n + res.target) * 32];
      float inf3[3], ptp[3];
      for (int k = 0; k < 3; k++) inf3[k] = q[3 * k] * p.u + q[3 * k + 1] * p.v + q[3 * k + 2];
      for (int k = 0; k < 3; k++) ptp[k] = inf3[k] + q[9 + k] * id[res.point];
      const float dx = inf3[0] / inf3[2] - ptp[0] / ptp[2], dy = inf3[1] / inf3[2] - ptp[1] / ptp[2];
      const float relBS = 0.01 * std::sqrt(dx * dx + dy * dy);  // 0.01 = one pixel
      if (relBS > p.maxRelBaseline) p.maxRelBaseline = relBS;
      p.numGoodResiduals++;
    } else {
      toRemove.push_back(i);
    }
    const int tid = frameHessians[res.target].frameID;
    for (int k = 0; k < 2; k++)
      if (p.lastResiduals_target[k] == tid) { p.lastResiduals_state[k] = res.state_state; break; }
  }
  lastRemovedResiduals.assign(toRemove.begin(), toRemove.end());
  if (!toRemove.empty()) {
    std::vector<int32_t> dropLocal;   // the device holds this rank's residuals only
    for (int i : toRemove) if (activeResiduals[i].point % nranks_ == rank_) dropLocal.push_back(local_of_res_[i]);
    if (!dropLocal.empty() && dmv_ba_drop_residuals(ba_, (int)dropLocal.size(), dropLocal.data()) != DMV_OK) { fail("dmv_ba_drop_residuals"); return NAN; }
    std::vector<char> gone(nr, 0);
    for (int i : toRemove) {
      gone[i] = 1;
      PointHessian& p = points[activeResiduals[i].point];
      const int tid = frameHessians[activeResiduals[i].target].frameID;
      for (int k = 0; k < 2; k++)
        if (p.lastResiduals_target[k] == tid) { p.lastResiduals_target[k] = -1; break; }
    }
    int w = 0;
    for (int i = 0; i < nr; i++)
      if (!gone[i]) activeResiduals[w++] = activeResiduals[i];
    activeResiduals.resize(w);
    rebuildResidualMaps();   // the device kept the relative order of the remaining residuals: the same rule gives the same local indices
  }
  return r.energy;
}

double WindowBA::finishOptimize() {  // FullSystemOptimize.cpp:L591-609
  FrameHessian& newest = frameHessians.back();
  double newStateZero[10] = {0, 0, 0, 0, 0, 0, newest.state[6], newest.state[7], 0, 0};
  newest.worldToCam_evalPT = newest.PRE_worldToCam;  // FrameHessian::setEvalPT (HessianBlocks.h:L209-215)
  newest.setState(newStateZero);
  for (int i = 0; i < 10; i++) newest.state_zero[i] = newStateZero[i];
  setAdjointsF();
  setPrecalcValues();
  return linearizeAll(true);
}

void WindowBA::flagPointsForRemoval(const std::vector<int>& flaggedFrames, std::vector<int>* toMarg, std::vector<int>* toDrop) {
  // FullSystem.cpp:L785-879 (fhsToKeepPoints is always empty there: the loop at L795 never runs)
  const int n = nf(), np = (int)points.size();
  std::vector<char> flagged(n, 0);
  for (int f : flaggedFrames) if (f >= 0 && f < n) flagged[f] = 1;
  std::vector<float> id(np);
  if (np > 0) getIdepths(id.data());  // the optimised depths live on the device
  std::vector<int> nres(np, 0), visInToMarg(np, 0);
  for (const PointFrameResidual& r : activeResiduals) {
    nres[r.point]++;
    if (r.state_state == 0 && flagged[r.target]) visInToMarg[r.point]++;
  }
  for (int i = 0; i < np; i++) {
    const PointHessian& p = points[i];
    if (id[i] * SCALE_IDEPTH < s.setting_minIdepth || nres[i] == 0) { toDrop->push_back(i); continue; }
    // PointHessian::isOOB (HessianBlocks.h:L476-499)
    bool oob = false;
    if (nres[i] >= s.setting_minGoodActiveResForMarg && p.numGoodResiduals > s.setting_minGoodResForMarg + 10 &&
        nres[i] - visInToMarg[i] < s.setting_minGoodActiveResForMarg)
      oob = true;
    else if (p.lastResiduals_state[0] == 1) oob = true;
    else if (nres[i] < 2) oob = false;
    else if (p.lastResiduals_state[0] == 2 && p.lastResiduals_state[1] == 2) oob = true;
    if (!oob && !flagged[p.host]) continue;
    // PointHessian::isInlierNew (HessianBlocks.h:L502-506)
    const bool inlier = nres[i] >= s.setting_minGoodActiveResForMarg && p.numGoodResiduals >= s.setting_minGoodResForMarg;
    (inlier ? toMarg : toDrop)->push_back(i);
  }
}

void WindowBA::setNewFrameEnergyTH() {  // FullSystemOptimize.cpp:L96-149 (no IMU cap)
  std::vector<float> allResVec(points.size() + 1);
  int n = 0;
  if (nranks_ == 1) {
    if (dmv_ba_get_target_energies(ba_, nf() - 1, allResVec.data(), (int)allResVec.size(), &n) != DMV_OK) { fail("dmv_ba_get_target_energies"); return; }
  } else {  // the percentile is over the residuals of ALL ranks: gather state_NewEnergyWithOutlier, keep the evaluated ones that target the newest frame
    const int nr = (int)activeResiduals.size();
    std::vector<float> nw(nr);
    if (nr > 0 && !fetchResidualOutputs(nullptr, nullptr, nw.data(), nullptr)) { fail("dmv_ba_get_residual_outputs"); return; }
    allResVec.resize(nr + 1);
    for (int i = 0; i < nr; i++)
      if (activeResiduals[i].target == nf() - 1 && nw[i] >= 0) allResVec[n++] = nw[i];
  }
  FrameHessian& newFrame = frameHessians.back();
  if (n == 0) { newFrame.frameEnergyTH = 12 * 12 * patternNum; return; }
  allResVec.resize(n);
  const int nthIdx = (int)(s.setting_frameEnergyTHN * n);
  std::nth_element(allResVec.begin(), allResVec.begin() + nthIdx, allResVec.end());
  const float nthElement = sqrtf(allResVec[nthIdx]);
  float th = nthElement * s.setting_frameEnergyTHFacMedian;
  th = 26.0f * s.setting_frameEnergyTHConstWeight + th * (1 - s.setting_frameEnergyTHConstWeight);
  th = th * th;
  th *= s.setting_overallEnergyTHWeight * s.setting_overallEnergyTHWeight;
  newFrame.frameEnergyTH = th;
}

void WindowBA::applyRes_Reductor() {
  if (dmv_ba_apply_res(ba_) != DMV_OK) fail("dmv_ba_apply_res");
}

double WindowBA::calcLEnergyF_MT() {  // EnergyFunctional.cpp:L411-431 (no linearised residuals; idepth priors: deltaF == 0 in DM-VIO)
  double E = 0;
  for (const FrameHessian& f : frameHessians)
    for (int i = 0; i < 8; i++) E += f.delta_prior[i] * f.prior[i] * f.delta_prior[i];
  float ec = 0;
  for (int i = 0; i < 4; i++) { const float d = (float)Hcalib.value_minus_value_zero[i]; ec += d * s.setting_initialCalibHessian * d; }
  return E + ec;
}

double WindowBA::calcMEnergyF() {  // EnergyFunctional.cpp:L324-346
  const int n = nf(), N = 8 * n + CPARS;
  if ((int)HM.size() != N * N) return 0;
  std::vector<double> delta(N);
  for (int i = 0; i < 4; i++) delta[i] = (double)(float)Hcalib.value_minus_value_zero[i];
  for (int h = 0; h < n; h++) for (int i = 0; i < 8; i++) delta[CPARS + 8 * h + i] = frameHessians[h].delta[i];
  double v = 0;
  for (int i = 0; i < N; i++) {
    double sacc = 2 * bM[i];
    for (int j = 0; j < N; j++) sacc += HM[(size_t)i * N + j] * delta[j];
    v += delta[i] * sacc;
  }
  return v;
}

void WindowBA::solveSystemF(int iteration, double lambda) {
  // EnergyFunctional.cpp:L841-996, default solver mode (SOLVER_ORTHOGONALIZE_X_LATER), no-GTSAM branch (L971-973)
  const int n = nf(), N = 8 * n + CPARS;
  last_HA.assign((size_t)N * N, 0.0); last_bA.assign(N, 0.0); last_Hsc.assign((size_t)N * N, 0.0); last_bsc.assign(N, 0.0);
  if (dmv_ba_accumulate(ba_, last_HA.data(), last_bA.data(), last_Hsc.data(), last_bsc.data(), &resInA) != DMV_OK) { fail("dmv_ba_accumulate"); return; }
  solved_since_makeIDX_ = true;  // the device keeps EFPoint::HdiF of this accumulation (dmv_ba_get_solve_HdiF) for marginalizePointsF
  std::vector<double> delta(N);
  for (int i = 0; i < 4; i++) delta[i] = (double)(float)Hcalib.value_minus_value_zero[i];
  for (int h = 0; h < n; h++) for (int i = 0; i < 8; i++) delta[CPARS + 8 * h + i] = frameHessians[h].delta[i];
  std::vector<double> HFinal((size_t)N * N), bFinal(N);
  for (int i = 0; i < N; i++) {
    double bm = bM[i];
    for (int j = 0; j < N; j++) bm += HM[(size_t)i * N + j] * delta[j];
    for (int j = 0; j < N; j++) HFinal[(size_t)i * N + j] = HM[(size_t)i * N + j] + last_HA[(size_t)i * N + j];
    bFinal[i] = bm + last_bA[i] - last_bsc[i];
  }
  // accumulateLF_MT with no linearised residuals == priors (AccumulatedTopHessian.cpp:L292-302)
  for (int i = 0; i < 4; i++) { HFinal[(size_t)i * N + i] += s.setting_initialCalibHessian; bFinal[i] += s.setting_initialCalibHessian * delta[i]; }
  for (int h = 0; h < n; h++)
    for (int i = 0; i < 8; i++) {
      const int k = CPARS + 8 * h + i;
      HFinal[(size_t)k * N + k] += frameHessians[h].prior[i];
      bFinal[k] += frameHessians[h].prior[i] * frameHessians[h].delta_prior[i];
    }
  lastHS.assign((size_t)N * N, 0.0);
  for (size_t i = 0; i < (size_t)N * N; i++) lastHS[i] = HFinal[i] - last_Hsc[i];
  lastbS = bFinal;
  for (int i = 0; i < N; i++) HFinal[(size_t)i * N + i] *= (1 + lambda);
  for (size_t i = 0; i < (size_t)N * N; i++) HFinal[i] -= last_Hsc[i] * (1.0 / (1 + lambda));
  if (computeBAUpdate) {  // EnergyFunctional.cpp:L958-968: the host consumer (GTSAM + IMU factors in DM-VIO) solves; same H / b / x conventions
    lastX = computeBAUpdate(HFinal, bFinal, lambda, n, lastHS);
    if ((int)lastX.size() != N) { err_ = "computeBAUpdate returned a vector of the wrong size"; lastX.assign(N, 0.0); }
  } else {
    std::vector<double> SVecI(N), Hs((size_t)N * N), bs(N), xs(N);
    for (int i = 0; i < N; i++) SVecI[i] = 1.0 / std::sqrt(HFinal[(size_t)i * N + i] + 10);
    for (int i = 0; i < N; i++) {
      for (int j = 0; j < N; j++) Hs[(size_t)i * N + j] = SVecI[i] * HFinal[(size_t)i * N + j] * SVecI[j];
      bs[i] = SVecI[i] * bFinal[i];
    }
    ldlt_solve(N, Hs.data(), bs.data(), xs.data());
    lastX.resize(N);
    for (int i = 0; i < N; i++) lastX[i] = SVecI[i] * xs[i];
  }
  if (iteration >= 2 && s.setting_orthogonalizeXLater) {  // L980-984: project x off the 7 gauge directions (6 pose + 1 scale)
    // the nullspaces depend on the evaluation points only (fixed during optimize): basis cached, keyed by the evaluation points themselves
    std::vector<double> key((size_t)12 * n);
    for (int h = 0; h < n; h++) {
      const SE3& T = frameHessians[h].worldToCam_evalPT;
      for (int i = 0; i < 9; i++) key[(size_t)12 * h + i] = T.R[i];
      for (int i = 0; i < 3; i++) key[(size_t)12 * h + 9 + i] = T.t[i];
    }
    if (key != gauge_key_) {
      std::vector<SE3> evalPT(n);
      for (int h = 0; h < n; h++) evalPT[h] = frameHessians[h].worldToCam_evalPT;
      gauge_U_ = gaugeBasis(windowNullspaces(evalPT, SCALE_XI_TRANS, SCALE_XI_ROT), s.setting_solverModeDelta);
      gauge_key_.swap(key);
    }
    gaugeProject(lastX, gauge_U_);
  }
  // resubstituteF_MT (EnergyFunctional.cpp:L267-289): frame / calib steps here, the per-point half is fused into the next linearizeAll
  for (int i = 0; i < 4; i++) Hcalib.step[i] = -lastX[i];
  for (int h = 0; h < n; h++) {
    for (int i = 0; i < 8; i++) frameHessians[h].step[i] = -lastX[CPARS + 8 * h + i];
    frameHessians[h].step[8] = frameHessians[h].step[9] = 0;
  }
  pending_x_ = lastX;
  have_pending_x_ = true;
}

void WindowBA::backupState() {  // FullSystemOptimize.cpp:L322-370 (no momentum)
  for (int i = 0; i < 4; i++) Hcalib.value_backup[i] = Hcalib.value[i];
  for (FrameHessian& f : frameHessians) for (int i = 0; i < 10; i++) f.state_backup[i] = f.state[i];
  dmv_ba_backup_points(ba_);
}

bool WindowBA::doStepFromBackup() {  // FullSystemOptimize.cpp:L224-317, stepfac = 1
  float sumA = 0, sumB = 0, sumT = 0, sumR = 0;
  double nv[4];
  for (int i = 0; i < 4; i++) nv[i] = Hcalib.value_backup[i] + Hcalib.step[i];
  Hcalib.setValue(nv);
  for (FrameHessian& f : frameHessians) {
    double ns[10];
    for (int i = 0; i < 10; i++) ns[i] = f.state_backup[i] + f.step[i];
    f.setState(ns);
    sumA += f.step[6] * f.step[6];
    sumB += f.step[7] * f.step[7];
    sumT += f.step[0] * f.step[0] + f.step[1] * f.step[1] + f.step[2] * f.step[2];
    sumR += f.step[3] * f.step[3] + f.step[4] * f.step[4] + f.step[5] * f.step[5];
  }
  const float nfr = (float)frameHessians.size();
  canbreak_frames_[0] = sumA / nfr; canbreak_frames_[1] = sumB / nfr; canbreak_frames_[2] = sumR / nfr; canbreak_frames_[3] = sumT / nfr;
  setPrecalcValues();
  return true;  // the convergence test needs sum |idepth_backup| of the points: evaluated after the fused linearizeAll
}

void WindowBA::loadSateBackup() {  // FullSystemOptimize.cpp:L371-388
  Hcalib.setValue(Hcalib.value_backup);
  for (FrameHessian& f : frameHessians) f.setState(f.state_backup);
  dmv_ba_restore_points(ba_);
  have_pending_x_ = false;
  setPrecalcValues();
}

int WindowBA::optimize(int mnumOptIts, std::vector<double>* energyLog, bool finish) {
  err_.clear();  // per-call status: an earlier, already reported failure must not fail this call
  // FullSystemOptimize.cpp:L417-647 without IMU / GTSAM / logging
  if (nf() < 2) return 0;
  if (nf() < 3) mnumOptIts = 20;
  if (nf() < 4) mnumOptIts = 15;
  // activeResiduals = every residual that is not linearised, each reset with resetOOB (L431-448)
  if (dmv_ba_reset_oob(ba_) != DMV_OK) { fail("dmv_ba_reset_oob"); return 0; }
  double lastEnergy = linearizeAll(false);
  double lastEnergyL = calcLEnergyF_MT();
  double lastEnergyM = calcMEnergyF();
  applyRes_Reductor();
  if (energyLog) energyLog->push_back(lastEnergy);
  double lambda = 1e-5;
  const double minLambda = 1e-5;
  int numIterations = 0;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
  for (int iteration = 0; iteration < mnumOptIts; iteration++) {
    const auto t0 = now();
    backupState();
    solveSystemF(iteration, lambda);
    const auto t1 = now();
    doStepFromBackup();
    const auto t2 = now();
    const double newEnergy = linearizeAll(false);
    const auto t3 = now();
    if (!std::isfinite(newEnergy) && !err_.empty()) return numIterations;
    const double newEnergyL = calcLEnergyF_MT();
    const double newEnergyM = calcMEnergyF();
    const auto t4 = now();
    profile_us[0] += us(t0, t1); profile_us[1] += us(t1, t2); profile_us[2] += us(t2, t3); profile_us[3] += us(t3, t4); profile_us[4] += 1;
    // doStepFromBackup's return value (L311-314), now that the device reported sum |idepth_backup|
    const float sumNID = step_sums_[2] > 0 ? (float)(step_sums_[1] / step_sums_[2]) : 0.f;
    bool canbreak = sqrtf(canbreak_frames_[0]) < 0.0005 * s.setting_thOptIterations && sqrtf(canbreak_frames_[1]) < 0.00005 * s.setting_thOptIterations &&
                    sqrtf(canbreak_frames_[2]) < 0.00005 * s.setting_thOptIterations &&
                    sqrtf(canbreak_frames_[3]) * sumNID < 0.00005 * s.setting_thOptIterations;
    if (newEnergy + newEnergyL + newEnergyM < lastEnergy + lastEnergyL + lastEnergyM) {
      applyRes_Reductor();
      lastEnergy = newEnergy; lastEnergyL = newEnergyL; lastEnergyM = newEnergyM;
      if (acceptBAUpdate) acceptBAUpdate(lastEnergy);
      lambda *= 0.25;
      lambda = std::max(lambda, minLambda);
    } else {
      // FullSystemOptimize.cpp:L574-580: restore, then RE-LINEARISE at the restored state: the new baseline energy (and frameEnergyTH) come from
      // that evaluation, which runs with the threshold the rejected linearisation produced.  One more fused launch; nothing is committed, the
      // committed linearisation of the accepted state stays what solveSystemF reads.
      loadSateBackup();
      lastEnergy = linearizeAll(false);
      lastEnergyL = calcLEnergyF_MT();
      lastEnergyM = calcMEnergyF();
      lambda *= 1e2;
    }
    if (!std::isfinite(lastEnergy) && !err_.empty()) return numIterations;  // a failed device call (err_ says which), not a diverged energy
    if (energyLog) energyLog->push_back(lastEnergy);
    numIterations++;
    if (canbreak && iteration >= s.setting_minOptIterations) break;
  }
  lastEnergyTotal = lastEnergy;
  if (finish) lastEnergyTotal = finishOptimize();
  return numIterations;
}

void WindowBA::syncResidualStates() {
  const int nr = (int)activeResiduals.size();
  std::vector<int32_t> ns(nr);
  std::vector<float> ne(nr), nw(nr), cp((size_t)nr * 3);
  if (!fetchResidualOutputs(ns.data(), ne.data(), nw.data(), cp.data())) { fail("dmv_ba_get_residual_outputs"); return; }
  for (int i = 0; i < nr; i++) {
    PointFrameResidual& r = activeResiduals[i];
    r.state_NewState = ns[i]; r.state_NewEnergy = ne[i]; r.state_NewEnergyWithOutlier = nw[i];
    for (int k = 0; k < 3; k++) r.centerProjectedTo[k] = cp[(size_t)3 * i + k];
  }
}
void WindowBA::getIdepths(float* idepth) { fetchPointFloats(0, idepth); }

int WindowBA::coarseTrackingRefInputs(float* Ku, float* Kv, float* nid, float* HdiF, int32_t* point, int cap) {
  err_.clear();
  const int np = (int)points.size(), newest = nf() - 1;
  if (newest < 0 || np == 0) return 0;
  std::vector<float> hdi(np);
  if (!fetchPointFloats(1, hdi.data())) { fail("dmv_ba_get_solve_HdiF"); return -1; }
  std::vector<int> res_of_point(np, -1);   // the point's residual into the newest frame
  std::vector<char> alive(np, 0);          // the point still has a residual (FullSystem::removeOutliers keeps it)
  for (int i = 0; i < (int)activeResiduals.size(); i++) {
    alive[activeResiduals[i].point] = 1;
    if (activeResiduals[i].target == newest) res_of_point[activeResiduals[i].point] = i;
  }
  const int tid = frameHessians[newest].frameID;
  int n = 0;
  for (int b = 0; b < np;) {
    int e = b;
    while (e < np && points[e].host == points[b].host) e++;
    for (int p : dmv::remove_outliers_order(b, e, alive)) {
      const PointHessian& ph = points[p];
      if (ph.lastResiduals_target[0] != tid || ph.lastResiduals_state[0] != 0 || res_of_point[p] < 0) continue;
      if (n == cap) { err_ = "coarseTrackingRefInputs: more than " + std::to_string(cap) + " entries"; return -1; }
      const PointFrameResidual& r = activeResiduals[res_of_point[p]];
      Ku[n] = r.centerProjectedTo[0]; Kv[n] = r.centerProjectedTo[1]; nid[n] = r.centerProjectedTo[2]; HdiF[n] = hdi[p];
      if (point) point[n] = p;
      n++;
    }
    b = e;
  }
  return n;
}

// ---- sharding
void WindowBA::rebuildResidualMaps() {
  const int nr = (int)activeResiduals.size();
  res_of_rank_.assign(nranks_, std::vector<int>());
  local_of_res_.assign(nr, 0);
  for (int i = 0; i < nr; i++) { std::vector<int>& l = res_of_rank_[activeResiduals[i].point % nranks_]; local_of_res_[i] = (int)l.size(); l.push_back(i); }
}
bool WindowBA::setSharding(int rank, int nranks) {
  if (nranks < 1 || rank < 0 || rank >= nranks) return fail("setSharding: bad rank / nranks");
  rank_ = rank; nranks_ = nranks;
  return true;
}
bool WindowBA::p2pExport(void* h64) { return dmv_ba_p2p_export(ba_, h64) == DMV_OK || fail("dmv_ba_p2p_export"); }
bool WindowBA::p2pImport(const void* handles) { return dmv_ba_p2p_import(ba_, nranks_, rank_, handles) == DMV_OK || fail("dmv_ba_p2p_import"); }
bool WindowBA::p2pSetup() {
  if (nranks_ == 1) return true;
  if (!allgather) return fail("sharded WindowBA needs the allgather callback");
  unsigned char mine[64];
  std::vector<unsigned char> all((size_t)64 * nranks_);
  if (!p2pExport(mine)) return false;
  allgather(mine, all.data(), 64);
  return p2pImport(all.data());
}
bool WindowBA::commInit(const void* uid) { return dmv_ba_comm_init(ba_, nranks_, rank_, uid) == DMV_OK || fail("dmv_ba_comm_init"); }

// every rank contributes its rows (local order), padded to the largest share; the result is scattered to global indices
template <class T> bool WindowBA::gatherRows(const std::vector<std::vector<int>>& of_rank, const T* local, int width, T* global) {
  if (nranks_ == 1) {
    const std::vector<int>& l = of_rank[0];
    for (size_t i = 0; i < l.size(); i++) for (int k = 0; k < width; k++) global[(size_t)l[i] * width + k] = local[i * width + k];
    return true;
  }
  if (!allgather) return fail("sharded WindowBA needs the allgather callback");
  size_t mx = 0;
  for (const std::vector<int>& l : of_rank) mx = std::max(mx, l.size());
  if (mx == 0) return true;
  std::vector<T> send(mx * width, T(0)), recv(mx * width * nranks_);
  std::copy(local, local + of_rank[rank_].size() * width, send.begin());
  allgather(send.data(), recv.data(), sizeof(T) * mx * width);
  for (int r = 0; r < nranks_; r++) {
    const std::vector<int>& l = of_rank[r];
    const T* src = recv.data() + (size_t)r * mx * width;
    for (size_t i = 0; i < l.size(); i++) for (int k = 0; k < width; k++) global[(size_t)l[i] * width + k] = src[i * width + k];
  }
  return true;
}

bool WindowBA::fetchResidualOutputs(int32_t* newState, float* newEnergy, float* newEnergyWithOutlier, float* cpt3) {
  if (res_of_rank_.empty()) return false;
  const int lr = (int)res_of_rank_[rank_].size();
  std::vector<int32_t> ns(lr);
  std::vector<float> ne(lr), nw(lr), cp((size_t)lr * 3);
  if (lr > 0 && dmv_ba_get_residual_outputs(ba_, newState ? ns.data() : nullptr, newEnergy ? ne.data() : nullptr, newEnergyWithOutlier ? nw.data() : nullptr,
                                             cpt3 ? cp.data() : nullptr, nullptr) != DMV_OK)
    return false;
  bool ok = true;
  if (newState) ok = gatherRows(res_of_rank_, ns.data(), 1, newState) && ok;
  if (newEnergy) ok = gatherRows(res_of_rank_, ne.data(), 1, newEnergy) && ok;
  if (newEnergyWithOutlier) ok = gatherRows(res_of_rank_, nw.data(), 1, newEnergyWithOutlier) && ok;
  if (cpt3) ok = gatherRows(res_of_rank_, cp.data(), 3, cpt3) && ok;
  return ok;
}

bool WindowBA::fetchPointFloats(int what, float* out) {
  if (pts_of_rank_.empty()) return false;
  const int lp = (int)pts_of_rank_[rank_].size();
  std::vector<float> loc(lp);
  if (lp > 0) {
    const int rc = what == 0 ? dmv_ba_get_idepth(ba_, loc.data(), nullptr) : dmv_ba_get_solve_HdiF(ba_, loc.data());
    if (rc != DMV_OK) return false;
  }
  return gatherRows(pts_of_rank_, loc.data(), 1, out);
}
void WindowBA::getFrameStates(double* st) const {
  for (int f = 0; f < nf(); f++) for (int i = 0; i < 10; i++) st[10 * f + i] = frameHessians[f].state[i];
}
double WindowBA::lastGpuMs() const { float ms[4] = {0, 0, 0, 0}; dmv_ba_last_timing(ba_, ms); return ms[0]; }

}  // namespace dmvio_b200
