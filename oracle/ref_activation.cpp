// TEST INFRASTRUCTURE ONLY — C entry points that drive the REFERENCE's own compiled CoarseDistanceMap (FullSystem/CoarseTracker.cpp: makeK,
// makeDistanceMap, addIntoDistFinal) for tests/test_ref_pin_activation.py and tests/golden/make_golden_activation.py.  The selection loop
// of FullSystem::activatePointsMT (FullSystem.cpp:L642-717) is a FullSystem member, which cannot be compiled here, so it is mirrored line for
// line around the reference's objects, as ref_harness.cpp's ref_win_activate mirrors optimizeImmaturePoint.  Built by ref_build.sh
// into a library of its own, linked with the reference objects it compiles and ref_harness.o.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "FullSystem/CoarseTracker.h"
#include "FullSystem/HessianBlocks.h"
#include "FullSystem/ImmaturePoint.h"
#include "util/globalCalib.h"
#include "util/settings.h"

using namespace dso;

extern "C" {

// A window of nf frames with poses worldToCam (R row-major, t; PRE_worldToCam / PRE_camToWorld as setEvalPT leaves them), active points
// (u, v, idepth_scaled, host) and immature points grouped by host.  Runs makeK, makeDistanceMap and the selection loop; writes the actions
// (0 keep, 1 delete, 2 optimise), toOptimize as indexes, the final fwdWarpedIDDistFinal ((w/2)*(h/2)) and the per-frame [KRKi | Kt] the
// loop computed (nf*12, the frame newest's entry included).  Returns the size of toOptimize.
int ref_act_select(int w, int h, const double K[4], int nf, int newest, const double* R9, const double* t3, const uint8_t* flagged, int na,
                   const float* au, const float* av, const float* aid, const int32_t* ah, const int32_t* off, const float* u, const float* v,
                   const float* idmin, const float* idmax, const int32_t* status, const float* interval, const float* quality, const float* type,
                   float currentMinActDist, float minTraceQuality, int32_t* action, int32_t* opt, float* map, float* tab12) {
  Eigen::Matrix3f Km;
  Km.setZero();
  Km(0, 0) = (float)K[0]; Km(1, 1) = (float)K[1]; Km(0, 2) = (float)K[2]; Km(1, 2) = (float)K[3]; Km(2, 2) = 1.f;
  setGlobalCalib(w, h, Km);
  setting_minTraceQuality = minTraceQuality;
  CalibHessian Hcalib;
  std::vector<Eigen::Vector3f> dI((size_t)w * h, Eigen::Vector3f::Zero());   // the constructors below sample colours at (8, 8)
  std::vector<FrameHessian*> frameHessians;
  for (int f = 0; f < nf; f++) {
    FrameHessian* fh = new FrameHessian();
    for (int l = 0; l < PYR_LEVELS; l++) { fh->dIp[l] = 0; fh->absSquaredGrad[l] = 0; }
    fh->dI = dI.data();
    fh->idx = f;
    fh->flaggedForMarginalization = flagged[f] != 0;
    Mat33 Rm; Vec3 tv;
    for (int i = 0; i < 3; i++) { tv[i] = t3[3 * f + i]; for (int j = 0; j < 3; j++) Rm(i, j) = R9[9 * f + 3 * i + j]; }
    fh->PRE_worldToCam = SE3(Rm, tv);
    fh->PRE_camToWorld = fh->PRE_worldToCam.inverse();
    frameHessians.push_back(fh);
  }
  for (int p = 0; p < na; p++) {
    ImmaturePoint ipt(8, 8, frameHessians[ah[p]], 1.f, &Hcalib);
    ipt.idepth_min = ipt.idepth_max = 1.f;
    PointHessian* ph = new PointHessian(&ipt, &Hcalib);
    ph->u = au[p]; ph->v = av[p];
    ph->setIdepthScaled(aid[p]);
    ph->setPointStatus(PointHessian::ACTIVE);
    frameHessians[ah[p]]->pointHessians.push_back(ph);
  }
  std::vector<ImmaturePoint*> all;
  for (int f = 0; f < nf; f++)
    for (int i = off[f]; i < off[f + 1]; i++) {
      ImmaturePoint* ip = new ImmaturePoint(8, 8, frameHessians[f], type[i], &Hcalib);
      ip->u = u[i]; ip->v = v[i]; ip->idepth_min = idmin[i]; ip->idepth_max = idmax[i];
      ip->lastTraceStatus = (ImmaturePointStatus)status[i];
      ip->lastTracePixelInterval = interval[i];
      ip->quality = quality[i];
      frameHessians[f]->immaturePoints.push_back(ip);
      all.push_back(ip);
      action[i] = 0;
    }
  CoarseDistanceMap* coarseDistanceMap = new CoarseDistanceMap(w, h);
  FrameHessian* newestHs = frameHessians[newest];

  // FullSystem.cpp:L644-717, with `delete ph` recorded as action 1 and toOptimize as indexes
  coarseDistanceMap->makeK(&Hcalib);
  coarseDistanceMap->makeDistanceMap(frameHessians, newestHs);
  std::vector<ImmaturePoint*> toOptimize; toOptimize.reserve(20000);
  int nopt = 0;
  for (FrameHessian* host : frameHessians) {
    SE3 fhToNew = newestHs->PRE_worldToCam * host->PRE_camToWorld;
    Mat33f KRKi = (coarseDistanceMap->K[1] * fhToNew.rotationMatrix().cast<float>() * coarseDistanceMap->Ki[0]);
    Vec3f Kt = (coarseDistanceMap->K[1] * fhToNew.translation().cast<float>());
    for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) tab12[12 * host->idx + 3 * r + c] = KRKi(r, c); tab12[12 * host->idx + 9 + r] = Kt[r]; }
    if (host == newestHs) continue;
    for (unsigned int i = 0; i < host->immaturePoints.size(); i += 1) {
      ImmaturePoint* ph = host->immaturePoints[i];
      const int gi = off[host->idx] + (int)i;
      ph->idxInImmaturePoints = i;
      if (!std::isfinite(ph->idepth_max) || ph->lastTraceStatus == IPS_OUTLIER) { action[gi] = 1; continue; }
      bool canActivate = (ph->lastTraceStatus == IPS_GOOD || ph->lastTraceStatus == IPS_SKIPPED || ph->lastTraceStatus == IPS_BADCONDITION ||
                          ph->lastTraceStatus == IPS_OOB) && ph->lastTracePixelInterval < 8 && ph->quality > setting_minTraceQuality &&
                         (ph->idepth_max + ph->idepth_min) > 0;
      if (!canActivate) {
        if (ph->host->flaggedForMarginalization || ph->lastTraceStatus == IPS_OOB) action[gi] = 1;
        continue;
      }
      Vec3f ptp = KRKi * Vec3f(ph->u, ph->v, 1) + Kt * (0.5f * (ph->idepth_max + ph->idepth_min));
      int u = ptp[0] / ptp[2] + 0.5f;
      int v = ptp[1] / ptp[2] + 0.5f;
      if ((u > 0 && v > 0 && u < wG[1] && v < hG[1])) {
        float dist = coarseDistanceMap->fwdWarpedIDDistFinal[u + wG[1] * v] + (ptp[0] - floorf((float)(ptp[0])));
        if (dist >= currentMinActDist * ph->my_type) {
          coarseDistanceMap->addIntoDistFinal(u, v);
          toOptimize.push_back(ph);
          action[gi] = 2;
          opt[nopt++] = gi;
        }
      } else {
        action[gi] = 1;
      }
    }
  }
  std::memcpy(map, coarseDistanceMap->fwdWarpedIDDistFinal, sizeof(float) * wG[1] * hG[1]);
  delete coarseDistanceMap;
  for (FrameHessian* fh : frameHessians) delete fh;   // deletes its pointHessians and immaturePoints
  return nopt;
}

// the reference's addIntoDistFinal for each cell of a list in order, on a map ((w/2)*(h/2)) given as input
void ref_act_grow(int w, int h, float* map, int nadd, const int32_t* add_xy) {
  Eigen::Matrix3f Km;
  Km.setZero();
  Km(0, 0) = 100.f; Km(1, 1) = 100.f; Km(0, 2) = w / 2; Km(1, 2) = h / 2; Km(2, 2) = 1.f;
  setGlobalCalib(w, h, Km);
  CalibHessian Hcalib;
  CoarseDistanceMap* cdm = new CoarseDistanceMap(w, h);
  cdm->makeK(&Hcalib);
  const int w1 = w / 2, h1 = h / 2;
  std::memcpy(cdm->fwdWarpedIDDistFinal, map, sizeof(float) * w1 * h1);
  for (int s = 0; s < nadd; s++) cdm->addIntoDistFinal(add_xy[2 * s], add_xy[2 * s + 1]);
  std::memcpy(map, cdm->fwdWarpedIDDistFinal, sizeof(float) * w1 * h1);
  delete cdm;
}
}
