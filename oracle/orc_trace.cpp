// TEST INFRASTRUCTURE ONLY — see orc_trace.h.
#include "orc_trace.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <utility>

namespace orc {

static const int patternP[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};  // util/settings.cpp:L296 (pattern 8)

// util/globalFuncs.h:L203-226 getInterpolatedElement33BiLin: [interpolated I, dx of the bilinear patch, dy of the bilinear patch]
static inline void interp33BiLin(const float* mat, float x, float y, int width, float out[3]) {
  const int ix = (int)x, iy = (int)y;
  const float* bp = mat + 3 * (ix + iy * width);
  const float tl = bp[0], tr = bp[3], bl = bp[3 * width], br = bp[3 * width + 3];
  const float dx = x - ix, dy = y - iy;
  const float topInt = dx * tr + (1 - dx) * tl;
  const float botInt = dx * br + (1 - dx) * bl;
  const float leftInt = dy * bl + (1 - dy) * tl;
  const float rightInt = dy * br + (1 - dy) * tr;
  out[0] = dx * rightInt + (1 - dx) * leftInt;
  out[1] = rightInt - leftInt;
  out[2] = botInt - topInt;
}
// util/globalFuncs.h:L160-175
static inline float interp31(const float* mat, float x, float y, int width) {
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = mat + 3 * (ix + iy * width);
  return dxdy * bp[3 * (1 + width)] + (dy - dxdy) * bp[3 * width] + (dx - dxdy) * bp[3] + (1 - dx - dy + dxdy) * bp[0];
}
// util/globalFuncs.h:L103-118
static inline void interp33(const float* mat, float x, float y, int width, float out[3]) {
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = mat + 3 * (ix + iy * width);
  for (int c = 0; c < 3; c++)
    out[c] = dxdy * bp[3 * (1 + width) + c] + (dy - dxdy) * bp[3 * width + c] + (dx - dxdy) * bp[3 + c] + (1 - dx - dy + dxdy) * bp[c];
}

bool initImmature(ImmaturePt& p, const float* dI, int w, int u, int v, const TraceSettings& s) {  // ImmaturePoint.cpp:L34-63
  p.u = (float)u; p.v = (float)v;
  p.idepth_min = 0; p.idepth_max = NAN; p.lastTraceStatus = IPS_UNINITIALIZED;
  p.gradH[0] = p.gradH[1] = p.gradH[2] = p.gradH[3] = 0;
  p.quality = 10000;
  p.lastTraceUV[0] = p.lastTraceUV[1] = 0; p.lastTracePixelInterval = 0;
  for (int idx = 0; idx < 8; idx++) {
    float ptc[3];
    interp33BiLin(dI, (float)(u + patternP[idx][0]), (float)(v + patternP[idx][1]), w, ptc);
    p.color[idx] = ptc[0];
    if (!std::isfinite(p.color[idx])) { p.energyTH = NAN; return false; }
    p.gradH[0] += ptc[1] * ptc[1]; p.gradH[1] += ptc[1] * ptc[2]; p.gradH[2] += ptc[2] * ptc[1]; p.gradH[3] += ptc[2] * ptc[2];
    p.weights[idx] = sqrtf(s.outlierTHSumComponent / (s.outlierTHSumComponent + (ptc[1] * ptc[1] + ptc[2] * ptc[2])));
  }
  p.energyTH = 8 * s.outlierTH;
  p.energyTH *= s.overallEnergyTHWeight * s.overallEnergyTHWeight;
  return true;
}

int traceOn(ImmaturePt& P, const float* dI, int w, int h, const float KRKi[9], const float Kt[3], const float aff[2], const TraceSettings& s,
            int32_t* diag) {
  int32_t scratch[IPD_N];
  int32_t* D = diag ? diag : scratch;
  for (int k = 0; k < IPD_N; k++) D[k] = 0;
  D[IPD_BEST_IDX] = -1; D[IPD_MAX_TIED_IDX] = -1;
  if (P.lastTraceStatus == IPS_OOB) { D[IPD_EXIT] = IPX_STICKY_OOB; return P.lastTraceStatus; }  // L79
  const float maxPixSearch = (w + h) * s.maxPixSearch;
  auto oob = [&](int exit) { D[IPD_EXIT] = exit; P.lastTraceUV[0] = -1; P.lastTraceUV[1] = -1; P.lastTracePixelInterval = 0; return P.lastTraceStatus = IPS_OOB; };
  // ---- project min and max (L98-176)
  float pr[3];
  for (int i = 0; i < 3; i++) pr[i] = (KRKi[3 * i] * P.u + KRKi[3 * i + 1] * P.v) + KRKi[3 * i + 2] * 1.0f;
  float ptpMin[3];
  for (int i = 0; i < 3; i++) ptpMin[i] = pr[i] + Kt[i] * P.idepth_min;
  const float uMin = ptpMin[0] / ptpMin[2], vMin = ptpMin[1] / ptpMin[2];
  int maxRotPatX = 0, maxRotPatY = 0;
  float rot[8][2];
  for (int idx = 0; idx < 8; idx++) {
    const float px = (float)patternP[idx][0], py = (float)patternP[idx][1];
    rot[idx][0] = KRKi[0] * px + KRKi[1] * py;
    rot[idx][1] = KRKi[3] * px + KRKi[4] * py;
    const int absX = (int)std::abs(rot[idx][0]), absY = (int)std::abs(rot[idx][1]);
    maxRotPatX = std::max(absX, maxRotPatX);
    maxRotPatY = std::max(absY, maxRotPatY);
  }
  const int boundU = std::max(4, maxRotPatX + 2), boundV = std::max(4, maxRotPatY + 2);
  if (!(uMin > boundU && vMin > boundV && uMin < w - boundU - 1 && vMin < h - boundV - 1)) return oob(IPX_UMIN_OOB);
  float dist, uMax, vMax, ptpMax[3];
  if (std::isfinite(P.idepth_max)) {
    for (int i = 0; i < 3; i++) ptpMax[i] = pr[i] + Kt[i] * P.idepth_max;
    uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
    if (!(uMax > boundU && vMax > boundV && uMax < w - boundU - 1 && vMax < h - boundV - 1)) return oob(IPX_UMAX_OOB);
    dist = (uMin - uMax) * (uMin - uMax) + (vMin - vMax) * (vMin - vMax);
    dist = sqrtf(dist);
    if (dist < s.trace_slackInterval) {
      D[IPD_EXIT] = IPX_SKIPPED;
      P.lastTraceUV[0] = (uMax + uMin) * 0.5f; P.lastTraceUV[1] = (vMax + vMin) * 0.5f;
      P.lastTracePixelInterval = dist;
      return P.lastTraceStatus = IPS_SKIPPED;
    }
  } else {
    dist = maxPixSearch;
    for (int i = 0; i < 3; i++) ptpMax[i] = pr[i] + Kt[i] * 0.01f;
    uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
    const float ddx = uMax - uMin, ddy = vMax - vMin;
    const float d = 1.0f / sqrtf(ddx * ddx + ddy * ddy);
    uMax = uMin + dist * ddx * d;
    vMax = vMin + dist * ddy * d;
    if (!(uMax > boundU && vMax > boundV && uMax < w - boundU - 1 && vMax < h - boundV - 1)) return oob(IPX_UMAX_OOB);
  }
  if (!(P.idepth_min < 0 || (ptpMin[2] > 0.75 && ptpMin[2] < 1.5))) return oob(IPX_DEPTH_RANGE);  // L179-185 (double literals: compared in double)
  // ---- error bounds (L188-206)
  float dx = s.trace_stepsize * (uMax - uMin);
  float dy = s.trace_stepsize * (vMax - vMin);
  const float* g = P.gradH;
  const float a = (dx * g[0] + dy * g[2]) * dx + (dx * g[1] + dy * g[3]) * dy;
  const float b = (dy * g[0] + (-dx) * g[2]) * dy + (dy * g[1] + (-dx) * g[3]) * (-dx);
  float errorInPixel = 0.2f + 0.2f * (a + b) / a;
  if (errorInPixel * s.trace_minImprovementFactor > dist && std::isfinite(P.idepth_max)) {
    D[IPD_EXIT] = IPX_BADCONDITION;
    P.lastTraceUV[0] = (uMax + uMin) * 0.5f; P.lastTraceUV[1] = (vMax + vMin) * 0.5f;
    P.lastTracePixelInterval = dist;
    return P.lastTraceStatus = IPS_BADCONDITION;
  }
  if (errorInPixel > 10) errorInPixel = 10;
  // ---- discrete search (L210-277)
  dx /= dist;
  dy /= dist;
  if (dist > maxPixSearch) {
    uMax = uMin + maxPixSearch * dx;
    vMax = vMin + maxPixSearch * dy;
    dist = maxPixSearch;
  }
  int numSteps = 1.9999f + dist / s.trace_stepsize;
  const float randShift = uMin * 1000 - floorf(uMin * 1000);
  float ptx = uMin - randShift * dx;
  float pty = vMin - randShift * dy;
  if (!std::isfinite(dx) || !std::isfinite(dy)) { D[IPD_EXIT] = IPX_NONFINITE_DIR; P.lastTracePixelInterval = 0; P.lastTraceUV[0] = -1; P.lastTraceUV[1] = -1; return P.lastTraceStatus = IPS_OOB; }
  float errors[100];
  float bestU = 0, bestV = 0, bestEnergy = 1e10;
  int bestIdx = -1;
  if (numSteps >= 100) numSteps = 99;
  for (int i = 0; i < numSteps; i++) {
    float energy = 0;
    for (int idx = 0; idx < 8; idx++) {
      const float hitColor = interp31(dI, (float)(ptx + rot[idx][0]), (float)(pty + rot[idx][1]), w);
      if (!std::isfinite(hitColor)) { energy += 1e5; D[IPD_NONFINITE_SEARCH]++; continue; }
      const float residual = hitColor - (float)(aff[0] * P.color[idx] + aff[1]);
      const float hw = fabs(residual) < s.huberTH ? 1 : s.huberTH / fabs(residual);
      energy += hw * residual * residual * (2 - hw);
    }
    errors[i] = energy;
    if (energy < bestEnergy) { bestU = ptx; bestV = pty; bestEnergy = energy; bestIdx = i; }
    ptx += dx;
    pty += dy;
  }
  D[IPD_NUM_STEPS] = numSteps;
  D[IPD_BEST_IDX] = bestIdx;
  for (int i = 0; i < numSteps; i++)
    if (bestIdx >= 0 && errors[i] == bestEnergy) { D[IPD_N_TIED]++; D[IPD_MAX_TIED_IDX] = i; }
  float secondBest = 1e10;
  for (int i = 0; i < numSteps; i++)
    if ((i < bestIdx - s.minTraceTestRadius || i > bestIdx + s.minTraceTestRadius) && errors[i] < secondBest) secondBest = errors[i];
  const float newQuality = secondBest / bestEnergy;
  if (newQuality < P.quality || numSteps > 10) P.quality = newQuality;
  // ---- GN refinement along the line (L280-353)
  float uBak = bestU, vBak = bestV, gnstepsize = 1, stepBack = 0;
  if (s.trace_GNIterations > 0) bestEnergy = 1e5;
  for (int it = 0; it < s.trace_GNIterations; it++) {
    D[IPD_GN_ITS]++;
    float H = 1, bb = 0, energy = 0;
    for (int idx = 0; idx < 8; idx++) {
      const float posU = (float)(bestU + rot[idx][0]);
      const float posV = (float)(bestV + rot[idx][1]);
      if (posU < 0 || posV < 0 || posU >= w - 1 || posV >= h - 1) return oob(IPX_GN_OOB);
      float hit[3];
      interp33(dI, posU, posV, w, hit);
      if (!std::isfinite((float)hit[0])) { energy += 1e5; D[IPD_NONFINITE_GN]++; continue; }
      const float residual = hit[0] - (aff[0] * P.color[idx] + aff[1]);
      const float dResdDist = dx * hit[1] + dy * hit[2];
      const float hw = fabs(residual) < s.huberTH ? 1 : s.huberTH / fabs(residual);
      H += hw * dResdDist * dResdDist;
      bb += hw * residual * dResdDist;
      energy += P.weights[idx] * P.weights[idx] * hw * residual * residual * (2 - hw);
    }
    if (energy > bestEnergy) {
      stepBack *= 0.5;
      bestU = uBak + stepBack * dx;
      bestV = vBak + stepBack * dy;
    } else {
      float step = -gnstepsize * bb / H;
      if (step < -0.5) step = -0.5;
      else if (step > 0.5) step = 0.5;
      if (!std::isfinite(step)) step = 0;
      uBak = bestU;
      vBak = bestV;
      stepBack = step;
      bestU += step * dx;
      bestV += step * dy;
      bestEnergy = energy;
    }
    if (fabsf(stepBack) < s.trace_GNThreshold) { D[IPD_GN_BREAK] = 1; break; }
  }
  // ---- energy-based outlier (L360-376)
  if (!(bestEnergy < P.energyTH * s.trace_extraSlackOnTH)) {
    P.lastTracePixelInterval = 0;
    P.lastTraceUV[0] = -1; P.lastTraceUV[1] = -1;
    if (P.lastTraceStatus == IPS_OUTLIER) { D[IPD_EXIT] = IPX_OUTLIER_TWICE; return P.lastTraceStatus = IPS_OOB; }
    D[IPD_EXIT] = IPX_OUTLIER;
    return P.lastTraceStatus = IPS_OUTLIER;
  }
  // ---- new interval (L380-402)
  if (dx * dx > dy * dy) {
    P.idepth_min = (pr[2] * (bestU - errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU - errorInPixel * dx));
    P.idepth_max = (pr[2] * (bestU + errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU + errorInPixel * dx));
  } else {
    P.idepth_min = (pr[2] * (bestV - errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV - errorInPixel * dy));
    P.idepth_max = (pr[2] * (bestV + errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV + errorInPixel * dy));
  }
  if (P.idepth_min > P.idepth_max) std::swap(P.idepth_min, P.idepth_max);
  if (!std::isfinite(P.idepth_min) || !std::isfinite(P.idepth_max) || (P.idepth_max < 0)) {
    D[IPD_EXIT] = IPX_BAD_INTERVAL;
    P.lastTracePixelInterval = 0;
    P.lastTraceUV[0] = -1; P.lastTraceUV[1] = -1;
    return P.lastTraceStatus = IPS_OUTLIER;
  }
  D[IPD_EXIT] = IPX_GOOD;
  P.lastTracePixelInterval = 2 * errorInPixel;
  P.lastTraceUV[0] = bestU; P.lastTraceUV[1] = bestV;
  return P.lastTraceStatus = IPS_GOOD;
}

}  // namespace orc

using namespace orc;
extern "C" {
int orc_ip_init(int n, const float* dI, int w, int h, const int32_t* u, const int32_t* v, float* color8, float* weights8, float* gradH4, float* energyTH,
                uint8_t* ok) {
  (void)h;
  TraceSettings s;
  int good = 0;
  for (int i = 0; i < n; i++) {
    ImmaturePt p;
    const bool o = initImmature(p, dI, w, u[i], v[i], s);
    std::memcpy(color8 + 8 * i, p.color, 32); std::memcpy(weights8 + 8 * i, p.weights, 32); std::memcpy(gradH4 + 4 * i, p.gradH, 16);
    energyTH[i] = p.energyTH;
    ok[i] = o; good += o;
  }
  return good;
}
static void ip_trace_all(int n, const float* dI, int w, int h, const float* KRKi, const float* Kt, const float* aff, const float* u, const float* v,
                         const float* color8, const float* weights8, const float* gradH4, const float* energyTH, float* idepth_min, float* idepth_max,
                         float* quality, int32_t* status, float* uv2, float* interval, int32_t* diag) {
  TraceSettings s;
  for (int i = 0; i < n; i++) {
    ImmaturePt p;
    p.u = u[i]; p.v = v[i];
    std::memcpy(p.color, color8 + 8 * i, 32); std::memcpy(p.weights, weights8 + 8 * i, 32); std::memcpy(p.gradH, gradH4 + 4 * i, 16);
    p.energyTH = energyTH[i]; p.idepth_min = idepth_min[i]; p.idepth_max = idepth_max[i]; p.quality = quality[i];
    p.lastTraceStatus = status[i]; p.lastTraceUV[0] = uv2[2 * i]; p.lastTraceUV[1] = uv2[2 * i + 1]; p.lastTracePixelInterval = interval[i];
    traceOn(p, dI, w, h, KRKi, Kt, aff, s, diag ? diag + (size_t)IPD_N * i : nullptr);
    idepth_min[i] = p.idepth_min; idepth_max[i] = p.idepth_max; quality[i] = p.quality; status[i] = p.lastTraceStatus;
    uv2[2 * i] = p.lastTraceUV[0]; uv2[2 * i + 1] = p.lastTraceUV[1]; interval[i] = p.lastTracePixelInterval;
  }
}
void orc_ip_trace(int n, const float* dI, int w, int h, const float* KRKi, const float* Kt, const float* aff, const float* u, const float* v,
                  const float* color8, const float* weights8, const float* gradH4, const float* energyTH, float* idepth_min, float* idepth_max,
                  float* quality, int32_t* status, float* uv2, float* interval) {
  ip_trace_all(n, dI, w, h, KRKi, Kt, aff, u, v, color8, weights8, gradH4, energyTH, idepth_min, idepth_max, quality, status, uv2, interval, nullptr);
}
void orc_ip_trace_diag(int n, const float* dI, int w, int h, const float* KRKi, const float* Kt, const float* aff, const float* u, const float* v,
                       const float* color8, const float* weights8, const float* gradH4, const float* energyTH, float* idepth_min, float* idepth_max,
                       float* quality, int32_t* status, float* uv2, float* interval, int32_t* diag) {
  ip_trace_all(n, dI, w, h, KRKi, Kt, aff, u, v, color8, weights8, gradH4, energyTH, idepth_min, idepth_max, quality, status, uv2, interval, diag);
}
}

// =====================================================================================================================
// Point activation (SURVEY.md §8f-2, second half): FullSystem::optimizeImmaturePoint (FullSystem/FullSystemOptPoint.cpp:L51-205) driving
// ImmaturePoint::linearizeResidual (FullSystem/ImmaturePoint.cpp:L498-565) with projectPoint / derive_idepth
// (FullSystem/ResidualProjections.h:L36-87).  Pinned: linearizeResidual is the reference's compiled code in oracle/_ref; the 60-line
// driver lives in FullSystem (not compiled there) and is mirrored by the harness.
// =====================================================================================================================
namespace orc {

struct ActFrameTables {
  int nf, w, h;
  float fxl, fyl, cxl, cyl, fxli, fyli;
  const float* const* dI;  // nf level-0 planes [I,dx,dy]
  const float* RT;         // [h*nf+t][12]: PRE_RTll row-major, PRE_tTll
  const float* aff;        // [h*nf+t][2]:  PRE_aff_mode
};
struct TmpRes { int state_state, state_NewState; double state_energy, state_NewEnergy; int target; };
enum { RS_IN = 0, RS_OOB = 1, RS_OUTLIER = 2 };

// ImmaturePoint::linearizeResidual
static double linearizeResidual(const ActFrameTables& F, int host, float pu, float pv, const float* color, const float* weights, float energyTH,
                                const float huberTH, const float outlierTHSlack, TmpRes* tmp, float& Hdd, float& bd, float idepth) {
  if (tmp->state_state == RS_OOB) { tmp->state_NewState = RS_OOB; return tmp->state_energy; }
  const float* R = F.RT + (size_t)(host * F.nf + tmp->target) * 12;
  const float* t = R + 9;
  const float* affLL = F.aff + (size_t)(host * F.nf + tmp->target) * 2;
  const float* dIl = F.dI[tmp->target];
  const float wM3G = (float)(F.w - 3), hM3G = (float)(F.h - 3);
  float energyLeft = 0;
  for (int idx = 0; idx < 8; idx++) {
    const int dx = patternP[idx][0], dy = patternP[idx][1];
    // projectPoint (ResidualProjections.h:L62-87)
    const float K0 = (pu + dx - F.cxl) * F.fxli, K1 = (pv + dy - F.cyl) * F.fyli, K2 = 1;
    float ptp[3];
    for (int i = 0; i < 3; i++) ptp[i] = ((R[3 * i] * K0 + R[3 * i + 1] * K1) + R[3 * i + 2] * K2) + t[i] * idepth;
    const float drescale = 1.0f / ptp[2];
    if (!(drescale > 0)) { tmp->state_NewState = RS_OOB; return tmp->state_energy; }
    const float u = ptp[0] * drescale, v = ptp[1] * drescale;
    const float Ku = u * F.fxl + F.cxl, Kv = v * F.fyl + F.cyl;
    if (!(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G)) { tmp->state_NewState = RS_OOB; return tmp->state_energy; }
    float hit[3];
    interp33(dIl, Ku, Kv, F.w, hit);
    if (!std::isfinite((float)hit[0])) { tmp->state_NewState = RS_OOB; return tmp->state_energy; }
    const float residual = hit[0] - (affLL[0] * color[idx] + affLL[1]);
    float hw = fabsf(residual) < huberTH ? 1 : huberTH / fabsf(residual);
    energyLeft += weights[idx] * weights[idx] * hw * residual * residual * (2 - hw);
    const float dxInterp = hit[1] * F.fxl, dyInterp = hit[2] * F.fyl;
    const float d_idepth = (dxInterp * drescale * (t[0] - t[2] * u) + dyInterp * drescale * (t[1] - t[2] * v)) * 1.0f;  // derive_idepth, SCALE_IDEPTH = 1
    hw *= weights[idx] * weights[idx];
    Hdd += (hw * d_idepth) * d_idepth;
    bd += (hw * residual) * d_idepth;
  }
  if (energyLeft > energyTH * outlierTHSlack) { energyLeft = energyTH * outlierTHSlack; tmp->state_NewState = RS_OUTLIER; }
  else tmp->state_NewState = RS_IN;
  tmp->state_NewEnergy = energyLeft;
  return energyLeft;
}

// FullSystem::optimizeImmaturePoint: returns 1 (activated), 0 (not well constrained: skipped), -1 (outlier / NaN depth)
static int optimizeImmaturePoint(const ActFrameTables& F, int host, float pu, float pv, const float* color, const float* weights, float energyTH,
                                 float idepth_min, float idepth_max, int minObs, float huberTH, float minIdepthH_act, int GNIts, float* idepth_out,
                                 int32_t* res_state /* nf */) {
  TmpRes res[16];
  int nres = 0;
  for (int f = 0; f < F.nf; f++) {
    res_state[f] = 255;
    if (f == host) continue;
    res[nres].state_NewEnergy = res[nres].state_energy = 0;
    res[nres].state_NewState = RS_OUTLIER;
    res[nres].state_state = RS_IN;
    res[nres].target = f;
    nres++;
  }
  float lastEnergy = 0, lastHdd = 0, lastbd = 0;
  float currentIdepth = (idepth_max + idepth_min) * 0.5f;
  for (int i = 0; i < nres; i++) {
    lastEnergy += linearizeResidual(F, host, pu, pv, color, weights, energyTH, huberTH, 1000, res + i, lastHdd, lastbd, currentIdepth);
    res[i].state_state = res[i].state_NewState;
    res[i].state_energy = res[i].state_NewEnergy;
  }
  *idepth_out = currentIdepth;
  if (!std::isfinite(lastEnergy) || lastHdd < minIdepthH_act) return 0;
  float lambda = 0.1;
  for (int iteration = 0; iteration < GNIts; iteration++) {
    float H = lastHdd;
    H *= 1 + lambda;
    const float step = (1.0 / H) * lastbd;
    const float newIdepth = currentIdepth - step;
    float newHdd = 0, newbd = 0, newEnergy = 0;
    for (int i = 0; i < nres; i++) newEnergy += linearizeResidual(F, host, pu, pv, color, weights, energyTH, huberTH, 1, res + i, newHdd, newbd, newIdepth);
    if (!std::isfinite(lastEnergy) || newHdd < minIdepthH_act) { *idepth_out = currentIdepth; return 0; }
    if (newEnergy < lastEnergy) {
      currentIdepth = newIdepth;
      lastHdd = newHdd; lastbd = newbd; lastEnergy = newEnergy;
      for (int i = 0; i < nres; i++) { res[i].state_state = res[i].state_NewState; res[i].state_energy = res[i].state_NewEnergy; }
      lambda *= 0.5;
    } else {
      lambda *= 5;
    }
    if (fabsf(step) < 0.0001 * currentIdepth) break;
  }
  *idepth_out = currentIdepth;
  if (!std::isfinite(currentIdepth)) return -1;
  int numGoodRes = 0;
  for (int i = 0; i < nres; i++) {
    res_state[res[i].target] = res[i].state_state;
    if (res[i].state_state == RS_IN) numGoodRes++;
  }
  if (numGoodRes < minObs) return -1;
  if (!std::isfinite(energyTH)) return -1;
  return 1;
}

}  // namespace orc

extern "C" void orc_ip_activate(int n, int nf, int w, int h, const float calib6[6], const float* dI_all, const float* RT, const float* aff,
                                const int32_t* host, const float* u, const float* v, const float* color8, const float* weights8, const float* energyTH,
                                const float* idepth_min, const float* idepth_max, int minObs, float huberTH, int32_t* status, float* idepth,
                                int32_t* res_state) {
  orc::ActFrameTables F;
  F.nf = nf; F.w = w; F.h = h;
  F.fxl = calib6[0]; F.fyl = calib6[1]; F.cxl = calib6[2]; F.cyl = calib6[3]; F.fxli = calib6[4]; F.fyli = calib6[5];
  const float* planes[16];
  for (int f = 0; f < nf; f++) planes[f] = dI_all + (size_t)f * w * h * 3;
  F.dI = planes; F.RT = RT; F.aff = aff;
  for (int i = 0; i < n; i++)
    status[i] = orc::optimizeImmaturePoint(F, host[i], u[i], v[i], color8 + 8 * i, weights8 + 8 * i, energyTH[i], idepth_min[i], idepth_max[i], minObs, huberTH,
                                           100.f, 3, idepth + i, res_state + (size_t)i * nf);
}
