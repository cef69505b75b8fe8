// ip_trace_kernel — ImmaturePoint::traceOn (reference FullSystem/ImmaturePoint.cpp:L77-437) for all immature points of one host
// frame against the newest frame, as FullSystem::traceNewCoarse does on every tracked frame (FullSystem.cpp:L541-584; SURVEY.md §8f-2).
//
// One warp per point (see ip_trace_kernel): the search positions, the best / second-best selection and the 8 pattern samples of the
// refinement are spread over the lanes.  The new frame's level-0 plane is the float4 texel plane already resident in the coarse-tracker
// handle (uploaded once per frame for tracking).
//
// THIS TRANSLATION UNIT IS COMPILED WITH -fmad=false: every expression keeps the reference's operation order and rounding (no FMA
// contraction; IEEE division and sqrt are nvcc's defaults), so the integer decisions (best step, status, GN accept/reject) and the
// float outputs are bit-identical to the reference's CPU code — tests/test_gpu_trace.py asserts equality, not a tolerance.
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include "ip_trace.h"
#include <cuda_runtime.h>
#include <math.h>

namespace dmv {

__device__ __constant__ int c_ip_pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};

// util/globalFuncs.h:L160-175 getInterpolatedElement31
__device__ __forceinline__ float ip_interp31(const float4* __restrict__ mat, float x, float y, int width) {
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float4* bp = mat + ix + iy * width;
  return dxdy * __ldg(bp + 1 + width).x + (dy - dxdy) * __ldg(bp + width).x + (dx - dxdy) * __ldg(bp + 1).x + (1 - dx - dy + dxdy) * __ldg(bp).x;
}
// util/globalFuncs.h:L103-118 getInterpolatedElement33
__device__ __forceinline__ void ip_interp33(const float4* __restrict__ mat, float x, float y, int width, float out[3]) {
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float4* bp = mat + ix + iy * width;
  const float4 br = __ldg(bp + 1 + width), bl = __ldg(bp + width), tr = __ldg(bp + 1), tl = __ldg(bp);
  out[0] = dxdy * br.x + (dy - dxdy) * bl.x + (dx - dxdy) * tr.x + (1 - dx - dy + dxdy) * tl.x;
  out[1] = dxdy * br.y + (dy - dxdy) * bl.y + (dx - dxdy) * tr.y + (1 - dx - dy + dxdy) * tl.y;
  out[2] = dxdy * br.z + (dy - dxdy) * bl.z + (dx - dxdy) * tr.z + (1 - dx - dy + dxdy) * tl.z;
}

// One WARP per immature point.  The reference walks the epipolar segment step by step (<= 99 positions x 8 bilinear samples) and keeps the
// best and second-best energies; here the positions are dealt to the 32 lanes (lane L takes steps L, L+32, L+64, L+96: at most 4 rounds
// instead of 99), the winner is a warp arg-min with the sequential scan's tie rule (lowest step index), the 8 pattern samples of a
// Gauss-Newton refinement step sit in 8 lanes and are folded in pattern order.  What is order-dependent in floating point is kept in the
// reference's order: the step positions are formed by the same chain of additions, every energy sums its 8 samples sequentially, the GN sums
// add the per-sample terms in index order.  All scalar bookkeeping is computed redundantly by every lane (identical values, no broadcast).
__device__ __forceinline__ float ip_step_energy(const IPTraceArgs& A, const float aff0, const float aff1, const float4* __restrict__ dI, const float (&rot)[8][2],
                                                const float (&color)[8], float ptx, float pty, int w) {
  float energy = 0;
#pragma unroll
  for (int idx = 0; idx < 8; idx++) {
    const float hitColor = ip_interp31(dI, (float)(ptx + rot[idx][0]), (float)(pty + rot[idx][1]), w);
    if (!isfinite(hitColor)) { energy = (float)((double)energy + 1e5); continue; }
    const float residual = hitColor - (float)(aff0 * color[idx] + aff1);
    const float hw = fabsf(residual) < A.s.huberTH ? 1 : A.s.huberTH / fabsf(residual);
    energy += hw * residual * residual * (2 - hw);
  }
  return energy;
}

__global__ void __launch_bounds__(128) ip_trace_kernel(const __grid_constant__ IPTraceArgs A) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // warp = point
  const int lane = threadIdx.x & 31;
  if (i >= A.n) return;
  const dmv_ip_settings& s = A.s;
  const int w = A.w, h = A.h;
  const float4* __restrict__ dI = A.img;
  const float* tabp = A.tab ? A.tab + 14 * A.set_of[i] : A.KRKi;   // KRKi | Kt | aff are contiguous in both cases
  const float* KRKi = tabp;
  const float* Kt = tabp + 9;
  const float aff0 = tabp[12], aff1 = tabp[13];
  const int status = A.status[i];
  if (status == 1) return;  // IPS_OOB stays OOB (ImmaturePoint.cpp:L79)
  const float u = A.u[i], v = A.v[i];
  float idepth_min = A.idepth_min[i], idepth_max = A.idepth_max[i];
  float color[8];
#pragma unroll
  for (int k = 0; k < 8; k++) color[k] = A.color[8 * i + k];
  const float g0 = A.gradH[4 * i], g1 = A.gradH[4 * i + 1], g2 = A.gradH[4 * i + 2], g3 = A.gradH[4 * i + 3];
  const float energyTH = A.energyTH[i];
#define IP_RETURN(st, ux, uy, itv) do { if (lane == 0) { A.status[i] = (st); A.uv[2 * i] = (ux); A.uv[2 * i + 1] = (uy); A.interval[i] = (itv); } return; } while (0)
  const float maxPixSearch = (w + h) * s.maxPixSearch;
  // ---- the segment [idepth_min, idepth_max] in the new frame (L98-185)
  float pr[3], ptpMin[3];
#pragma unroll
  for (int k = 0; k < 3; k++) pr[k] = (KRKi[3 * k] * u + KRKi[3 * k + 1] * v) + KRKi[3 * k + 2] * 1.0f;
#pragma unroll
  for (int k = 0; k < 3; k++) ptpMin[k] = pr[k] + Kt[k] * idepth_min;
  const float uMin = ptpMin[0] / ptpMin[2], vMin = ptpMin[1] / ptpMin[2];
  int maxRotPatX = 0, maxRotPatY = 0;
  float rot[8][2];
#pragma unroll
  for (int idx = 0; idx < 8; idx++) {
    const float px = (float)c_ip_pattern[idx][0], py = (float)c_ip_pattern[idx][1];
    rot[idx][0] = KRKi[0] * px + KRKi[1] * py;
    rot[idx][1] = KRKi[3] * px + KRKi[4] * py;
    maxRotPatX = max((int)fabsf(rot[idx][0]), maxRotPatX);
    maxRotPatY = max((int)fabsf(rot[idx][1]), maxRotPatY);
  }
  const int boundU = max(4, maxRotPatX + 2), boundV = max(4, maxRotPatY + 2);
  auto inside = [&](float x, float y) { return x > boundU && y > boundV && x < w - boundU - 1 && y < h - boundV - 1; };
  if (!inside(uMin, vMin)) IP_RETURN(1, -1.f, -1.f, 0.f);
  float dist, uMax, vMax, ptpMax[3];
  if (isfinite(idepth_max)) {
#pragma unroll
    for (int k = 0; k < 3; k++) ptpMax[k] = pr[k] + Kt[k] * idepth_max;
    uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
    if (!inside(uMax, vMax)) IP_RETURN(1, -1.f, -1.f, 0.f);
    dist = (uMin - uMax) * (uMin - uMax) + (vMin - vMax) * (vMin - vMax);
    dist = sqrtf(dist);
    if (dist < s.trace_slackInterval) IP_RETURN(3, (uMax + uMin) * 0.5f, (vMax + vMin) * 0.5f, dist);
  } else {
    dist = maxPixSearch;
#pragma unroll
    for (int k = 0; k < 3; k++) ptpMax[k] = pr[k] + Kt[k] * 0.01f;
    uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
    const float ddx = uMax - uMin, ddy = vMax - vMin;
    const float d = 1.0f / sqrtf(ddx * ddx + ddy * ddy);
    uMax = uMin + dist * ddx * d;
    vMax = vMin + dist * ddy * d;
    if (!inside(uMax, vMax)) IP_RETURN(1, -1.f, -1.f, 0.f);
  }
  if (!(idepth_min < 0 || ((double)ptpMin[2] > 0.75 && (double)ptpMin[2] < 1.5))) IP_RETURN(1, -1.f, -1.f, 0.f);
  // ---- error bound along / across the gradient (L188-206)
  float dx = s.trace_stepsize * (uMax - uMin);
  float dy = s.trace_stepsize * (vMax - vMin);
  const float a = (dx * g0 + dy * g2) * dx + (dx * g1 + dy * g3) * dy;
  const float b = (dy * g0 + (-dx) * g2) * dy + (dy * g1 + (-dx) * g3) * (-dx);
  float errorInPixel = 0.2f + 0.2f * (a + b) / a;
  if (errorInPixel * s.trace_minImprovementFactor > dist && isfinite(idepth_max)) IP_RETURN(4, (uMax + uMin) * 0.5f, (vMax + vMin) * 0.5f, dist);
  if (errorInPixel > 10) errorInPixel = 10;
  // ---- discrete search (L210-277), positions dealt to the lanes
  dx /= dist;
  dy /= dist;
  if (dist > maxPixSearch) {
    uMax = uMin + maxPixSearch * dx;
    vMax = vMin + maxPixSearch * dy;
    dist = maxPixSearch;
  }
  int numSteps = 1.9999f + dist / s.trace_stepsize;
  const float randShift = uMin * 1000 - floorf(uMin * 1000);
  if (!isfinite(dx) || !isfinite(dy)) IP_RETURN(1, -1.f, -1.f, 0.f);
  if (numSteps >= 100) numSteps = 99;
  float posx[4], posy[4];   // positions of steps lane + 32 k: the reference's running sums ptx += dx, reproduced addition by addition
  {
    float ptx = uMin - randShift * dx, pty = vMin - randShift * dy;
#pragma unroll
    for (int k = 0; k < 4; k++) { posx[k] = 0.f; posy[k] = 0.f; }
    for (int st = 0; st < numSteps; st++) {
      if ((st & 31) == lane) {
        const int k = st >> 5;
        if (k == 0) { posx[0] = ptx; posy[0] = pty; } else if (k == 1) { posx[1] = ptx; posy[1] = pty; }
        else if (k == 2) { posx[2] = ptx; posy[2] = pty; } else { posx[3] = ptx; posy[3] = pty; }
      }
      ptx += dx;
      pty += dy;
    }
  }
  float err[4];
  float bestEnergy = 1e10f, bestU = 0, bestV = 0;
  int bestIdx = -1;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int st = lane + 32 * k;
    err[k] = 0.f;
    if (32 * k < numSteps) {            // warp-uniform round
      if (st < numSteps) {
        err[k] = ip_step_energy(A, aff0, aff1, dI, rot, color, posx[k], posy[k], w);
        if (err[k] < bestEnergy) { bestU = posx[k]; bestV = posy[k]; bestEnergy = err[k]; bestIdx = st; }   // a lane's steps ascend: first minimum wins
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {   // warp arg-min with the sequential scan's rule: smaller energy, on equal energies the smaller step index
    const float oE = __shfl_xor_sync(0xffffffffu, bestEnergy, m), oU = __shfl_xor_sync(0xffffffffu, bestU, m), oV = __shfl_xor_sync(0xffffffffu, bestV, m);
    const int oI = __shfl_xor_sync(0xffffffffu, bestIdx, m);
    if (oI >= 0 && (bestIdx < 0 || oE < bestEnergy || (oE == bestEnergy && oI < bestIdx))) { bestEnergy = oE; bestU = oU; bestV = oV; bestIdx = oI; }
  }
  float secondBest = 1e10f;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int st = lane + 32 * k;
    if (st < numSteps && (st < bestIdx - s.minTraceTestRadius || st > bestIdx + s.minTraceTestRadius) && err[k] < secondBest) secondBest = err[k];
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const float o = __shfl_xor_sync(0xffffffffu, secondBest, m);
    if (o < secondBest) secondBest = o;
  }
  const float newQuality = secondBest / bestEnergy;
  float quality = A.quality[i];
  if (newQuality < quality || numSteps > 10) quality = newQuality;
  __syncwarp();
  if (lane == 0) A.quality[i] = quality;
  // ---- Gauss-Newton refinement along the line (L280-353): lane idx < 8 samples pattern pixel idx, the sums fold in pattern order
  float uBak = bestU, vBak = bestV, stepBack = 0;
  const float gnstepsize = 1;
  if (s.trace_GNIterations > 0) bestEnergy = 1e5f;
  const int idx8 = lane & 7;
  const float wgt = A.weights[8 * i + idx8];
  float colL = 0.f, rx = 0.f, ry = 0.f;
#pragma unroll
  for (int k = 0; k < 8; k++) if (k == idx8) { colL = color[k]; rx = rot[k][0]; ry = rot[k][1]; }
  for (int it = 0; it < s.trace_GNIterations; it++) {
    const float posU = (float)(bestU + rx), posV = (float)(bestV + ry);
    const bool oob = (posU < 0 || posV < 0 || posU >= w - 1 || posV >= h - 1);
    if (__any_sync(0xffffffffu, oob)) IP_RETURN(1, -1.f, -1.f, 0.f);
    float hit[3];
    ip_interp33(dI, posU, posV, w, hit);
    const bool fin = isfinite(hit[0]);
    const float residual = hit[0] - (aff0 * colL + aff1);
    const float dResdDist = dx * hit[1] + dy * hit[2];
    const float hw = fabsf(residual) < s.huberTH ? 1 : s.huberTH / fabsf(residual);
    const float tH = hw * dResdDist * dResdDist, tb = hw * residual * dResdDist, tE = wgt * wgt * hw * residual * residual * (2 - hw);
    float H = 1, bb = 0, energy = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const bool f = __shfl_sync(0xffffffffu, (int)fin, k) != 0;
      const float sH = __shfl_sync(0xffffffffu, tH, k), sb = __shfl_sync(0xffffffffu, tb, k), sE = __shfl_sync(0xffffffffu, tE, k);
      if (!f) { energy = (float)((double)energy + 1e5); continue; }
      H += sH; bb += sb; energy += sE;
    }
    if (energy > bestEnergy) {
      stepBack = (float)((double)stepBack * 0.5);
      bestU = uBak + stepBack * dx;
      bestV = vBak + stepBack * dy;
    } else {
      float step = -gnstepsize * bb / H;
      if (step < -0.5f) step = -0.5f;
      else if (step > 0.5f) step = 0.5f;
      if (!isfinite(step)) step = 0;
      uBak = bestU;
      vBak = bestV;
      stepBack = step;
      bestU += step * dx;
      bestV += step * dy;
      bestEnergy = energy;
    }
    if (fabsf(stepBack) < s.trace_GNThreshold) break;
  }
  // ---- energy-based outlier test (L360-376) and the new depth interval (L380-402)
  if (!(bestEnergy < energyTH * s.trace_extraSlackOnTH)) IP_RETURN(status == 2 ? 1 : 2, -1.f, -1.f, 0.f);
  if (dx * dx > dy * dy) {
    idepth_min = (pr[2] * (bestU - errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU - errorInPixel * dx));
    idepth_max = (pr[2] * (bestU + errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU + errorInPixel * dx));
  } else {
    idepth_min = (pr[2] * (bestV - errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV - errorInPixel * dy));
    idepth_max = (pr[2] * (bestV + errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV + errorInPixel * dy));
  }
  if (idepth_min > idepth_max) { const float tmp = idepth_min; idepth_min = idepth_max; idepth_max = tmp; }
  if (lane == 0) { A.idepth_min[i] = idepth_min; A.idepth_max[i] = idepth_max; }   // the reference assigns the members before the final validity test
  if (!isfinite(idepth_min) || !isfinite(idepth_max) || (idepth_max < 0)) IP_RETURN(2, -1.f, -1.f, 0.f);
  IP_RETURN(0, bestU, bestV, 2 * errorInPixel);
#undef IP_RETURN
}

// ImmaturePoint::ImmaturePoint (ImmaturePoint.cpp:L34-63): pattern colours, gradient weights, gradH and energyTH from the HOST frame's level-0
// plane (getInterpolatedElement33BiLin, util/globalFuncs.h:L203-226) for integer pixels (u, v); ok = 0 where a colour is not finite
// (the reference then leaves energyTH = NaN and the caller drops the point)
__global__ void __launch_bounds__(128) ip_init_kernel(const __grid_constant__ IPInitArgs A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n || (A.n_dev && i >= *A.n_dev)) return;
  const int u = A.u[i], v = A.v[i];
  float g0 = 0, g1 = 0, g2 = 0, g3 = 0;
  bool ok = true;
  float col[8], wgt[8];
#pragma unroll
  for (int idx = 0; idx < 8; idx++) {
    col[idx] = 0.f; wgt[idx] = 0.f;
    if (!ok) continue;
    const float x = (float)(u + c_ip_pattern[idx][0]), y = (float)(v + c_ip_pattern[idx][1]);
    const int ix = (int)x, iy = (int)y;
    const float4* bp = A.img + ix + iy * A.w;
    const float tl = __ldg(bp).x, tr = __ldg(bp + 1).x, bl = __ldg(bp + A.w).x, br = __ldg(bp + A.w + 1).x;
    const float dx = x - ix, dy = y - iy;
    const float topInt = dx * tr + (1 - dx) * tl;
    const float botInt = dx * br + (1 - dx) * bl;
    const float leftInt = dy * bl + (1 - dy) * tl;
    const float rightInt = dy * br + (1 - dy) * tr;
    const float c0 = dx * rightInt + (1 - dx) * leftInt, c1 = rightInt - leftInt, c2 = botInt - topInt;
    col[idx] = c0;
    if (!isfinite(c0)) { ok = false; continue; }
    g0 += c1 * c1; g1 += c1 * c2; g2 += c2 * c1; g3 += c2 * c2;
    wgt[idx] = sqrtf(A.outlierTHSumComponent / (A.outlierTHSumComponent + (c1 * c1 + c2 * c2)));
  }
#pragma unroll
  for (int idx = 0; idx < 8; idx++) { A.color[8 * i + idx] = col[idx]; A.weights[8 * i + idx] = wgt[idx]; }
  A.gradH[4 * i] = g0; A.gradH[4 * i + 1] = g1; A.gradH[4 * i + 2] = g2; A.gradH[4 * i + 3] = g3;
  float eth = 8 * A.outlierTH;
  eth *= A.overallEnergyTHWeight * A.overallEnergyTHWeight;
  A.energyTH[i] = ok ? eth : __int_as_float(0x7fc00000);
  A.ok[i] = ok ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// ip_activate_kernel — FullSystem::optimizeImmaturePoint (FullSystem/FullSystemOptPoint.cpp:L51-205) with ImmaturePoint::linearizeResidual
// (FullSystem/ImmaturePoint.cpp:L498-565), projectPoint / derive_idepth (FullSystem/ResidualProjections.h:L36-87).
// EIGHT LANES per immature point (lane = pattern pixel), 4 points per warp: a residual's 8 samples are taken at once, its energy / Hdd / bd
// sums are folded in pattern order by every lane of the group (same additions, same order as the scalar loop), including the reference's
// behaviour on an out-of-bounds sample: the residual becomes OOB but the sums keep the terms of the samples BEFORE the first bad one.
// Same -fmad=false rule as the tracing kernel: bit-identical to the CPU code (float/double promotions of the reference kept explicitly).
// ---------------------------------------------------------------------------------------------------------------------
struct IPResState { int state, newState; double energy, newEnergy; };

// linearizeResidual for (point, target f) by the point's 8 lanes; every lane returns the same value and updates its copy of (Hdd, bd, rs)
__device__ __forceinline__ double ip_linearize_group(const IPActArgs& A, const int host, const int f, const float pu, const float pv, const float colL,
                                                     const float wL, const float energyTH, const float outlierTHSlack, IPResState& rs, float& Hdd, float& bd,
                                                     const float idepth, const int lane) {
  const bool skip = (rs.state == 1);   // an OOB residual stays OOB (uniform within the group; the warp's other groups still need this group's lanes in the shuffles)
  const int idx = lane & 7, base = lane & ~7;
  const float* R = A.RT + (size_t)(host * A.nf + f) * 12;
  const float* t = R + 9;
  const float* affLL = A.aff + (size_t)(host * A.nf + f) * 2;
  const float4* __restrict__ dIl = A.img[f];
  const float wM3G = (float)(A.w - 3), hM3G = (float)(A.h - 3);
  const int pdx = c_ip_pattern[idx][0], pdy = c_ip_pattern[idx][1];
  const float K0 = (pu + pdx - A.cxl) * A.fxli, K1 = (pv + pdy - A.cyl) * A.fyli, K2 = 1;
  float ptp[3];
#pragma unroll
  for (int i = 0; i < 3; i++) ptp[i] = ((R[3 * i] * K0 + R[3 * i + 1] * K1) + R[3 * i + 2] * K2) + t[i] * idepth;
  const float drescale = 1.0f / ptp[2];
  const float u = ptp[0] * drescale, v = ptp[1] * drescale;
  const float Ku = u * A.fxl + A.cxl, Kv = v * A.fyl + A.cyl;
  bool bad = skip || !(drescale > 0) || !(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G);
  float hit[3] = {0.f, 0.f, 0.f};
  if (!bad) {
    ip_interp33(dIl, Ku, Kv, A.w, hit);
    bad = !isfinite(hit[0]);
  }
  const float residual = hit[0] - (affLL[0] * colL + affLL[1]);
  float hw = fabsf(residual) < A.huberTH ? 1 : A.huberTH / fabsf(residual);
  const float tE = wL * wL * hw * residual * residual * (2 - hw);
  const float dxInterp = hit[1] * A.fxl, dyInterp = hit[2] * A.fyl;
  const float d_idepth = (dxInterp * drescale * (t[0] - t[2] * u) + dyInterp * drescale * (t[1] - t[2] * v)) * 1.0f;
  hw *= wL * wL;
  const float tH = (hw * d_idepth) * d_idepth, tb = (hw * residual) * d_idepth;
  const unsigned badmask = (__ballot_sync(0xffffffffu, bad) >> base) & 0xffu;
  const int first_bad = badmask ? (__ffs(badmask) - 1) : 8;   // the scalar loop returns at this sample; the earlier ones have been added
  float energyLeft = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const float sE = __shfl_sync(0xffffffffu, tE, base + k), sH = __shfl_sync(0xffffffffu, tH, base + k), sb = __shfl_sync(0xffffffffu, tb, base + k);
    if (k < first_bad && !skip) { energyLeft += sE; Hdd += sH; bd += sb; }
  }
  if (skip || first_bad < 8) { rs.newState = 1; return rs.energy; }
  if (energyLeft > energyTH * outlierTHSlack) { energyLeft = energyTH * outlierTHSlack; rs.newState = 2; }
  else rs.newState = 0;
  rs.newEnergy = energyLeft;
  return energyLeft;
}

__global__ void __launch_bounds__(128) ip_activate_kernel(const __grid_constant__ IPActArgs A) {
  const int lane = threadIdx.x & 31;
  const int i_raw = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // 8 lanes per point
  const bool active = i_raw < A.n;
  const int i = active ? i_raw : A.n - 1;   // groups beyond the list shadow the last point (the warp's shuffles need every lane) and write nothing
  const bool writer = active && (lane & 7) == 0;
  const int nf = A.nf, host = A.host[i];
  const float pu = A.u[i], pv = A.v[i], energyTH = A.energyTH[i];
  const float colL = A.color[8 * i + (lane & 7)], wL = A.weights[8 * i + (lane & 7)];
  int* rs_out = A.res_state + (size_t)i * nf;
  IPResState res[DMV_MAX_FRAMES];   // indexed by target frame with compile-time indices only (registers)
#pragma unroll
  for (int f = 0; f < DMV_MAX_FRAMES; f++) { res[f].state = 0; res[f].newState = 2; res[f].energy = 0; res[f].newEnergy = 0; }
  float lastEnergy = 0, lastHdd = 0, lastbd = 0;
  float currentIdepth = (A.idepth_max[i] + A.idepth_min[i]) * 0.5f;
  bool done = false;   // per group; the warp keeps executing every step (shuffles), a finished group only stops updating / writing
  int status_out = 0;
#pragma unroll
  for (int f = 0; f < DMV_MAX_FRAMES; f++) {
    if (f < nf && f != host) {
      lastEnergy = (float)((double)lastEnergy + ip_linearize_group(A, host, f, pu, pv, colL, wL, energyTH, 1000.f, res[f], lastHdd, lastbd, currentIdepth, lane));
      res[f].state = res[f].newState;
      res[f].energy = res[f].newEnergy;
    }
  }
  float idepth_out = currentIdepth;
  if (!isfinite(lastEnergy) || lastHdd < A.minIdepthH_act) { done = true; status_out = 0; }
  float lambda = 0.1f;
  for (int iteration = 0; iteration < A.GNIts; iteration++) {
    if (__all_sync(0xffffffffu, done)) break;
    float H = lastHdd;
    H *= 1 + lambda;
    const float step = (float)((1.0 / (double)H) * (double)lastbd);
    const float newIdepth = currentIdepth - step;
    float newHdd = 0, newbd = 0, newEnergy = 0;
#pragma unroll
    for (int f = 0; f < DMV_MAX_FRAMES; f++)
      if (f < nf && f != host)
        newEnergy = (float)((double)newEnergy + ip_linearize_group(A, host, f, pu, pv, colL, wL, energyTH, 1.f, res[f], newHdd, newbd, newIdepth, lane));
    if (done) continue;
    if (!isfinite(lastEnergy) || newHdd < A.minIdepthH_act) { idepth_out = currentIdepth; status_out = 0; done = true; continue; }
    if (newEnergy < lastEnergy) {
      currentIdepth = newIdepth;
      lastHdd = newHdd; lastbd = newbd; lastEnergy = newEnergy;
#pragma unroll
      for (int f = 0; f < DMV_MAX_FRAMES; f++) { res[f].state = res[f].newState; res[f].energy = res[f].newEnergy; }
      lambda = (float)((double)lambda * 0.5);
    } else {
      lambda *= 5;
    }
    if ((double)fabsf(step) < 0.0001 * (double)currentIdepth) { done = true; status_out = 2; }   // 2 = loop left normally (decided below)
  }
  if (!done || status_out == 2) {   // the loop ended by its break / its bound: the reference's epilogue (FullSystemOptPoint.cpp:L170-205)
    idepth_out = currentIdepth;
    if (!isfinite(currentIdepth)) status_out = -1;
    else {
      int numGoodRes = 0;
#pragma unroll
      for (int f = 0; f < DMV_MAX_FRAMES; f++)
        if (f < nf && f != host && res[f].state == 0) numGoodRes++;
      status_out = (numGoodRes < A.minObs || !isfinite(energyTH)) ? -1 : 1;
      if (writer) {
#pragma unroll
        for (int f = 0; f < DMV_MAX_FRAMES; f++)
          if (f < nf) rs_out[f] = (f != host) ? res[f].state : 255;
      }
    }
    if (writer && !isfinite(currentIdepth)) {
      for (int f = 0; f < nf; f++) rs_out[f] = 255;
    }
  } else if (writer) {
    for (int f = 0; f < nf; f++) rs_out[f] = 255;
  }
  if (writer) { A.idepth[i] = idepth_out; A.status[i] = status_out; }
}

void launch_ip_activate(const IPActArgs& A, cudaStream_t s) { ip_activate_kernel<<<(A.n + 15) / 16, 128, 0, s>>>(A); }  // 8 lanes per point

void launch_ip_init(const IPInitArgs& A, cudaStream_t s) { ip_init_kernel<<<(A.n + 127) / 128, 128, 0, s>>>(A); }

void launch_ip_trace(const IPTraceArgs& A, cudaStream_t s) { ip_trace_kernel<<<(A.n + 3) / 4, 128, 0, s>>>(A); }  // 4 warps = 4 points per CTA

}  // namespace dmv
