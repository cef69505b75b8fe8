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
// The flag affects device code only, so the C-ABI entry points of the three kernels (end of the file) are compiled here too.
#include "ct_handle.h"
#include "ba_handle.h"
#include "ip_store.h"
#include "ip_trace.h"
#include <cstring>
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

// The point arrays (ipw layout), IPTraceMember and IPTraceArgs are declared in ip_trace.h.
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

// One launch serves up to DMV_CT_TRACE_MANY_MAX handles.  Each member's points start at a CTA (first[k] is a multiple of 4 warps), so the
// member lookup depends on blockIdx alone: the scan and the member's descriptor live in uniform registers, and the kernel keeps the
// 72 registers of its one-handle form (7 CTAs per SM).  Warps past a member's last point return at once; the kernel has no block-level
// synchronisation and returns per warp.
__global__ void __launch_bounds__(128, 7) ip_trace_kernel(const __grid_constant__ IPTraceArgs A) {
  const int lane = threadIdx.x & 31;
  const int cta_warp = 4 * blockIdx.x;
  int mem = 0;
  while (cta_warp >= A.first[mem + 1]) mem++;   // the grid covers first[n] warps; skips empty members (first[mem] == first[mem + 1])
  const IPTraceMember& M = A.m[mem];
  const int i = cta_warp + (threadIdx.x >> 5) - A.first[mem];   // warp = point
  if (i >= M.n) return;
  float* const ip = M.ip;
  const size_t cap = M.cap;
  int* const st_out = reinterpret_cast<int*>(ip + ipw::status * cap);
  float* const uv_out = ip + ipw::uv * cap;
  float* const iv_out = ip + ipw::interval * cap;
  const dmv_ip_settings& s = A.s;
  const int w = M.w, h = M.h;
  const float4* __restrict__ dI = M.img;
  const float* tabp = ip + ipw::tables * cap + 14 * reinterpret_cast<const int*>(ip)[ipw::set * cap + i];
  const float* KRKi = tabp;
  const float* Kt = tabp + 9;
  const float aff0 = tabp[12], aff1 = tabp[13];
  const int status = st_out[i];
  if (status == 1) return;  // IPS_OOB stays OOB (ImmaturePoint.cpp:L79)
  const float u = ip[ipw::u * cap + i], v = ip[ipw::v * cap + i];
  float idepth_min = ip[ipw::idepth_min * cap + i], idepth_max = ip[ipw::idepth_max * cap + i];
  float color[8];
#pragma unroll
  for (int k = 0; k < 8; k++) color[k] = ip[ipw::color * cap + 8 * i + k];
  const float* gH = ip + ipw::gradH * cap + 4 * i;
  const float g0 = gH[0], g1 = gH[1], g2 = gH[2], g3 = gH[3];
  const float energyTH = ip[ipw::energyTH * cap + i];
#define IP_RETURN(st, ux, uy, itv) do { if (lane == 0) { st_out[i] = (st); uv_out[2 * i] = (ux); uv_out[2 * i + 1] = (uy); iv_out[i] = (itv); } return; } while (0)
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
  float quality = ip[ipw::quality * cap + i];
  if (newQuality < quality || numSteps > 10) quality = newQuality;
  __syncwarp();
  if (lane == 0) ip[ipw::quality * cap + i] = quality;
  // ---- Gauss-Newton refinement along the line (L280-353): lane idx < 8 samples pattern pixel idx, the sums fold in pattern order
  float uBak = bestU, vBak = bestV, stepBack = 0;
  const float gnstepsize = 1;
  if (s.trace_GNIterations > 0) bestEnergy = 1e5f;
  const int idx8 = lane & 7;
  const float wgt = ip[ipw::weights * cap + 8 * i + idx8];
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
  if (lane == 0) { ip[ipw::idepth_min * cap + i] = idepth_min; ip[ipw::idepth_max * cap + i] = idepth_max; }   // the reference assigns the members before the final validity test
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
struct IPActArgs {
  int n, nf, w, h, minObs, GNIts;
  float fxl, fyl, cxl, cyl, fxli, fyli, huberTH, minIdepthH_act;
  const float4* img[DMV_MAX_FRAMES];
  const float* RT;    // [h*nf+t][12]
  const float* aff;   // [h*nf+t][2]
  const int* host;
  const float *u, *v, *color, *weights, *energyTH, *idepth_min, *idepth_max;
  int* status;
  float* idepth;
  int* res_state;     // [n][nf]
};
struct IPResState { int state, newState; double energy, newEnergy; };

// linearizeResidual for (point, target f) by the point's 8 lanes; every lane returns the same value and updates its copy of (Hdd, bd, rs).
// Every group of the warp calls it for every f < nf: the 4 points of a warp may have different hosts, and the shuffles and the ballot below
// name all 32 lanes, so a group whose host is f runs them too, adds nothing and returns 0 without touching rs.
__device__ __forceinline__ double ip_linearize_group(const IPActArgs& A, const int host, const int f, const float pu, const float pv, const float colL,
                                                     const float wL, const float energyTH, const float outlierTHSlack, IPResState& rs, float& Hdd, float& bd,
                                                     const float idepth, const int lane) {
  const bool own = (f != host);        // f == host: no residual (the group only takes part in the warp's shuffles)
  const bool skip = !own || (rs.state == 1);   // an OOB residual stays OOB (uniform within the group; the warp's other groups still need this group's lanes in the shuffles)
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
  if (!own) return 0.0;
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
    if (f < nf) {   // warp-uniform; f == host is decided per group inside (the call holds warp-wide shuffles)
      const double e = ip_linearize_group(A, host, f, pu, pv, colL, wL, energyTH, 1000.f, res[f], lastHdd, lastbd, currentIdepth, lane);
      if (f != host) {
        lastEnergy = (float)((double)lastEnergy + e);
        res[f].state = res[f].newState;
        res[f].energy = res[f].newEnergy;
      }
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
    for (int f = 0; f < DMV_MAX_FRAMES; f++) {
      if (f < nf) {
        const double e = ip_linearize_group(A, host, f, pu, pv, colL, wL, energyTH, 1.f, res[f], newHdd, newbd, newIdepth, lane);
        if (f != host) newEnergy = (float)((double)newEnergy + e);
      }
    }
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

void launch_ip_init(const IPInitArgs& A, cudaStream_t s) { ip_init_kernel<<<(A.n + 127) / 128, 128, 0, s>>>(A); }

void ip_trace_args(IPTraceArgs& A, int n, const dmv_ip_settings* settings) {
  std::memset(&A, 0, sizeof(A));
  A.n = n;
  if (settings) A.s = *settings; else dmv_ip_default_settings(&A.s);
}

void ip_trace_member(IPTraceArgs& A, int i, const dmv_ct* c, float* ip, int cap, int np) {
  A.first[i + 1] = A.first[i] + (np + 3) / 4 * 4;   // whole CTAs per member
  if (np > 0) { A.m[i].img = c->d_img[0]; A.m[i].ip = ip; A.m[i].cap = cap; A.m[i].w = c->w[0]; A.m[i].h = c->h[0]; A.m[i].n = np; }
}

int ip_trace_launch(dmv_ct* const* hs, const IPTraceArgs& A) {
  const cudaStream_t s = hs[0]->stream;
  for (int i = 1; i < A.n; i++) CK(ct_order_behind(hs[i], s));   // behind each member's frame uploads and the copies its caller queued there
  ip_trace_kernel<<<A.first[A.n] / 4, 128, 0, s>>>(A);   // 4 warps = 4 points per CTA
  for (int i = 0; i < A.n; i++)
    if (A.m[i].n > 0) hs[i]->launches++;
  CK(cudaGetLastError());
  return DMV_OK;
}

// d_act / h_act hold n points; RT and the window's PRE_aff_mode staged in h_act
static int act_stage(dmv_ba* b, int n, const float* RT) {
  b->act_n = -1;   // the staging no longer holds the last activation's entries
  if (n > b->act_cap) {
    b->act_cap = 0;
    const int cap = std::max(n, 2048);
    const size_t words = act_layout(cap).words;
    CK(b->d_act.reserve(words));
    CK(b->h_act.reserve(words));
    b->act_cap = cap;
  }
  const ActLayout o = act_layout(b->act_cap);
  const int nf = b->nf;
  float* hb = b->h_act;
  std::memcpy(hb + o.rt, RT, sizeof(float) * 12 * nf * nf);
  const BAIter& it = b->h_up->it;
  for (int k = 0; k < nf * nf; k++) { hb[o.aff + 2 * k] = it.precalc[k][24]; hb[o.aff + 2 * k + 1] = it.precalc[k][25]; }  // PRE_aff_mode
  return DMV_OK;
}

// ip_activate_kernel on the n points staged in d_act, the read-back (and the rows' lastTraceStatus when trace_status is not NULL) and one
// synchronisation
static int act_launch(dmv_ba* b, int n, int minObs, int32_t* status, float* idepth, int32_t* res_state, int32_t* trace_status) {
  const int nf = b->nf;
  const ActLayout o = act_layout(b->act_cap);
  float* hb = b->h_act;
  float* d = b->d_act;
  const BAIter& it = b->h_up->it;
  IPActArgs A;
  A.n = n; A.nf = nf; A.w = b->cfg.w; A.h = b->cfg.h; A.minObs = minObs; A.GNIts = 3;  // setting_GNItsOnPointActivation
  A.fxl = it.calib[0]; A.fyl = it.calib[1]; A.cxl = it.calib[2]; A.cyl = it.calib[3]; A.fxli = it.calib[4]; A.fyli = it.calib[5];
  A.huberTH = b->prm.huberTH; A.minIdepthH_act = 100.f;                                      // setting_minIdepthH_act
  for (int f = 0; f < MAXF; f++) A.img[f] = f < nf ? b->d_img[b->slots[f]].get() : nullptr;
  A.RT = d + o.rt; A.aff = d + o.aff; A.host = reinterpret_cast<const int*>(d + o.host);
  A.u = d + o.u; A.v = d + o.v; A.color = d + o.col; A.weights = d + o.wgt; A.energyTH = d + o.eth; A.idepth_min = d + o.min; A.idepth_max = d + o.max;
  A.status = reinterpret_cast<int*>(d + o.st); A.idepth = d + o.id; A.res_state = reinterpret_cast<int*>(d + o.rs);
  ip_activate_kernel<<<(A.n + 15) / 16, 128, 0, b->stream>>>(A);   // 8 lanes per point
  b->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(hb + o.st, d + o.st, sizeof(float) * (o.rs - o.st + (size_t)nf * n), cudaMemcpyDeviceToHost, b->stream));
  if (trace_status) CK(cudaMemcpyAsync(hb + o.ts, d + o.ts, 4 * (size_t)n, cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  std::memcpy(status, hb + o.st, 4 * (size_t)n); std::memcpy(idepth, hb + o.id, 4 * (size_t)n);
  std::memcpy(res_state, hb + o.rs, 4 * (size_t)n * nf);
  if (trace_status) std::memcpy(trace_status, hb + o.ts, 4 * (size_t)n);
  return DMV_OK;
}

// The activation's rows fed from a store: row j = toOptimize entry opt[j], an index into the groups' concatenation; group f's row i is the
// store's row src[f] + i - off[f].  Copies host frame f, u, v, color8, weights8, energyTH, idepth_min, idepth_max and lastTraceStatus
// into dmv_ba_activate_points' staging.
struct ActGatherArgs {
  int n, nf, scap;
  int off[MAXF + 1], src[MAXF];
  const int* opt;
  const unsigned* pts;
  unsigned* d;        // d_act
  ActLayout o;
};
__global__ void __launch_bounds__(128) ip_act_gather_kernel(const __grid_constant__ ActGatherArgs G) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= G.n) return;
  const int i = G.opt[j];
  int f = 0;
  while (G.off[f + 1] <= i) f++;
  const size_t r = G.src[f] + (i - G.off[f]), scap = G.scap;
  const ActLayout& o = G.o;
  G.d[o.host + j] = f;
  G.d[o.u + j] = G.pts[ipw::u * scap + r];
  G.d[o.v + j] = G.pts[ipw::v * scap + r];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    G.d[o.col + 8 * j + k] = G.pts[ipw::color * scap + 8 * r + k];
    G.d[o.wgt + 8 * j + k] = G.pts[ipw::weights * scap + 8 * r + k];
  }
  G.d[o.eth + j] = G.pts[ipw::energyTH * scap + r];
  G.d[o.min + j] = G.pts[ipw::idepth_min * scap + r];
  G.d[o.max + j] = G.pts[ipw::idepth_max * scap + r];
  G.d[o.ts + j] = G.pts[ipw::status * scap + r];
}

int ip_act_from_store(dmv_ba* b, const dmv_ip_store* s, const int* imm_offset, const int* slot, const int* d_opt, int n, const float* RT, int minObs,
                      int32_t* status, float* idepth, int32_t* res_state, int32_t* trace_status) {
  if (n == 0) return DMV_OK;
  CK(cudaSetDevice(b->device));
  const int rc = act_stage(b, n, RT);
  if (rc != DMV_OK) return rc;
  ActGatherArgs G;
  G.n = n; G.nf = b->nf; G.scap = s->cap[s->cur];
  for (int f = 0; f < b->nf; f++) { G.off[f] = imm_offset[f]; G.src[f] = slot[f] >= 0 ? ip_store_first(s, slot[f]) : 0; }
  G.off[b->nf] = imm_offset[b->nf];
  G.opt = d_opt;
  G.pts = reinterpret_cast<const unsigned*>(s->d_pts[s->cur].get());
  G.d = reinterpret_cast<unsigned*>(b->d_act.get());
  G.o = act_layout(b->act_cap);
  CK(cudaMemcpyAsync(b->d_act, b->h_act, sizeof(float) * G.o.host, cudaMemcpyHostToDevice, b->stream));
  ip_act_gather_kernel<<<(n + 127) / 128, 128, 0, b->stream>>>(G);
  return act_launch(b, n, minObs, status, idepth, res_state, trace_status);
}

}  // namespace dmv

using namespace dmv;

void dmv_ip_default_settings(dmv_ip_settings* s) {
  s->maxPixSearch = 0.027f; s->trace_stepsize = 1.0f; s->trace_GNThreshold = 0.1f; s->trace_extraSlackOnTH = 1.2f; s->trace_slackInterval = 1.5f;
  s->trace_minImprovementFactor = 2.f; s->huberTH = 9.f; s->trace_GNIterations = 3; s->minTraceTestRadius = 2;
}

// ImmaturePoint constructor on the resident frame (ip_init_kernel)
int dmv_ct_init_points(dmv_ct* c, int n, const int32_t* u, const int32_t* v, float* color8, float* weights8, float* gradH4, float* energyTH, int32_t* ok) {
  if (!c || n < 0 || (n > 0 && (!u || !v || !color8 || !weights8 || !gradH4 || !energyTH || !ok))) return set_error(DMV_ERR_INVALID, "null argument");
  if (n == 0) return DMV_OK;
  for (int i = 0; i < n; i++)
    if (u[i] < 2 || v[i] < 2 || u[i] >= c->w[0] - 3 || v[i] >= c->h[0] - 3) return set_error(DMV_ERR_INVALID, "point %d (%d,%d): the pattern leaves the image", i, u[i], v[i]);
  CK(cudaSetDevice(c->device));
  CK(ct_reserve_ip(c, n));
  CK(ct_wait_staging(c));
  const size_t cap = c->ip_cap;
  float* hb = c->h_ip;
  float* d = c->d_ip;
  // layout (words): u | v | color*8 | weights*8 | gradH*4 | energyTH | ok
  std::memcpy(hb, u, 4 * (size_t)n); std::memcpy(hb + cap, v, 4 * (size_t)n);
  CK(cudaMemcpyAsync(d, hb, sizeof(float) * 2 * cap, cudaMemcpyHostToDevice, c->stream));
  IPInitArgs A;
  A.n = n; A.w = c->w[0]; A.n_dev = nullptr;
  A.outlierTHSumComponent = 50.f * 50.f; A.outlierTH = 12.f * 12.f; A.overallEnergyTHWeight = 1.f;  // util/settings.cpp:L111-114, L159
  A.u = reinterpret_cast<const int*>(d); A.v = reinterpret_cast<const int*>(d + cap);
  A.color = d + 2 * cap; A.weights = d + 10 * cap; A.gradH = d + 18 * cap; A.energyTH = d + 22 * cap; A.ok = reinterpret_cast<int*>(d + 23 * cap);
  A.img = c->d_img[0];
  launch_ip_init(A, c->stream);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(hb + 2 * cap, d + 2 * cap, sizeof(float) * 22 * cap, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  std::memcpy(color8, hb + 2 * cap, 32 * (size_t)n); std::memcpy(weights8, hb + 10 * cap, 32 * (size_t)n); std::memcpy(gradH4, hb + 18 * cap, 16 * (size_t)n);
  std::memcpy(energyTH, hb + 22 * cap, 4 * (size_t)n); std::memcpy(ok, hb + 23 * cap, 4 * (size_t)n);
  return DMV_OK;
}

// dmv_ct_trace_points_multi's checks of one handle's job, in its order; *n = the job's point count.  No CUDA call.
static int ip_trace_check(const dmv_ct_trace_job& j, int* n) {
  if (j.nsets < 0 || (j.nsets > 0 && (!j.sets || !j.tables14))) return set_error(DMV_ERR_INVALID, "null argument");
  *n = 0;
  for (int k = 0; k < j.nsets; k++) {
    const dmv_ip_points* p = &j.sets[k];
    if (p->n < 0 || (p->n > 0 && (!p->u || !p->v || !p->color8 || !p->weights8 || !p->gradH4 || !p->energyTH || !p->idepth_min || !p->idepth_max || !p->quality ||
                                  !p->lastTraceStatus || !p->lastTraceUV2 || !p->lastTracePixelInterval)))
      return set_error(DMV_ERR_INVALID, "incomplete dmv_ip_points (set %d)", k);
    *n += p->n;
  }
  if (*n > 0 && j.nsets > 64) return set_error(DMV_ERR_INVALID, "at most 64 host frames per call");
  return DMV_OK;
}

// The immature points of n handles (n = 1: dmv_ct_trace_points_multi) traced in ONE launch of ip_trace_kernel.  Every job is checked before
// anything is allocated, copied or launched (`many`: a job's error names its member).  Member i's points go through its own staging area
// d_ip / h_ip, uploaded on its own stream; the launch goes on handles[0]'s stream behind every member's queued work, the downloads follow it
// there, and one synchronisation ends the call.
// h_ip is written without ct_wait_staging: an upload still in flight reads h_scratch, never h_ip, and every call that fills h_ip synchronises
// its stream before it returns, so nothing can be reading h_ip here.
static int ip_trace_run(dmv_ct* const* hs, int n, const dmv_ct_trace_job* jobs, const dmv_ip_settings* settings, bool many) {
  int np[DMV_CT_TRACE_MANY_MAX];
  int total = 0;
  for (int i = 0; i < n; i++) {
    const int rc = ip_trace_check(jobs[i], &np[i]);
    if (rc != DMV_OK) return many ? ct_member_error(rc, i) : rc;
    total += np[i];
  }
  if (total == 0) return DMV_OK;
  CK(cudaSetDevice(hs[0]->device));
  for (int i = 0; i < n; i++)
    if (np[i] > 0) CK(ct_reserve_ip(hs[i], np[i]));
  IPTraceArgs A;
  ip_trace_args(A, n, settings);
  const cudaStream_t s = hs[0]->stream;
  for (int i = 0; i < n; i++) {
    dmv_ct* c = hs[i];
    const dmv_ct_trace_job& j = jobs[i];
    ip_trace_member(A, i, c, c->d_ip, c->ip_cap, np[i]);
    if (np[i] > 0) {
      const size_t cap = c->ip_cap;
      float* hb = c->h_ip;
      size_t at = 0;
      for (int k = 0; k < j.nsets; k++) {
        const dmv_ip_points* p = &j.sets[k];
        const size_t m = (size_t)p->n;
        if (m == 0) continue;
        std::memcpy(hb + ipw::u * cap + at, p->u, 4 * m); std::memcpy(hb + ipw::v * cap + at, p->v, 4 * m);
        std::memcpy(hb + ipw::color * cap + 8 * at, p->color8, 32 * m); std::memcpy(hb + ipw::weights * cap + 8 * at, p->weights8, 32 * m);
        std::memcpy(hb + ipw::gradH * cap + 4 * at, p->gradH4, 16 * m); std::memcpy(hb + ipw::energyTH * cap + at, p->energyTH, 4 * m);
        std::memcpy(hb + ipw::idepth_min * cap + at, p->idepth_min, 4 * m); std::memcpy(hb + ipw::idepth_max * cap + at, p->idepth_max, 4 * m);
        std::memcpy(hb + ipw::quality * cap + at, p->quality, 4 * m); std::memcpy(hb + ipw::status * cap + at, p->lastTraceStatus, 4 * m);
        std::memcpy(hb + ipw::uv * cap + 2 * at, p->lastTraceUV2, 8 * m); std::memcpy(hb + ipw::interval * cap + at, p->lastTracePixelInterval, 4 * m);
        int* setp = reinterpret_cast<int*>(hb + ipw::set * cap + at);
        for (size_t q = 0; q < m; q++) setp[q] = k;
        at += m;
      }
      std::memcpy(hb + ipw::tables * cap, j.tables14, sizeof(float) * 14 * (size_t)j.nsets);
      CK(cudaMemcpyAsync(c->d_ip, hb, sizeof(float) * (ipw::tables * cap + 14 * (size_t)j.nsets), cudaMemcpyHostToDevice, c->stream));
    }
  }
  const int rc = ip_trace_launch(hs, A);
  if (rc != DMV_OK) return rc;
  for (int i = 0; i < n; i++) {   // the 7 in/out words per point
    if (np[i] == 0) continue;
    const size_t cap = hs[i]->ip_cap;
    CK(cudaMemcpyAsync(hs[i]->h_ip + ipw::idepth_min * cap, hs[i]->d_ip + ipw::idepth_min * cap, sizeof(float) * ipw::inout * cap, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  for (int i = 0; i < n; i++) {
    hs[i]->staging_busy = false;   // every member's queued work completed before the kernel started
    const size_t cap = hs[i]->ip_cap;
    const float* hb = hs[i]->h_ip;
    size_t at = 0;
    for (int k = 0; k < jobs[i].nsets; k++) {
      const dmv_ip_points* p = &jobs[i].sets[k];
      const size_t m = (size_t)p->n;
      if (m == 0) continue;
      std::memcpy(p->idepth_min, hb + ipw::idepth_min * cap + at, 4 * m); std::memcpy(p->idepth_max, hb + ipw::idepth_max * cap + at, 4 * m);
      std::memcpy(p->quality, hb + ipw::quality * cap + at, 4 * m); std::memcpy(p->lastTraceStatus, hb + ipw::status * cap + at, 4 * m);
      std::memcpy(p->lastTraceUV2, hb + ipw::uv * cap + 2 * at, 8 * m); std::memcpy(p->lastTracePixelInterval, hb + ipw::interval * cap + at, 4 * m);
      at += m;
    }
  }
  return DMV_OK;
}

// immature points of SEVERAL host frames traced against the resident newest frame in ONE launch (ip_trace_kernel): FullSystem::traceNewCoarse's
// loop over the window's keyframes (FullSystem.cpp:L554-575) collapsed into one upload, one kernel, one download
int dmv_ct_trace_points_multi(dmv_ct* c, int nsets, const dmv_ip_points* sets, const float* tables14, const dmv_ip_settings* settings) {
  if (!c) return set_error(DMV_ERR_INVALID, "null argument");
  dmv_ct_trace_job j;
  j.nsets = nsets; j.sets = sets; j.tables14 = tables14;
  return ip_trace_run(&c, 1, &j, settings, false);
}

// dmv_ct_trace_points_multi for n handles in one launch.  Every check precedes the first allocation, copy or launch.
int dmv_ct_trace_many(dmv_ct* const* handles, int n, const dmv_ct_trace_job* jobs, const dmv_ip_settings* settings) {
  if (!handles || !jobs) return set_error(DMV_ERR_INVALID, "null argument");
  const int rc = ct_check_members(handles, n, DMV_CT_TRACE_MANY_MAX);
  if (rc != DMV_OK) return rc;
  return ip_trace_run(handles, n, jobs, settings, true);
}

// one host frame's immature points traced against the resident newest frame
int dmv_ct_trace_points(dmv_ct* c, const dmv_ip_points* p, const float KRKi[9], const float Kt[3], const float aff[2], const dmv_ip_settings* settings) {
  if (!c || !p || !KRKi || !Kt || !aff) return set_error(DMV_ERR_INVALID, "null argument");
  float tab[14];
  std::memcpy(tab, KRKi, 36); std::memcpy(tab + 9, Kt, 12); std::memcpy(tab + 12, aff, 8);
  return dmv_ct_trace_points_multi(c, 1, p, tab, settings);
}

// FullSystem::optimizeImmaturePoint for a batch of immature points (ip_activate_kernel) on the BA handle's window
int dmv_ba_activate_points(dmv_ba* b, const dmv_ba_activate_args* a) {
  if (!b || !a) return set_error(DMV_ERR_INVALID, "null argument");
  if (b->nf < 2 || !b->have_state) return set_error(DMV_ERR_STATE, "dmv_ba_set_window + dmv_ba_set_state first");
  if (a->n < 0 || (a->n > 0 && (!a->host || !a->u || !a->v || !a->color8 || !a->weights8 || !a->energyTH || !a->idepth_min || !a->idepth_max || !a->RT ||
                                !a->status || !a->idepth || !a->res_state)))
    return set_error(DMV_ERR_INVALID, "incomplete dmv_ba_activate_args");
  if (a->n == 0) {
    b->act_n = 0;
    return DMV_OK;
  }
  const int n = a->n, nf = b->nf;
  for (int i = 0; i < n; i++)
    if (a->host[i] < 0 || a->host[i] >= nf) return set_error(DMV_ERR_INVALID, "point %d: host %d out of range", i, a->host[i]);
  CK(cudaSetDevice(b->device));
  const int rc = act_stage(b, n, a->RT);
  if (rc != DMV_OK) return rc;
  const ActLayout o = act_layout(b->act_cap);
  float* hb = b->h_act;
  std::memcpy(hb + o.host, a->host, 4 * (size_t)n); std::memcpy(hb + o.u, a->u, 4 * (size_t)n); std::memcpy(hb + o.v, a->v, 4 * (size_t)n);
  std::memcpy(hb + o.col, a->color8, 32 * (size_t)n); std::memcpy(hb + o.wgt, a->weights8, 32 * (size_t)n); std::memcpy(hb + o.eth, a->energyTH, 4 * (size_t)n);
  std::memcpy(hb + o.min, a->idepth_min, 4 * (size_t)n); std::memcpy(hb + o.max, a->idepth_max, 4 * (size_t)n);
  CK(cudaMemcpyAsync(b->d_act, hb, sizeof(float) * o.st, cudaMemcpyHostToDevice, b->stream));
  const int rc2 = act_launch(b, n, a->minObs, a->status, a->idepth, a->res_state, nullptr);
  if (rc2 == DMV_OK) b->act_n = n;
  return rc2;
}
