// sm_90a kernel + C-ABI of CoarseInitializer::calcResAndGS (FullSystem/CoarseInitializer.cpp:L333-625): the two-frame direct initialiser's
// linearisation — 8-pixel pattern per point, one inverse depth per point eliminated by a Schur complement (DESIGN.md §5c).
//
//   ci_res_gs_kernel   8 lanes per point (one per pattern pixel), 4 points per warp: project, 4-tap float4 gather from the new frame's level
//                      plane and the first frame's, Huber residual, the point's JbBuffer row (xor-butterfly over the 8 lanes), outlier test,
//                      and BOTH accumulations in the same pass: Accumulator9 of [dp0..dp7, r] over pixels of good points (lane-local 45
//                      products) and the weighted Accumulator9 of the Schur rows.  The reference needs three passes because alphaOpt depends
//                      on the whole set (L544-557) — but only through EAlpha, which the reference never updates (dso issue #52 behaviour,
//                      reproduced): alphaEnergy = alphaW * |t|^2 * npts is known BEFORE the launch, so one pass suffices.  It is
//                      evaluated in double and rounded to float once, like the reference's, so the cap and res3[1] match it bit for bit.
//                      Block reduction -> per-CTA fp64 partials -> the last CTA (ticket) folds them in a fixed order: deterministic, one launch.
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace dmv {

constexpr int CI_THREADS = 256;
constexpr int CI_NRED = 45 + 45 + 3;  // acc9 | acc9SC | energy sum, #good_new, pad

struct CIParams {
  float RKi[9], t[3];
  float fx, fy, cx, cy;
  float aff0, aff1;        // exp(a), b
  float huber, alphaOpt, coupling;
  int w, h, n;
};

struct CIPoints {
  const float *u, *v, *outlierTH;                        // set once per level
  const float *idepth_new, *energy, *iR;                 // per evaluation (energy: 2 per point)
  const unsigned char* isGood;
  unsigned char* isGood_new;                             // outputs
  float *energy_new, *maxstep, *lastHessian_new, *Jb;    // energy_new: 2 per point, Jb: 10 per point
};

__device__ __forceinline__ float ci_group_sum(float a) {
  a += __shfl_xor_sync(0xffffffffu, a, 4);
  a += __shfl_xor_sync(0xffffffffu, a, 2);
  a += __shfl_xor_sync(0xffffffffu, a, 1);
  return a;
}

__device__ __forceinline__ float4 ci_bilin(const float4* __restrict__ img, float x, float y, int w) {
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float4* bp = img + (size_t)iy * w + ix;
  const float4 tl = __ldg(bp), tr = __ldg(bp + 1), bl = __ldg(bp + w), br = __ldg(bp + w + 1);
  const float w11 = dxdy, w10 = dy - dxdy, w01 = dx - dxdy, w00 = 1 - dx - dy + dxdy;
  return make_float4(w11 * br.x + w10 * bl.x + w01 * tr.x + w00 * tl.x, w11 * br.y + w10 * bl.y + w01 * tr.y + w00 * tl.y,
                     w11 * br.z + w10 * bl.z + w01 * tr.z + w00 * tl.z, 0.f);
}

__global__ void __launch_bounds__(CI_THREADS) ci_res_gs_kernel(const __grid_constant__ CIParams P, const __grid_constant__ CIPoints Q,
                                                               const float4* __restrict__ imgRef, const float4* __restrict__ imgNew,
                                                               double* __restrict__ partial, unsigned int* __restrict__ ticket, double* __restrict__ out) {
  __shared__ float s_red[CI_THREADS / 32][CI_NRED];
  __shared__ bool s_last;
  const int tid = threadIdx.x, px = tid & 7, lane = tid & 31, warp = tid >> 5;
  // staticPattern[8] (util/settings.h:L232-244, pattern 8)
  const int pdx = (px == 0) ? 0 : (px == 1) ? -1 : (px == 2) ? 1 : (px == 3) ? -2 : (px == 4) ? 0 : (px == 5) ? 2 : (px == 6) ? -1 : 0;
  const int pdy = (px == 0) ? -2 : (px == 1) ? -1 : (px == 2) ? -1 : (px == 3) ? 0 : (px == 4) ? 0 : (px == 5) ? 0 : (px == 6) ? 1 : 2;
  float acc[45], accsc[45];
#pragma unroll
  for (int e = 0; e < 45; e++) acc[e] = accsc[e] = 0.f;
  float accE = 0.f, accN = 0.f;

  for (int base = blockIdx.x * (CI_THREADS / 8); base < P.n; base += gridDim.x * (CI_THREADS / 8)) {  // warp-uniform trip count
    const int i = base + (tid >> 3);
    const bool have = i < P.n;
    const int ii = have ? i : P.n - 1;
    const float pu = __ldg(Q.u + ii), pv = __ldg(Q.v + ii), id = __ldg(Q.idepth_new + ii);
    const bool wasGood = have && __ldg(Q.isGood + ii) != 0;
    const float e0 = __ldg(Q.energy + 2 * ii), e1 = __ldg(Q.energy + 2 * ii + 1);
    float J[9], dd = 0.f, en = 0.f, mstep = 1e10f;
#pragma unroll
    for (int k = 0; k < 9; k++) J[k] = 0.f;
    bool ok = wasGood;
    if (wasGood) {  // L390-455, this lane's pattern pixel
      const float x = pu + pdx, y = pv + pdy;
      const float p0 = P.RKi[0] * x + P.RKi[1] * y + P.RKi[2] + P.t[0] * id;
      const float p1 = P.RKi[3] * x + P.RKi[4] * y + P.RKi[5] + P.t[1] * id;
      const float p2 = P.RKi[6] * x + P.RKi[7] * y + P.RKi[8] + P.t[2] * id;
      const float uu = p0 / p2, vv = p1 / p2;
      const float Ku = P.fx * uu + P.cx, Kv = P.fy * vv + P.cy;
      const float new_idepth = id / p2;
      ok = Ku > 1.f && Kv > 1.f && Ku < (float)(P.w - 2) && Kv < (float)(P.h - 2) && new_idepth > 0.f;
      if (ok) {
        const float4 hit = ci_bilin(imgNew, Ku, Kv, P.w);
        const float rlR = ci_bilin(imgRef, x, y, P.w).x;
        ok = isfinite(rlR) && isfinite(hit.x);
        if (ok) {
          const float residual = hit.x - P.aff0 * rlR - P.aff1;
          const float ar = fabsf(residual);
          float hw = ar < P.huber ? 1.f : P.huber / ar;
          en = hw * residual * residual * (2.f - hw);
          const float dxdd = (P.t[0] - P.t[2] * uu) / p2, dydd = (P.t[1] - P.t[2] * vv) / p2;
          if (hw < 1.f) hw = sqrtf(hw);
          const float dxI = hw * hit.y * P.fx, dyI = hw * hit.z * P.fy;
          J[0] = new_idepth * dxI;
          J[1] = new_idepth * dyI;
          J[2] = -new_idepth * (uu * dxI + vv * dyI);
          J[3] = -uu * vv * dxI - (1.f + vv * vv) * dyI;
          J[4] = (1.f + uu * uu) * dxI + uu * vv * dyI;
          J[5] = -vv * dxI + uu * dyI;
          J[6] = -hw * P.aff0 * rlR;
          J[7] = -hw;
          J[8] = hw * residual;
          dd = dxI * dxdd + dyI * dydd;
          const float mx = dxdd * P.fx, my = dydd * P.fy;
          mstep = fminf(1e10f, 1.0f / sqrtf(mx * mx + my * my));   // `if (maxstep < point->maxstep)` from 1e10 (L371, L447-448)
        }
      }
    }
    // the point's verdict and its JbBuffer row: sums over the 8 lanes of the group (every lane ends with the totals)
    const unsigned grp = 0xffu << (lane & 24);
    const bool allok = (__ballot_sync(0xffffffffu, ok) & grp) == grp;
    float Jb[10];
#pragma unroll
    for (int k = 0; k < 8; k++) Jb[k] = ci_group_sum(J[k] * dd);
    Jb[8] = ci_group_sum(J[8] * dd);
    Jb[9] = ci_group_sum(dd * dd);
    const float energy = ci_group_sum(en);
    mstep = fminf(mstep, __shfl_xor_sync(0xffffffffu, mstep, 4));
    mstep = fminf(mstep, __shfl_xor_sync(0xffffffffu, mstep, 2));
    mstep = fminf(mstep, __shfl_xor_sync(0xffffffffu, mstep, 1));
    const bool good = wasGood && allok && !(energy > __ldg(Q.outlierTH + ii) * 20.f);   // L457-466
    // Schur row (L562-586): alphaOpt is known before the launch (see the file header)
    const float lastH = Jb[9];
    if (good) {
      Jb[8] += P.alphaOpt * (id - 1.f);
      Jb[9] += P.alphaOpt;
      if (P.alphaOpt == 0.f) {
        Jb[8] += P.coupling * (id - __ldg(Q.iR + ii));
        Jb[9] += P.coupling;
      }
      Jb[9] = 1.f / (1.f + Jb[9]);
    }
    const float g = good ? 1.f : 0.f;
    const float wsc = (good && px == 0) ? Jb[9] : 0.f;   // one lane of the group carries the point's Schur contribution
    {
      int e = 0;
#pragma unroll
      for (int r = 0; r < 9; r++) {
        const float Jr = J[r] * g, Sr = Jb[r] * wsc;
#pragma unroll
        for (int c = r; c < 9; c++, e++) { acc[e] += Jr * J[c]; accsc[e] += Sr * Jb[c]; }
      }
    }
    if (px == 0 && have) {
      accE += good ? energy : e0;   // E.updateSingle (L386, L459, L468)
      accN += g;
      Q.isGood_new[i] = good ? 1 : 0;
      Q.energy_new[2 * i] = good ? energy : e0;
      Q.energy_new[2 * i + 1] = good ? (id - 1.f) * (id - 1.f) : e1;   // L531-540
      Q.maxstep[i] = mstep;
      Q.lastHessian_new[i] = good ? lastH : 0.f;
    }
    if (have && px < 5) {  // the row as it stands after L562-586 (read by doStep, L919-946); zeros for points that are not good
      Q.Jb[(size_t)10 * i + 2 * px] = good ? Jb[2 * px] : 0.f;
      Q.Jb[(size_t)10 * i + 2 * px + 1] = good ? Jb[2 * px + 1] : 0.f;
    }
  }

  // block reduction: warp shuffles, warp partials through shared memory, fp64 per-CTA partial
  auto wsum = [](float a) {
    a += __shfl_xor_sync(0xffffffffu, a, 16);
    a += __shfl_xor_sync(0xffffffffu, a, 8);
    a += __shfl_xor_sync(0xffffffffu, a, 4);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    return a;
  };
#pragma unroll
  for (int e = 0; e < 45; e++) {
    const float a = wsum(acc[e]), b = wsum(accsc[e]);
    if (lane == 0) { s_red[warp][e] = a; s_red[warp][45 + e] = b; }
  }
  {
    const float a = wsum(accE), b = wsum(accN);
    if (lane == 0) { s_red[warp][90] = a; s_red[warp][91] = b; s_red[warp][92] = 0.f; }
  }
  __syncthreads();
  if (tid < CI_NRED) {
    double s = 0.0;
#pragma unroll
    for (int wv = 0; wv < CI_THREADS / 32; wv++) s += (double)s_red[wv][tid];
    partial[(size_t)blockIdx.x * CI_NRED + tid] = s;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last) {
    __threadfence();
    if (tid < CI_NRED) {
      double s = 0.0;
      for (int bk = 0; bk < (int)gridDim.x; bk++) s += __ldcg(&partial[(size_t)bk * CI_NRED + tid]);
      out[tid] = s;
    }
    if (tid == 0) *ticket = 0u;
  }
}

}  // namespace dmv

using namespace dmv;

struct dmv_ci {
  dmv_ci_config cfg;
  int device = 0;
  Stream stream;
  int w[DMV_MAX_PYR_LEVELS], h[DMV_MAX_PYR_LEVELS], n[DMV_MAX_PYR_LEVELS];
  float fx[DMV_MAX_PYR_LEVELS], fy[DMV_MAX_PYR_LEVELS], cx[DMV_MAX_PYR_LEVELS], cy[DMV_MAX_PYR_LEVELS];
  bool haveK[DMV_MAX_PYR_LEVELS], haveFirst[DMV_MAX_PYR_LEVELS], haveNew[DMV_MAX_PYR_LEVELS];
  DevBuf<float4> d_first[DMV_MAX_PYR_LEVELS], d_new[DMV_MAX_PYR_LEVELS];
  DevBuf<float> d_stage;                    // AoS3 staging of one level-0 plane
  DevBuf<float> d_static[DMV_MAX_PYR_LEVELS];   // u | v | outlierTH          (3 * max_points)
  DevBuf<float> d_in;                       // idepth_new | energy(2) | iR           (4 * max_points)
  DevBuf<unsigned char> d_good;             // isGood | isGood_new                   (2 * max_points)
  DevBuf<float> d_outp;                     // energy_new(2) | maxstep | lastHessian_new | Jb(10)   (14 * max_points)
  PinnedBuf<float> h_pin;                   // pinned staging, 18 * max_points floats + bytes
  DevBuf<double> d_partial, d_out;
  PinnedBuf<double> h_out;
  DevBuf<unsigned int> d_ticket;
  int grid_max = 0;
  long long launches = 0;
};

extern "C" {

static int ci_allocate(dmv_ci* c, const dmv_ci_config* cfg);

int dmv_ci_create(const dmv_ci_config* cfg, dmv_ci** out) {
  if (!cfg || !out) return set_error(DMV_ERR_INVALID, "null argument");
  if (cfg->w < 16 || cfg->h < 16 || cfg->levels < 1 || cfg->levels > DMV_MAX_PYR_LEVELS || cfg->max_points < 1)
    return set_error(DMV_ERR_INVALID, "bad dmv_ci_config");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return set_error(DMV_ERR_NO_DEVICE, "no CUDA device: dmvio_b200 has no CPU path");
  if (cfg->device < 0 || cfg->device >= ndev) return set_error(DMV_ERR_INVALID, "device %d out of range", cfg->device);
  CK(cudaSetDevice(cfg->device));
  dmv_ci* c = new dmv_ci();
  const int rc = ci_allocate(c, cfg);
  if (rc != DMV_OK) {  // allocation failed half-way: the members release what exists, the failing call's error message is kept
    delete c;
    return rc;
  }
  *out = c;
  return DMV_OK;
}

static int ci_allocate(dmv_ci* c, const dmv_ci_config* cfg) {
  c->cfg = *cfg;
  c->device = cfg->device;
  CK(cudaStreamCreateWithFlags(c->stream.put(), cudaStreamNonBlocking));
  const size_t mp = (size_t)cfg->max_points;
  for (int l = 0; l < cfg->levels; l++) {
    c->w[l] = cfg->w >> l; c->h[l] = cfg->h >> l; c->n[l] = 0;
    c->haveK[l] = c->haveFirst[l] = c->haveNew[l] = false;
    CK(c->d_first[l].alloc((size_t)c->w[l] * c->h[l]));
    CK(c->d_new[l].alloc((size_t)c->w[l] * c->h[l]));
    CK(c->d_static[l].alloc(3 * mp));
  }
  CK(c->d_stage.alloc(3 * (size_t)cfg->w * cfg->h));
  CK(c->d_in.alloc(4 * mp));
  CK(c->d_good.alloc(2 * mp));
  CK(c->d_outp.alloc(14 * mp));
  CK(c->h_pin.alloc(20 * mp));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
  c->grid_max = 2 * sms;
  CK(c->d_partial.alloc((size_t)CI_NRED * c->grid_max));
  CK(c->d_out.alloc(CI_NRED));
  CK(c->h_out.alloc(CI_NRED));
  CK(c->d_ticket.alloc(1));
  CK(cudaMemset(c->d_ticket, 0, sizeof(unsigned int)));
  return DMV_OK;
}

int dmv_ci_destroy(dmv_ci* c) {
  if (!c) return DMV_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  delete c;
  return DMV_OK;
}

int dmv_ci_set_K(dmv_ci* c, int l, float fx, float fy, float cx, float cy) {
  if (!c || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "level out of range");
  c->fx[l] = fx; c->fy[l] = fy; c->cx[l] = cx; c->cy[l] = cy; c->haveK[l] = true;
  return DMV_OK;
}

static int ci_upload(dmv_ci* c, int l, const float* dIp, float4* dst) {
  const size_t npx = (size_t)c->w[l] * c->h[l];
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->d_stage, dIp, sizeof(float) * 3 * npx, cudaMemcpyHostToDevice, c->stream));
  launch_repack(c->d_stage, dst, (int)npx, c->stream);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));   // pageable source + shared staging buffer
  return DMV_OK;
}
int dmv_ci_upload_first(dmv_ci* c, int l, const float* dIp) {
  if (!c || !dIp || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad argument");
  const int rc = ci_upload(c, l, dIp, c->d_first[l]);
  if (rc == DMV_OK) c->haveFirst[l] = true;
  return rc;
}
int dmv_ci_upload_new(dmv_ci* c, int l, const float* dIp) {
  if (!c || !dIp || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad argument");
  const int rc = ci_upload(c, l, dIp, c->d_new[l]);
  if (rc == DMV_OK) c->haveNew[l] = true;
  return rc;
}

int dmv_ci_set_points(dmv_ci* c, int l, int n, const float* u, const float* v, const float* outlierTH) {
  if (!c || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "level out of range");
  if (n < 0 || n > c->cfg.max_points || (n > 0 && (!u || !v || !outlierTH))) return set_error(DMV_ERR_INVALID, "bad point set (capacity %d)", c->cfg.max_points);
  CK(cudaSetDevice(c->device));
  const size_t mp = (size_t)c->cfg.max_points;
  if (n > 0) {
    std::memcpy(c->h_pin, u, sizeof(float) * n); std::memcpy(c->h_pin + mp, v, sizeof(float) * n); std::memcpy(c->h_pin + 2 * mp, outlierTH, sizeof(float) * n);
    CK(cudaMemcpyAsync(c->d_static[l], c->h_pin, sizeof(float) * 3 * mp, cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  c->n[l] = n;
  return DMV_OK;
}

int dmv_ci_calc_res_and_gs(dmv_ci* c, const dmv_ci_eval_args* a, dmv_ci_eval_result* r) {
  if (!c || !a || !r) return set_error(DMV_ERR_INVALID, "null argument");
  const int l = a->level;
  if (l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "level out of range");
  if (!c->haveK[l] || !c->haveFirst[l] || !c->haveNew[l]) return set_error(DMV_ERR_STATE, "dmv_ci_set_K + dmv_ci_upload_first + dmv_ci_upload_new first");
  const int n = c->n[l];
  if (n < 1) return set_error(DMV_ERR_STATE, "dmv_ci_set_points first");
  if (!a->idepth_new || !a->isGood || !a->energy2 || !a->iR) return set_error(DMV_ERR_INVALID, "incomplete dmv_ci_eval_args");
  CK(cudaSetDevice(c->device));
  const size_t mp = (size_t)c->cfg.max_points;
  // L544-557: EAlpha is never updated by the reference (its alpha loop feeds E instead), so alphaEnergy depends on the pose alone.  The
  // reference evaluates alphaW * (EAlpha.A + |t|^2 * npts) in double and rounds ONCE, on assignment (L540): rounding |t|^2 * npts to float
  // first and multiplying in float is 1 ulp off for about a third of the poses, and near alphaW |t|^2 = alphaK it flips the cap below (alphaOpt
  // alphaW <-> 0) and the caller's `res3[1] == alphaK * npts` snap test.
  const double tsq = (double)a->t_d[0] * a->t_d[0] + (double)a->t_d[1] * a->t_d[1] + (double)a->t_d[2] * a->t_d[2];
  float alphaEnergy = (float)((double)a->alphaW * (0.0 + tsq * n));
  float alphaOpt;
  if (alphaEnergy > a->alphaK * n) { alphaOpt = 0.f; alphaEnergy = a->alphaK * n; }
  else alphaOpt = a->alphaW;
  // per-evaluation point state: one pinned block, one copy
  float* hp = c->h_pin;
  std::memcpy(hp, a->idepth_new, sizeof(float) * n);
  std::memcpy(hp + mp, a->energy2, sizeof(float) * 2 * n);
  std::memcpy(hp + 3 * mp, a->iR, sizeof(float) * n);
  unsigned char* hb = reinterpret_cast<unsigned char*>(hp + 4 * mp);
  std::memcpy(hb, a->isGood, n);
  CK(cudaMemcpyAsync(c->d_in, hp, sizeof(float) * 4 * mp, cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(c->d_good, hb, n, cudaMemcpyHostToDevice, c->stream));
  CIParams P;
  for (int i = 0; i < 9; i++) P.RKi[i] = a->RKi[i];
  for (int i = 0; i < 3; i++) P.t[i] = (float)a->t_d[i];
  P.fx = c->fx[l]; P.fy = c->fy[l]; P.cx = c->cx[l]; P.cy = c->cy[l];
  P.aff0 = a->r2new_aff[0]; P.aff1 = a->r2new_aff[1];
  P.huber = a->huberTH; P.alphaOpt = alphaOpt; P.coupling = a->couplingWeight;
  P.w = c->w[l]; P.h = c->h[l]; P.n = n;
  CIPoints Q;
  Q.u = c->d_static[l]; Q.v = c->d_static[l] + mp; Q.outlierTH = c->d_static[l] + 2 * mp;
  Q.idepth_new = c->d_in; Q.energy = c->d_in + mp; Q.iR = c->d_in + 3 * mp;
  Q.isGood = c->d_good; Q.isGood_new = c->d_good + mp;
  Q.energy_new = c->d_outp; Q.maxstep = c->d_outp + 2 * mp; Q.lastHessian_new = c->d_outp + 3 * mp; Q.Jb = c->d_outp + 4 * mp;
  const int grid = std::max(1, std::min(c->grid_max, (n + CI_THREADS / 8 - 1) / (CI_THREADS / 8)));
  ci_res_gs_kernel<<<grid, CI_THREADS, 0, c->stream>>>(P, Q, c->d_first[l], c->d_new[l], c->d_partial, c->d_ticket, c->d_out);
  CK(cudaGetLastError());
  c->launches++;
  CK(cudaMemcpyAsync(c->h_out, c->d_out, sizeof(double) * CI_NRED, cudaMemcpyDeviceToHost, c->stream));
  float* ho = hp + 5 * mp;  // outputs behind the inputs in the pinned block
  unsigned char* hgo = reinterpret_cast<unsigned char*>(hp + 19 * mp);
  CK(cudaMemcpyAsync(ho, c->d_outp, sizeof(float) * 14 * mp, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(hgo, c->d_good + mp, n, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  if (a->isGood_new) std::memcpy(a->isGood_new, hgo, n);
  if (a->energy_new2) std::memcpy(a->energy_new2, ho, sizeof(float) * 2 * n);
  if (a->maxstep) std::memcpy(a->maxstep, ho + 2 * mp, sizeof(float) * n);
  if (a->lastHessian_new) std::memcpy(a->lastHessian_new, ho + 3 * mp, sizeof(float) * n);
  if (a->JbBuffer_new10) std::memcpy(a->JbBuffer_new10, ho + 4 * mp, sizeof(float) * 10 * n);
  // Accumulator9 -> H_out / b_out (L588-611)
  const double* o = c->h_out;
  float H9[9][9], S9[9][9];
  int e = 0;
  for (int i = 0; i < 9; i++)
    for (int j = i; j < 9; j++, e++) { H9[i][j] = H9[j][i] = (float)o[e]; S9[i][j] = S9[j][i] = (float)o[45 + e]; }
  for (int i = 0; i < 8; i++) {
    for (int j = 0; j < 8; j++) { r->H[i * 8 + j] = H9[i][j]; r->Hsc[i * 8 + j] = S9[i][j]; }
    r->b[i] = H9[i][8]; r->bsc[i] = S9[i][8];
  }
  r->H[0] += alphaOpt * n; r->H[9] += alphaOpt * n; r->H[18] += alphaOpt * n;
  for (int k = 0; k < 3; k++) r->b[k] += (float)a->t_log[k] * alphaOpt * n;
  r->H[9] = (float)(r->H[9] + a->weightZeroPriorY);
  r->b[1] = (float)(r->b[1] + a->weightZeroPriorY * a->t_d[1]);
  r->H[0] = (float)(r->H[0] + a->weightZeroPriorX);
  r->b[0] = (float)(r->b[0] + a->weightZeroPriorX * a->t_d[0]);
  r->res3[0] = (float)o[90];       // E.A of the first pass (the alpha pass adds to E after its finish(): A unchanged, num grows)
  r->res3[1] = alphaEnergy;
  r->res3[2] = (float)(2 * n);     // E.num: one updateSingle per point in each of the two passes
  r->alphaOpt = alphaOpt;
  r->n_good_new = (int)o[91];
  return DMV_OK;
}

int dmv_ci_kernel_launch_count(dmv_ci* c, long long* n) {
  if (!c || !n) return set_error(DMV_ERR_INVALID, "null argument");
  *n = c->launches;
  return DMV_OK;
}

}  // extern "C"
