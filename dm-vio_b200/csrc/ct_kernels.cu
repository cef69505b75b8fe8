// sm_90a kernels + C-ABI of the coarse direct-image-alignment path (DESIGN.md §5).
//
//   ct_res_gs_kernel   CoarseTracker::calcRes (CoarseTracker.cpp:L361-517) fused with calcGSSSE (L299-356): one thread per
//                      reference point: project, 4-tap float4 gather from the new frame's level plane, Huber residual,
//                      energy / saturation counters / flow indicators and the 45 unique entries of the weighted 9x9
//                      outer product.  Block reduction (ct_block_sum), per-block fp64 partials, and the last
//                      block to finish (threadfence + ticket) folds the partials in a fixed order -> deterministic, one launch.
//                      The buf_warped_* lists of the reference are never materialised.
//   ct_track_cluster_kernel   CoarseTracker::trackNewestCoarse in one launch (below).
//   ct_track_many_kernel      the same for up to DMV_CT_TRACK_MANY_MAX handles in one launch, one cluster per handle.
//   ct_track_tries_kernel     FullSystem::trackNewCoarse's loop over up to DMV_CT_MAX_TRIES initial poses in one launch.
//   ct_track_tries_many_kernel   the same for up to DMV_CT_TRACK_MANY_MAX handles in one launch, one cluster per handle.
// The entry points of the features built on the handle's resident frame live beside their kernels: ct_ingest.cu (raw frames), ct_depth.cu
// (makeCoarseDepthL0), ip_trace.cu (immature points) and ps_select.cu (pixel selection); the handle's layout is ct_handle.h.
#include "ct_handle.h"
#include "inv3.h"
#include <cuda.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>

namespace dmv {

constexpr int CT_NRED = 45 + 8;  // 45 outer-product entries + E, nE, nSat, nWarped, shiftT, shiftRT, shiftNum, pad
constexpr int CT_THREADS = 256;

struct CTParams {
  float RKi[9], t[3], Ki[9];
  float fx, fy, cx, cy;
  float affa, affb, a_gs, b0;
  float cutoff, huber, maxEnergy;
  int w, h, n, lvl, want_gs;
};

// one reference point (x, y, id, refColor): CoarseTracker::calcRes (L399-483) + its row of calcGSSSE (L316-336), added into v[]; the 4 taps
// come from the level plane in shared memory (SMEM: staged by TMA, plane_s) or from global memory (img)
template <bool SMEM>
__device__ __forceinline__ void ct_eval_accumulate(const CTParams& P, int i, const float x, const float y, const float id, const float refColor,
                                                   const float4* __restrict__ img, const float4* plane_s, float v[64]) {
  const float p0 = P.RKi[0] * x + P.RKi[1] * y + P.RKi[2] + P.t[0] * id;
  const float p1 = P.RKi[3] * x + P.RKi[4] * y + P.RKi[5] + P.t[1] * id;
  const float p2 = P.RKi[6] * x + P.RKi[7] * y + P.RKi[8] + P.t[2] * id;
  const float u = p0 / p2, vv = p1 / p2;
  const float Ku = P.fx * u + P.cx, Kv = P.fy * vv + P.cy;
  const float new_idepth = id / p2;
  if (P.lvl == 0 && (i & 31) == 0) {  // flow indicators (CoarseTracker.cpp:L416-447)
    const float k0 = P.Ki[0] * x + P.Ki[1] * y + P.Ki[2], k1 = P.Ki[3] * x + P.Ki[4] * y + P.Ki[5], k2 = P.Ki[6] * x + P.Ki[7] * y + P.Ki[8];
    const float T0 = k0 + P.t[0] * id, T1 = k1 + P.t[1] * id, T2 = k2 + P.t[2] * id;
    const float M0 = k0 - P.t[0] * id, M1 = k1 - P.t[1] * id, M2 = k2 - P.t[2] * id;
    const float q0 = P.RKi[0] * x + P.RKi[1] * y + P.RKi[2] - P.t[0] * id;
    const float q1 = P.RKi[3] * x + P.RKi[4] * y + P.RKi[5] - P.t[1] * id;
    const float q2 = P.RKi[6] * x + P.RKi[7] * y + P.RKi[8] - P.t[2] * id;
    const float KuT = P.fx * (T0 / T2) + P.cx, KvT = P.fy * (T1 / T2) + P.cy;
    const float KuT2 = P.fx * (M0 / M2) + P.cx, KvT2 = P.fy * (M1 / M2) + P.cy;
    const float Ku3 = P.fx * (q0 / q2) + P.cx, Kv3 = P.fy * (q1 / q2) + P.cy;
    v[49] += (KuT - x) * (KuT - x) + (KvT - y) * (KvT - y) + (KuT2 - x) * (KuT2 - x) + (KvT2 - y) * (KvT2 - y);
    v[50] += (Ku - x) * (Ku - x) + (Kv - y) * (Kv - y) + (Ku3 - x) * (Ku3 - x) + (Kv3 - y) * (Kv3 - y);
    v[51] += 2.f;
  }
  if (Ku > 2.f && Kv > 2.f && Ku < (float)(P.w - 3) && Kv < (float)(P.h - 3) && new_idepth > 0.f) {
    const int ix = (int)Ku, iy = (int)Kv;
    const float dx = Ku - ix, dy = Kv - iy, dxdy = dx * dy;
    float4 tl, tr, bl, br;
    if constexpr (SMEM) {
      const float4* bp = plane_s + iy * P.w + ix;
      tl = bp[0]; tr = bp[1]; bl = bp[P.w]; br = bp[P.w + 1];
    } else {
      const float4* bp = img + (size_t)iy * P.w + ix;
      tl = __ldg(bp); tr = __ldg(bp + 1); bl = __ldg(bp + P.w); br = __ldg(bp + P.w + 1);
    }
    const float w11 = dxdy, w10 = dy - dxdy, w01 = dx - dxdy, w00 = 1 - dx - dy + dxdy;
    const float h0 = w11 * br.x + w10 * bl.x + w01 * tr.x + w00 * tl.x;
    const float h1 = w11 * br.y + w10 * bl.y + w01 * tr.y + w00 * tl.y;
    const float h2 = w11 * br.z + w10 * bl.z + w01 * tr.z + w00 * tl.z;
    if (isfinite(h0)) {
      const float residual = h0 - (P.affa * refColor + P.affb);
      const float ar = fabsf(residual);
      const float hw = ar < P.huber ? 1.f : P.huber / ar;
      if (ar > P.cutoff) {
        v[45] += P.maxEnergy; v[46] += 1.f; v[47] += 1.f;
      } else {
        v[45] += hw * residual * residual * (2.f - hw); v[46] += 1.f; v[48] += 1.f;
        if (P.want_gs) {  // calcGSSSE row (L316-336) and Accumulator9::updateSSE_eighted (MatrixAccumulators.h:L1091-1166)
          const float gx = h1 * P.fx, gy = h2 * P.fy;
          float J[9];
          J[0] = new_idepth * gx;
          J[1] = new_idepth * gy;
          J[2] = 0.f - new_idepth * (u * gx + vv * gy);
          J[3] = 0.f - ((u * vv) * gx + gy * (1.f + vv * vv));
          J[4] = (u * vv) * gy + gx * (1.f + u * u);
          J[5] = u * gy - vv * gx;
          J[6] = P.a_gs * (P.b0 - refColor);
          J[7] = -1.f;
          J[8] = residual;
          int e = 0;
#pragma unroll
          for (int r = 0; r < 9; r++) {
            const float Jw = J[r] * hw;
#pragma unroll
            for (int c = r; c < 9; c++) v[e++] += Jw * J[c];
          }
        }
      }
    }
  }
}

// block reduction of the 53 sums of a block of NW warps (v[53..63] = 0 pads; v is overwritten).  Per warp a transposing butterfly: 62
// shuffles, after which lane L holds the warp sums of entries 2L and 2L+1.  It pairs lanes at distance 16, 8, 4, 2, 1, the addition tree
// of a per-entry xor reduction (53 x 5 shuffles), and gives the same bits.  Then thread k < CT_NRED returns the sum of entry k over the
// warps, in fp64 and in warp order.
template <int NW>
__device__ __forceinline__ double ct_block_sum(float v[64], float (*red)[64]) {
  static_assert(CT_NRED <= 64, "");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int st = 0; st < 5; st++) {
    const int hstep = 32 >> st, m = 16 >> st;
    const bool up = (lane & m) != 0;
#pragma unroll
    for (int k = 0; k < 32; k++)
      if (k < hstep) v[k] = (up ? v[k + hstep] : v[k]) + __shfl_xor_sync(0xffffffffu, up ? v[k] : v[k + hstep], m);
  }
  red[warp][2 * lane] = v[0];
  red[warp][2 * lane + 1] = v[1];
  __syncthreads();
  double sm = 0.0;
  if (threadIdx.x < CT_NRED) {
#pragma unroll
    for (int wv = 0; wv < NW; wv++) sm += (double)red[wv][threadIdx.x];
  }
  return sm;
}

// fold of the per-CTA fp64 partials in a FIXED order with the loads in flight together: thread (q, k) adds quarter q of the CTAs for
// entry k (independent loads, batches of 8), then thread k adds the four quarter sums.  A plain `for (bk) s += partial[bk]` loop issues
// one L2 round trip per CTA (~0.35 us each, 13 us for 39 CTAs) because every add waits for its own load.
__device__ __forceinline__ void ct_fold(const double* __restrict__ partial, int G, double (*s_q)[CT_NRED], double* s_sum) {
  const int tid = threadIdx.x;
  if (tid < 4 * CT_NRED) {
    const int q = tid / CT_NRED, k = tid - q * CT_NRED;
    const int per = (G + 3) >> 2, b0 = q * per, b1 = min(G, b0 + per);
    double sm = 0.0;
    for (int bk = b0; bk < b1; bk += 8) {
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; u++) v[u] = (bk + u < b1) ? __ldcg(&partial[(size_t)(bk + u) * CT_NRED + k]) : 0.0;
#pragma unroll
      for (int u = 0; u < 8; u++) sm += v[u];
    }
    s_q[q][k] = sm;
  }
  __syncthreads();
  if (tid < CT_NRED) s_sum[tid] = ((s_q[0][tid] + s_q[1][tid]) + s_q[2][tid]) + s_q[3][tid];
}

__global__ void __launch_bounds__(CT_THREADS) ct_res_gs_kernel(CTParams P, const float* __restrict__ pc_u, const float* __restrict__ pc_v,
                                                               const float* __restrict__ pc_id, const float* __restrict__ pc_col,
                                                               const float4* __restrict__ img, double* __restrict__ partial,
                                                               unsigned int* __restrict__ ticket, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float v[64];
#pragma unroll
  for (int k = 0; k < 64; k++) v[k] = 0.f;
  if (i < P.n) ct_eval_accumulate<false>(P, i, pc_u[i], pc_v[i], pc_id[i], pc_col[i], img, nullptr, v);
  __shared__ float s_red[CT_THREADS / 32][64];
  const double bs = ct_block_sum<CT_THREADS / 32>(v, s_red);
  if (threadIdx.x < CT_NRED) partial[(size_t)blockIdx.x * CT_NRED + threadIdx.x] = bs;
  // ---- last block folds the per-block partials in block order
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int tk = atomicAdd(ticket, 1u);
    s_last = (tk == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {  // block-uniform
    __threadfence();
    __shared__ double s_q[4][CT_NRED];
    __shared__ double s_sum[CT_NRED];
    ct_fold(partial, (int)gridDim.x, s_q, s_sum);
    __syncthreads();
    if (threadIdx.x < CT_NRED) out[threadIdx.x] = s_sum[threadIdx.x];
    if (threadIdx.x == 0) *ticket = 0u;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// The state machine of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:L539-770, visual-only branch L639-683), which lets
// ct_track_cluster_kernel run the whole Levenberg-Marquardt loop over all pyramid levels in ONE launch instead of ~21 launch + sync
// round trips per frame.  CTTrack holds the launch's inputs; CTLM is the scalar state, one copy per CTA in shared memory.  After each
// evaluation every CTA holds the same folded sums, and warp 0 advances its copy in double (ct_advance_warp: accept/reject, level
// schedule, damped 8x8 system, LDL^T, SE3 exp, the operands of the next evaluation).  Identical inputs give identical decisions in every
// CTA, so no broadcast is needed.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int CT_L = DMV_MAX_PYR_LEVELS;
// a track's result in the handle's pinned block h_out, which also takes ct_res_gs_kernel's 53 sums; written by CTA 0 of the cluster
struct CTTrackOut {
  double R[9], t[3], a, b, lastResiduals[5], flow[3];
  double good, iterations, evaluations, status;
  double pevals;   // dmv_ct_last_point_evaluations; the tries kernels write only this
};
static_assert(sizeof(CTTrackOut) == 27 * sizeof(double), "CTTrackOut must fit the first 27 of h_out's 64 doubles");
struct CTTrack {
  int levels, coarsest;
  int n[CT_L], w[CT_L], h[CT_L];
  float fx[CT_L], fy[CT_L], cx[CT_L], cy[CT_L];
  float Ki[CT_L][9];
  const float *u[CT_L], *v[CT_L], *id[CT_L], *col[CT_L];
  const float4* img[CT_L];
  double R0[9], t0[3], a0, b0;   // lastToNew_out / aff_g2l_out on entry
  double ref_a, ref_b;           // lastRef_aff_g2l
  float ref_exposure, new_exposure;
  float huber, cutoffTH, affModeA, affModeB;
  double minRes[5];
  int staged[CT_L];              // level l's plane is TMA-staged (ct_make_tensor_maps encoded its map)
  CTTrackOut* out;              // pinned host
};

struct CTLM {  // the scalar state of trackNewestCoarse, one copy per CTA (shared memory), advanced by thread 0
  double R[9], t[3], a, b;          // refToNew_current, aff_g2l_current
  double Rn[9], tn[3], an, bn;      // candidate
  double H[2][64], bb[2][8], res[2][6];   // [cur]: linearisation at the current pose (resOld); [cur^1]: the evaluation that just finished
  int cur;
  double inc[8];
  double lastResiduals[5], flow[3];
  float RKi[9], tf[3], affLL[2], cutoff;  // operands of the pending evaluation
  float lambda, rep;
  int lvl, iteration, phase, haveRepeated, iterations, evaluations, done, good, status;
  double A[64], rhs[8], Lf[64], Df[8], incs[8], EV[18];   // the damped 8x8 system of the pending LM step, its LDL^T factors, its solution
  double pevals;                  // sum over the evaluations of the level's reference-point count (measurement: algorithmic bytes = 64 B each)
  int need_solve, need_request;   // need_request: 1 = evaluate at (R, t, a, b), 2 = at the candidate (Rn, tn, an, bn) = exp(incs) * (R, t)
  double minRes[5];               // minResForAbort: T.minRes, or in ct_track_tries_kernel the loop's achievedRes (CTLoop)
};
enum { CT_PH_INIT = 0, CT_PH_LM = 1 };

// Vec6 of calcRes (L508-516) and H, b of calcGSSSE (L341-355) from the 53 folded sums, one output per thread (tid < 78)
__device__ __forceinline__ void ct_finish_parallel(const double* o, double* res6, double* H, double* b, int tid) {
  const int npad = ((int)o[48] + 3) & ~3;
  const double inv = (double)(1.0f / (float)npad);
  if (tid < 72) {
    const int r = tid >> 3, c = (tid < 64) ? (tid & 7) : 8;   // tid 64..71: r = 8 -> handled below as the b column
    const int rr = (tid < 64) ? r : (tid - 64);
    const int lo = rr < c ? rr : c, hi = rr < c ? c : rr;
    const int e = lo * 9 - (lo * (lo - 1)) / 2 + (hi - lo);     // upper-triangular index of the 9x9 accumulator
    const double scr = (rr == 6) ? 10.0 : (rr == 7 ? 1000.0 : 1.0);
    if (tid < 64) {
      const double scc = (c == 6) ? 10.0 : (c == 7 ? 1000.0 : 1.0);
      H[rr * 8 + c] = o[e] * inv * scr * scc;
    } else {
      b[rr] = o[e] * inv * scr;
    }
  } else if (tid == 72) {
    res6[0] = o[45]; res6[1] = o[46];
    res6[2] = (double)((float)o[49] / ((float)o[51] + 0.1f));
    res6[3] = 0;
    res6[4] = (double)((float)o[50] / ((float)o[51] + 0.1f));
    res6[5] = (double)((float)o[47] / (float)o[46]);
  }
}
__device__ void ct_begin_level(const CTTrack& T, CTLM& S) {
  S.rep = 1.f;
  S.phase = CT_PH_INIT;
  S.need_request = 1;   // evaluate at the current pose
}
// Hl.ldlt().solve(-b) for the 8x8 system (L639-665): plain LDL^T (ct_factor_warp / ct_propose_post below).  A parameter that is not
// optimised (setting_affineOptModeA/B < 0: the reference solves the 6x6 / 7x7 sub-system) is padded with an identity row/column and a zero
// right-hand side: the extra terms are exact zeros, the other components come out bit-identical.
// one LM trial step from the current linearisation (L605-683), in three parts: the warp sets up the damped system and factorises it
// (row i of L in lane i: the 8^3/3 multiply-adds and the 28 divisions of the scalar version collapse to 8 dependent column steps), lane 0
// substitutes and updates the pose.  Every element sees the same operations in the same order as the scalar LDL^T: bit-identical result.
__device__ void ct_propose_pre(const CTTrack& T, CTLM& S) {  // lane 0: bookkeeping only; the damped system is built by the warp (ct_build_system_warp)
  S.iterations++;
  S.need_solve = 1;
}
__device__ __forceinline__ void ct_build_system_warp(const CTTrack& T, CTLM& S) {
  const int lane = threadIdx.x & 31;
  const double* Hc = S.H[S.cur];
  const double* bc = S.bb[S.cur];
  const bool fixA = T.affModeA < 0, fixB = T.affModeB < 0;
#pragma unroll
  for (int e = lane; e < 64; e += 32) {
    const int i = e >> 3, j = e & 7;
    const bool fi = (i == 6 && fixA) || (i == 7 && fixB), fj = (j == 6 && fixA) || (j == 7 && fixB);
    double vv = Hc[e];
    if (i == j) vv *= (1 + S.lambda);
    S.A[e] = (fi || fj) ? ((i == j) ? 1.0 : 0.0) : vv;
  }
  if (lane < 8) {
    const bool fi = (lane == 6 && fixA) || (lane == 7 && fixB);
    S.rhs[lane] = fi ? 0.0 : -bc[lane];
  }
}
// LDL^T of S.A by one warp (all 32 lanes execute; lane i & 7 mirrors row i, lanes 0..7 write)
__device__ __forceinline__ void ct_factor_warp(CTLM& S) {
  const int lane = threadIdx.x & 31, i = lane & 7;
  double Ai[8], Li[8], D[8];
#pragma unroll
  for (int k = 0; k < 8; k++) { Ai[k] = S.A[i * 8 + k]; Li[k] = 0.0; }
#pragma unroll
  for (int j = 0; j < 8; j++) {
    double sm = Ai[j];
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k < j) {
        const double Ljk = __shfl_sync(0xffffffffu, Li[k], j);   // row j's entry (lane j's own row when i == j)
        sm -= Li[k] * Ljk * D[k];
      }
    const double dj = __shfl_sync(0xffffffffu, sm, j);
    D[j] = dj;
    if (i > j) Li[j] = dj != 0.0 ? sm / dj : 0.0;
  }
  if (lane < 8) {
#pragma unroll
    for (int k = 0; k < 8; k++) S.Lf[i * 8 + k] = Li[k];
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 8; k++) S.Df[k] = D[k];
    }
  }
}
__device__ void ct_propose_post(const CTTrack& T, CTLM& S) {
  double y[8], inc[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    double sm = S.rhs[i];
#pragma unroll
    for (int k = 0; k < 8; k++) if (k < i) sm -= S.Lf[i * 8 + k] * y[k];
    y[i] = sm;
  }
#pragma unroll
  for (int i = 0; i < 8; i++) y[i] = S.Df[i] != 0.0 ? y[i] / S.Df[i] : 0.0;
#pragma unroll
  for (int i = 7; i >= 0; i--) {
    double sm = y[i];
#pragma unroll
    for (int k = 0; k < 8; k++) if (k > i) sm -= S.Lf[k * 8 + i] * inc[k];
    inc[i] = sm;
  }
  float extrapFac = 1;
  const float lambdaExtrapolationLimit = 0.001f;
  if (S.lambda < lambdaExtrapolationLimit) extrapFac = sqrtf(sqrtf(lambdaExtrapolationLimit / S.lambda));
#pragma unroll
  for (int i = 0; i < 8; i++) inc[i] *= extrapFac;
  double incScaled[8];
#pragma unroll
  for (int i = 0; i < 8; i++) incScaled[i] = inc[i];
  incScaled[6] *= 10.0;    // SCALE_A
  incScaled[7] *= 1000.0;  // SCALE_B
  double ssum = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) ssum += incScaled[i];
  if (!isfinite(ssum)) {
#pragma unroll
    for (int i = 0; i < 8; i++) incScaled[i] = 0;
  }
#pragma unroll
  for (int i = 0; i < 8; i++) { S.incs[i] = incScaled[i]; S.inc[i] = inc[i]; }
  S.an = S.a + incScaled[6];
  S.bn = S.b + incScaled[7];
  S.phase = CT_PH_LM;
  S.need_solve = 0;
  S.need_request = 2;   // evaluate at the candidate exp(incs) * (R, t)
}
// SE3::exp(incs) * (R, t) -> (Rn, tn) and the operands of the next calcRes, spread over the lanes of warp 0: each lane forms one output
// element with the same expression in double a single thread would use.
__device__ __forceinline__ void ct_pose_request_warp(const CTTrack& T, CTLM& S, const bool from_candidate) {
  const int lane = threadIdx.x & 31;
  if (from_candidate) {
    const double* xi = S.incs;
    const double wx = xi[3], wy = xi[4], wz = xi[5];
    const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
    double ca, cb, cc;
    if (th < 1e-8) { ca = 1.0 - th2 / 6.0; cb = 0.5 - th2 / 24.0; cc = 1.0 / 6.0 - th2 / 120.0; }
    else { double sn, cs; sincos(th, &sn, &cs); ca = sn / th; cb = (1.0 - cs) / th2; cc = (th - sn) / (th2 * th); }
    const double W[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    if (lane < 18) {  // lanes 0..8: E = I + ca W + cb W^2, lanes 9..17: V = I + cb W + cc W^2
      const int e = lane % 9, i = e / 3, j = e - 3 * i;
      const double w2 = W[i * 3] * W[j] + W[i * 3 + 1] * W[3 + j] + W[i * 3 + 2] * W[6 + j];
      const double I = (e % 4 == 0) ? 1.0 : 0.0;
      S.EV[lane] = (lane < 9) ? I + ca * W[e] + cb * w2 : I + cb * W[e] + cc * w2;
    }
    __syncwarp();
    const double* E = S.EV;
    const double* V = S.EV + 9;
    if (lane < 9) {
      const int i = lane / 3, j = lane - 3 * i;
      S.Rn[lane] = E[i * 3] * S.R[j] + E[i * 3 + 1] * S.R[3 + j] + E[i * 3 + 2] * S.R[6 + j];
    } else if (lane < 12) {
      const int i = lane - 9;
      const double et = V[i * 3] * xi[0] + V[i * 3 + 1] * xi[1] + V[i * 3 + 2] * xi[2];
      S.tn[i] = E[i * 3] * S.t[0] + E[i * 3 + 1] * S.t[1] + E[i * 3 + 2] * S.t[2] + et;
    }
    __syncwarp();
  }
  // operands of calcRes (CoarseTracker.cpp:L377-379): RKi = R.cast<float>() * Ki[lvl], t.cast<float>(), affLL.cast<float>()
  const double* R = from_candidate ? S.Rn : S.R;
  const double* t = from_candidate ? S.tn : S.t;
  const double a = from_candidate ? S.an : S.a, b = from_candidate ? S.bn : S.b;
  if (lane < 9) {
    const int i = lane / 3, j = lane - 3 * i;
    const float* Ki = T.Ki[S.lvl];
    S.RKi[lane] = (float)R[i * 3] * Ki[j] + (float)R[i * 3 + 1] * Ki[3 + j] + (float)R[i * 3 + 2] * Ki[6 + j];
  } else if (lane < 12) {
    S.tf[lane - 9] = (float)t[lane - 9];
  } else if (lane == 12) {
    float eF = T.ref_exposure, eT = T.new_exposure;  // AffLight::fromToVecExposure (util/NumType.h:L174-186)
    if (eF == 0 || eT == 0) eT = eF = 1;
    const double aa = exp(a - T.ref_a) * eT / eF;
    S.affLL[0] = (float)aa;
    S.affLL[1] = (float)(b - aa * T.ref_b);
    S.cutoff = T.cutoffTH * S.rep;
    S.evaluations++;
    S.pevals += (double)T.n[S.lvl];
  }
}
__device__ void ct_end_level(const CTTrack& T, CTLM& S) {  // L722-745
  const int lvl = S.lvl;
  const double* resOld = S.res[S.cur];
  S.lastResiduals[lvl] = sqrtf((float)(resOld[0] / resOld[1]));
  S.flow[0] = resOld[2]; S.flow[1] = resOld[3]; S.flow[2] = resOld[4];
  if (isnan(S.lastResiduals[lvl]) || S.lastResiduals[lvl] > 1.5 * S.minRes[lvl]) { S.done = 1; S.good = 0; S.status = 2; return; }
  if (S.rep > 1 && !S.haveRepeated) { S.haveRepeated = 1; ct_begin_level(T, S); return; }  // lvl++ ; continue  => the same level again
  S.lvl = lvl - 1;
  if (S.lvl < 0) {  // L747-769
    S.done = 1;
    bool good = true;
    if ((T.affModeA != 0 && (fabsf((float)S.a) > 1.2f)) || (T.affModeB != 0 && (fabsf((float)S.b) > 200.f))) good = false;
    float eF = T.ref_exposure, eT = T.new_exposure;
    if (eF == 0 || eT == 0) eT = eF = 1;
    const double ra = exp(S.a - T.ref_a) * eT / eF, rb = S.b - ra * T.ref_b;
    if ((T.affModeA == 0 && (fabsf(logf((float)ra)) > 1.5f)) || (T.affModeB == 0 && (fabsf((float)rb) > 200.f))) good = false;
    if (T.affModeA < 0) S.a = 0;
    if (T.affModeB < 0) S.b = 0;
    S.good = good ? 1 : 0;
    return;
  }
  ct_begin_level(T, S);
}
// thread 0: the evaluation that just finished sits in S.res/H/bb[cur^1] (ct_finish_parallel); decide what to evaluate next
__device__ void ct_advance(const CTTrack& T, CTLM& S) {
  const int maxIterations[5] = {10, 20, 50, 50, 50};
  const int nw = S.cur ^ 1;
  const double* res = S.res[nw];
  if (S.phase == CT_PH_INIT) {  // L566-578: first evaluation of a level, cutoff doubling while too many residuals saturate
    S.cur = nw;                 // this evaluation becomes the current linearisation (resOld, H, b)
    if (res[5] > 0.6 && (S.rep < 50 || res[5] > 0.99)) { S.rep *= 2; S.need_request = 1; return; }
    S.lambda = 0.01f;
    S.iteration = 0;
    if (S.iteration >= maxIterations[S.lvl]) { ct_end_level(T, S); return; }
    ct_propose_pre(T, S);
    return;
  }
  // CT_PH_LM: accept / reject (L686-716)
  const double* resOld = S.res[S.cur];
  const bool accept = (res[0] / res[1]) < (resOld[0] / resOld[1]);
  if (accept) {
    S.cur = nw;  // calcGSSSE at the accepted pose == the H,b of the evaluation that just finished
    S.a = S.an; S.b = S.bn;
    for (int i = 0; i < 9; i++) S.R[i] = S.Rn[i];
    for (int i = 0; i < 3; i++) S.t[i] = S.tn[i];
    S.lambda *= 0.5f;
  } else {
    S.lambda *= 4;
    if (S.lambda < 0.001f) S.lambda = 0.001f;
  }
  double incNorm = 0;
  for (int i = 0; i < 8; i++) incNorm += S.inc[i] * S.inc[i];
  incNorm = sqrt(incNorm);
  S.iteration++;
  if (!(incNorm > 1e-3) || S.iteration >= maxIterations[S.lvl]) { ct_end_level(T, S); return; }
  ct_propose_pre(T, S);
}
// one step of the state machine, executed by warp 0 of every CTA
__device__ __forceinline__ void ct_advance_warp(const CTTrack& T, CTLM& S) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) { S.need_request = 0; ct_advance(T, S); }
  __syncwarp();
  if (S.need_solve) {  // warp-uniform (shared memory)
    ct_build_system_warp(T, S);
    __syncwarp();
    ct_factor_warp(S);
    __syncwarp();
    if (lane == 0) ct_propose_post(T, S);
    __syncwarp();
  }
  if (S.need_request) ct_pose_request_warp(T, S, S.need_request == 2);
}

// ---------------------------------------------------------------------------------------------------------------------
// ct_track_cluster_kernel — the trackNewestCoarse state machine above on ONE THREAD-BLOCK CLUSTER (sm_90+ hardware feature):
//   * the CTAs of the cluster exchange their fp64 partials through DISTRIBUTED SHARED MEMORY (st.shared::cluster into every peer's
//     slot) and meet at the hardware cluster barrier (barrier.cluster.arrive/wait): no global-memory partials, no atomics, no spinning
//     on an L2 counter — a few hundred ns per evaluation (~4 us through a chip-wide software grid barrier);
//   * pyramid levels whose float4 plane fits in shared memory (80x60 at 640x480: 76.8 KB; 64x64 at 512^2; 40x30) are staged ONCE per
//     level by TMA (cp.async.bulk.tensor.2d, multicast to every CTA of the cluster, completion on an mbarrier) and every Levenberg-
//     Marquardt evaluation of that level gathers its 4 taps per point from shared memory instead of L2;
//   * the block reduction of the 53 sums is ct_block_sum's transposing butterfly, as in ct_res_gs_kernel.
// Every CTA folds the cluster's partials in rank order and advances the same scalar state machine: identical decisions everywhere.
// A sequential LM chain is latency-bound: fewer, closer SMs with a hardware barrier beat a chip-wide software barrier (DESIGN.md §5).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int CTC_THREADS = 512;
constexpr int CTC_SLOTS = 2;                // reference points per thread kept in registers (2 x 16 x 512 = 16384 points per level)
constexpr int CTC_MAXC = 16;                 // CTAs per cluster (8 portable, 16 with the non-portable opt-in)
constexpr int CTC_PLANE_BYTES = 80 * 1024;   // largest level plane staged in shared memory
struct alignas(64) CTMaps { CUtensorMap lvl[CT_L]; };   // level planes as 2-D tensors of 16-byte texels (encoded as pairs of fp64)

struct CTLoop {   // the variables of trackNewCoarse's try loop (FullSystem.cpp:L406-413), one copy per CTA, advanced by thread 0 after each try
  double achieved[5];              // achievedRes: the next try's minResForAbort
  double R[9], t[3], a, b, flowVecs[3];   // the winner's lastF_2_fh, aff_g2l, lastFlowIndicators
  double pevals;                   // point evaluations of the tries so far
  int haveOneGood, winner, trackingGood, tries, stop;
};

struct alignas(128) CTCSmem {
  unsigned char plane[CTC_PLANE_BYTES];      // TMA destination: the staged level, row-major float4
  double xch[2][CTC_MAXC][CT_NRED + 3];      // [parity][source CTA][sum]: written by every CTA of the cluster through DSMEM
  float red[CTC_THREADS / 32][64];           // per-warp sums (transposed butterfly output)
  double s_sum[CT_NRED + 3];
  CTLM S;
  CTLoop loop;                               // ct_track_tries_kernel: trackNewCoarse's loop variables
  unsigned long long mbar;                   // TMA completion barrier
};

__device__ __forceinline__ unsigned ctc_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned ctc_size() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void ctc_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned ctc_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned ctc_cluster_id() { unsigned r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }

// ---------------------------------------------------------------------------------------------------------------------
// ct_track_tries_kernel — the try loop of FullSystem::trackNewCoarse (FullSystem.cpp:L412-506, visual-only) in one launch on one cluster:
// the tries run one after the other through the trackNewestCoarse body below, each with the loop's achievedRes as its minResForAbort, and
// after each try thread 0 of every CTA applies the loop's bookkeeping to its own copy of the loop variables (CTLoop).  Every CTA holds the
// same LM state after a try, so every CTA takes the same decisions, the break included, without any exchange.
// ---------------------------------------------------------------------------------------------------------------------
typedef double CTPose[12];         // one try of lastF_2_fh_tries: R row-major, t
struct CTTryLoop {                 // the loop's inputs besides the try table
  int n;
  float reTrackThreshold;
  double lastCoarseRMSE0;
  dmv_ct_tries_result* out;        // pinned host
};
struct CTTries {                   // ct_track_tries_kernel's __grid_constant__ parameter block
  CTTrack T;                       // the handle's descriptors; T.a0, T.b0 = aff_last_2_l
  CTMaps maps;
  CTPose pose[DMV_CT_MAX_TRIES];
  CTTryLoop L;
};
static_assert(sizeof(CTTries) <= 32764, "CTTries exceeds the 32,764-byte kernel-parameter limit (CUDA >= 12.1, sm_70+)");

// the loop's bookkeeping after try k (L427-488) from the tracker's state S after it; sets the break (L486)
__device__ void ct_tries_step(const CTTryLoop& Q, CTLoop& W, const CTLM& S, int k) {
  const bool good = S.status == 0 && S.good;   // trackingIsGood: false after an abort
  W.tries = k + 1;
  W.pevals += S.pevals;
  if (good) W.trackingGood = 1;
  const double* lastRes = S.lastResiduals;   // reset to NaN at the start of the try (CoarseTracker.cpp:L551), set up to its last level end
  if (good && isfinite((float)lastRes[0]) && !(lastRes[0] >= W.achieved[0])) {   // a new winner (L467-473)
    for (int i = 0; i < 3; i++) W.flowVecs[i] = S.flow[i];
    for (int i = 0; i < 9; i++) W.R[i] = S.R[i];
    for (int i = 0; i < 3; i++) W.t[i] = S.t[i];
    W.a = S.a; W.b = S.b;
    W.haveOneGood = 1; W.winner = k;
  }
  if (W.haveOneGood)   // take over achieved res (L476-483)
    for (int i = 0; i < 5; i++)
      if (!isfinite((float)W.achieved[i]) || W.achieved[i] > lastRes[i]) W.achieved[i] = lastRes[i];
  W.stop = W.haveOneGood && W.achieved[0] < Q.lastCoarseRMSE0 * (double)Q.reTrackThreshold;
}

// one frame tracked by the calling cluster (TRIES: the tries pose[0 .. Q->n) one after the other).  T and maps are __grid_constant__
// kernel parameters (the tensor map must stay in parameter space: its address is the operand of the TMA copy); the try table may lie in
// parameter space (ct_track_tries_kernel) or in the handle's pinned host memory (ct_track_tries_many_kernel).
template <bool TRIES>
__device__ __forceinline__ void ct_track_cluster(const CTTrack& T, const CTMaps& maps, const CTPose* pose, const CTTryLoop* Q) {
  extern __shared__ __align__(128) unsigned char ctc_raw[];
  CTCSmem& M = *reinterpret_cast<CTCSmem*>(ctc_raw);
  CTLM& S = M.S;
  const int tid = threadIdx.x;
  const unsigned rank = ctc_rank(), NC = ctc_size();
  int par = 0, staged_lvl = -1, cached_lvl = -1;
  unsigned mphase = 0;
  float4 pts[CTC_SLOTS];
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(ctc_smem_u32(&M.mbar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if constexpr (TRIES) {   // Vec5::Constant(NAN), haveOneGood = false, trackingGoodRet = false (L406-413)
      CTLoop& W = M.loop;
      for (int i = 0; i < 5; i++) W.achieved[i] = __longlong_as_double(0x7ff8000000000000ll);
      W.pevals = 0; W.haveOneGood = 0; W.winner = -1; W.trackingGood = 0; W.tries = 0; W.stop = 0;
    }
  }
  // the staged plane, its mbarrier phase and the cached reference points stay valid from one try to the next: the frame is the same
  for (int kt = 0;; kt++) {   // one track per pass; the plain kernels make one pass
    if (tid == 0) {
      const double* R0 = TRIES ? pose[kt] : T.R0;
      const double* t0 = TRIES ? pose[kt] + 9 : T.t0;
      for (int i = 0; i < 9; i++) S.R[i] = R0[i];
      for (int i = 0; i < 3; i++) S.t[i] = t0[i];
      S.a = T.a0; S.b = T.b0;
      for (int i = 0; i < 5; i++) S.lastResiduals[i] = __longlong_as_double(0x7ff8000000000000ll);  // NAN
      for (int i = 0; i < 3; i++) S.flow[i] = 1000;
      for (int i = 0; i < 5; i++) S.minRes[i] = TRIES ? M.loop.achieved[i] : T.minRes[i];
      S.haveRepeated = 0; S.iterations = 0; S.evaluations = 0; S.done = 0; S.good = 0; S.status = 0; S.cur = 0; S.need_solve = 0; S.pevals = 0;
      S.lvl = T.coarsest;
      ct_begin_level(T, S);
    }
    __syncthreads();
    if (tid < 32) ct_pose_request_warp(T, S, false);
    __syncthreads();
    if (kt == 0) ctc_cluster_sync();  // every CTA's mbarrier exists before the first multicast copy can signal it
    while (!S.done) {
      const int l = S.lvl;
      // ---- level change: stage the plane with TMA if the host encoded its map (one multicast copy issued by CTA 0 lands in every CTA's
      // shared memory); the host decides, so the kernel never issues a copy on a zeroed descriptor
      const bool fits = T.staged[l] != 0;
      if (fits && staged_lvl != l) {
        const unsigned bytes = (unsigned)(T.w[l] * T.h[l] * sizeof(float4));
        if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ctc_smem_u32(&M.mbar)), "r"(bytes) : "memory");
        ctc_cluster_sync();  // all barriers armed (and nobody still reads the previous level's plane)
        if (rank == 0 && tid == 0) {
          const unsigned short mask = (unsigned short)((1u << NC) - 1u);
          asm volatile(
              "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
                  ctc_smem_u32(M.plane)),
              "l"(&maps.lvl[l]), "r"(ctc_smem_u32(&M.mbar)), "r"(0), "r"(0), "h"(mask)
              : "memory");
        }
        {  // wait for the bytes (try_wait suspends the thread between probes)
          const unsigned mb = ctc_smem_u32(&M.mbar);
          unsigned done = 0;
          while (!done)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(mb), "r"(mphase) : "memory");
        }
        mphase ^= 1u;
        staged_lvl = l;
      }
      // ---- one evaluation: calcRes + calcGSSSE at the requested pose
      CTParams P;
#pragma unroll
      for (int i = 0; i < 9; i++) { P.RKi[i] = S.RKi[i]; P.Ki[i] = T.Ki[l][i]; }
#pragma unroll
      for (int i = 0; i < 3; i++) P.t[i] = S.tf[i];
      P.fx = T.fx[l]; P.fy = T.fy[l]; P.cx = T.cx[l]; P.cy = T.cy[l];
      P.affa = S.affLL[0]; P.affb = S.affLL[1]; P.a_gs = S.affLL[0]; P.b0 = (float)T.ref_b;
      P.cutoff = S.cutoff; P.huber = T.huber; P.maxEnergy = 2 * T.huber * S.cutoff - T.huber * T.huber;
      P.w = T.w[l]; P.h = T.h[l]; P.n = T.n[l]; P.lvl = l; P.want_gs = 1;
      float v[64];
#pragma unroll
      for (int k = 0; k < 64; k++) v[k] = 0.f;
      const int stride = (int)NC * CTC_THREADS, first = (int)rank * CTC_THREADS + tid;
      if (cached_lvl != l) {  // the level's reference points of this thread stay in registers for all evaluations of the level
#pragma unroll
        for (int k = 0; k < CTC_SLOTS; k++) {
          const int i = first + k * stride;
          if (i < P.n) { pts[k] = make_float4(__ldg(T.u[l] + i), __ldg(T.v[l] + i), __ldg(T.id[l] + i), __ldg(T.col[l] + i)); }
        }
        cached_lvl = l;
      }
#pragma unroll
      for (int k = 0; k < CTC_SLOTS; k++) {
        const int i = first + k * stride;
        if (i < P.n) {
          if (fits) ct_eval_accumulate<true>(P, i, pts[k].x, pts[k].y, pts[k].z, pts[k].w, T.img[l], reinterpret_cast<const float4*>(M.plane), v);
          else ct_eval_accumulate<false>(P, i, pts[k].x, pts[k].y, pts[k].z, pts[k].w, T.img[l], nullptr, v);
        }
      }
      for (int i = first + CTC_SLOTS * stride; i < P.n; i += stride) {  // more points than register slots: stream the rest
        if (fits) ct_eval_accumulate<true>(P, i, __ldg(T.u[l] + i), __ldg(T.v[l] + i), __ldg(T.id[l] + i), __ldg(T.col[l] + i), T.img[l], reinterpret_cast<const float4*>(M.plane), v);
        else ct_eval_accumulate<false>(P, i, __ldg(T.u[l] + i), __ldg(T.v[l] + i), __ldg(T.id[l] + i), __ldg(T.col[l] + i), T.img[l], nullptr, v);
      }
      // ---- CTA: fp64 sum over the warps, pushed into EVERY CTA's exchange slot through distributed shared memory
      const double bs = ct_block_sum<CTC_THREADS / 32>(v, M.red);
      if (tid < CT_NRED) {
        const unsigned local = ctc_smem_u32(&M.xch[par][rank][tid]);
        for (unsigned c = 0; c < NC; c++) {
          unsigned remote;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(c));
          asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(remote), "d"(bs) : "memory");
        }
      }
      ctc_cluster_sync();  // release / acquire at cluster scope: every CTA's partials are visible in every CTA's shared memory
      if (tid < CT_NRED) {
        double sm = 0.0;
        for (unsigned c = 0; c < NC; c++) sm += M.xch[par][c][tid];  // rank order: bit-identical in every CTA
        M.s_sum[tid] = sm;
      }
      par ^= 1;
      __syncthreads();
      ct_finish_parallel(M.s_sum, S.res[S.cur ^ 1], S.H[S.cur ^ 1], S.bb[S.cur ^ 1], tid);
      __syncthreads();
      if (tid < 32) ct_advance_warp(T, S);
      __syncthreads();
    }
    if constexpr (!TRIES) {
      break;
    } else {
      if (tid == 0) ct_tries_step(*Q, M.loop, S, kt);
      __syncthreads();
      if (M.loop.stop || kt + 1 == Q->n) break;   // the same in every CTA of the cluster
    }
  }
  ctc_cluster_sync();  // nobody leaves while a peer may still write into its shared memory
  if (rank == 0 && tid == 0) {
    if constexpr (TRIES) {   // L491-497 when no try was good: try 0's pose, aff_last_2_l, zero flow
      const CTLoop& W = M.loop;
      dmv_ct_tries_result* o = Q->out;
      const bool one = W.haveOneGood != 0;
      for (int i = 0; i < 9; i++) o->R[i] = one ? W.R[i] : pose[0][i];
      for (int i = 0; i < 3; i++) o->t[i] = one ? W.t[i] : pose[0][9 + i];
      o->a = one ? W.a : T.a0; o->b = one ? W.b : T.b0;
      for (int i = 0; i < 5; i++) { o->achievedRes[i] = W.achieved[i]; o->lastResiduals[i] = S.lastResiduals[i]; }
      for (int i = 0; i < 3; i++) { o->flowVecs[i] = one ? W.flowVecs[i] : 0.0; o->flowIndicators[i] = S.flow[i]; }
      o->trackingGood = W.trackingGood; o->haveOneGood = W.haveOneGood; o->winner = one ? W.winner : -1;
      o->tries = W.tries; o->tries_started = W.tries;
      T.out->pevals = W.pevals;
    } else {
      CTTrackOut* o = T.out;
      const bool ok = (S.status == 0);   // an aborted track returns the input pose, like the reference's early return
      for (int i = 0; i < 9; i++) o->R[i] = ok ? S.R[i] : T.R0[i];
      for (int i = 0; i < 3; i++) o->t[i] = ok ? S.t[i] : T.t0[i];
      o->a = ok ? S.a : T.a0; o->b = ok ? S.b : T.b0;
      for (int i = 0; i < 5; i++) o->lastResiduals[i] = S.lastResiduals[i];
      for (int i = 0; i < 3; i++) o->flow[i] = S.flow[i];
      o->good = S.good; o->iterations = S.iterations; o->evaluations = S.evaluations; o->status = S.status; o->pevals = S.pevals;
    }
  }
}

__global__ void __launch_bounds__(CTC_THREADS, 1) ct_track_cluster_kernel(const __grid_constant__ CTTrack T, const __grid_constant__ CTMaps maps) {
  ct_track_cluster<false>(T, maps, nullptr, nullptr);
}

// dmv_ct_track_many: cluster i tracks member i, independently of every other cluster (no inter-cluster synchronisation, so clusters beyond
// the co-resident ones simply start when earlier ones retire).  The descriptors of all members travel in the parameter block.
struct CTTrackMany {
  CTTrack T[DMV_CT_TRACK_MANY_MAX];
  CTMaps maps[DMV_CT_TRACK_MANY_MAX];
};
static_assert(sizeof(CTTrackMany) <= 32764, "CTTrackMany exceeds the 32,764-byte kernel-parameter limit (CUDA >= 12.1, sm_70+)");

__global__ void __launch_bounds__(CTC_THREADS, 1) ct_track_many_kernel(const __grid_constant__ CTTrackMany B) {
  const unsigned i = ctc_cluster_id();
  ct_track_cluster<false>(B.T[i], B.maps[i], nullptr, nullptr);
}

__global__ void __launch_bounds__(CTC_THREADS, 1) ct_track_tries_kernel(const __grid_constant__ CTTries Q) {
  ct_track_cluster<true>(Q.T, Q.maps, Q.pose, &Q.L);
}

// dmv_ct_track_tries_many: cluster i runs member i's try loop, independently of every other cluster, as ct_track_many_kernel tracks.  The
// 16 try tables (48 KB) do not fit in the parameter block beside the descriptors; each lies in its handle's pinned memory (h_pose), and
// thread 0 of each CTA reads a try's 12 doubles from there when the try starts.
struct CTTriesMany {
  CTTrack T[DMV_CT_TRACK_MANY_MAX];
  CTMaps maps[DMV_CT_TRACK_MANY_MAX];
  CTTryLoop L[DMV_CT_TRACK_MANY_MAX];
  const CTPose* pose[DMV_CT_TRACK_MANY_MAX];   // pinned host, in[i].n tries
};
static_assert(sizeof(CTTriesMany) <= 32764, "CTTriesMany exceeds the 32,764-byte kernel-parameter limit (CUDA >= 12.1, sm_70+)");

__global__ void __launch_bounds__(CTC_THREADS, 1) ct_track_tries_many_kernel(const __grid_constant__ CTTriesMany B) {
  const unsigned i = ctc_cluster_id();
  ct_track_cluster<true>(B.T[i], B.maps[i], B.pose[i], &B.L[i]);
}

}  // namespace dmv

using namespace dmv;

void dmv::CTPartDelete::operator()(CTMaps* p) const { delete p; }

int dmv::ct_build_pyramid(dmv_ct* c, int first_level) {
  for (int l = first_level; l < c->cfg.levels; l++) {
    if (l > 0) {
      launch_pyr_down(c->d_img[l - 1], c->d_gray[l], c->w[l], c->h[l], c->w[l - 1], c->stream);
      c->launches++;
    }
    launch_make_dI(c->d_gray[l], c->d_img[l], c->w[l], c->h[l], c->stream);
    c->launches++;
  }
  CK(cudaGetLastError());
  return DMV_OK;
}

extern "C" {

static int ct_allocate(dmv_ct* c, const dmv_ct_config* cfg);

int dmv_ct_create(const dmv_ct_config* cfg, dmv_ct** out) {
  if (!cfg || !out) return set_error(DMV_ERR_INVALID, "null argument");
  if (cfg->levels < 1 || cfg->levels > DMV_MAX_PYR_LEVELS || cfg->w < 16 || cfg->h < 16 || cfg->max_points < 1)
    return set_error(DMV_ERR_INVALID, "bad config");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return set_error(DMV_ERR_NO_DEVICE, "no CUDA device: dmvio_b200 has no CPU path");
  }
  if (cfg->device < 0 || cfg->device >= ndev) return set_error(DMV_ERR_INVALID, "device out of range");
  CK(cudaSetDevice(cfg->device));
  dmv_ct* c = new dmv_ct();
  const int rc = ct_allocate(c, cfg);
  if (rc != DMV_OK) {  // allocation failed half-way: the members release what exists, the failing call's error message is kept
    delete c;
    return rc;
  }
  *out = c;
  return DMV_OK;
}

static int ct_allocate(dmv_ct* c, const dmv_ct_config* cfg) {
  c->cfg = *cfg;
  c->device = cfg->device;
  CK(cudaStreamCreateWithFlags(c->stream.put(), cudaStreamNonBlocking));
  CK(cudaEventCreate(c->ev[0].put()));
  CK(cudaEventCreate(c->ev[1].put()));
  CK(cudaEventCreateWithFlags(c->ev_order.put(), cudaEventDisableTiming));
  for (int l = 0; l < cfg->levels; l++) {
    c->w[l] = cfg->w >> l; c->h[l] = cfg->h >> l; c->haveK[l] = false; c->n[l] = 0;
    const size_t npx = (size_t)c->w[l] * c->h[l];
    CK(c->d_img[l].alloc(npx));
    CK(c->d_gray[l].alloc(npx));
    CK(c->d_u[l].alloc(cfg->max_points));
    CK(c->d_v[l].alloc(cfg->max_points));
    CK(c->d_id[l].alloc(cfg->max_points));
    CK(c->d_col[l].alloc(cfg->max_points));
  }
  const size_t npx0 = (size_t)cfg->w * cfg->h;
  CK(c->d_stage.alloc(npx0 * 3));
  const int maxBlocks = (cfg->max_points + CT_THREADS - 1) / CT_THREADS;
  CK(c->d_partial.alloc((size_t)CT_NRED * maxBlocks));  // ct_res_gs_kernel's per-block partials
  CK(c->d_ticket.alloc(1));
  CK(cudaMemset(c->d_ticket, 0, sizeof(unsigned int)));
  CK(c->h_out.alloc(64));
  CK(c->h_scratch.alloc(std::max(npx0 * 3, (size_t)cfg->max_points * 4)));
  return DMV_OK;
}

int dmv_ct_destroy(dmv_ct* c) {
  if (!c) return DMV_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  delete c;
  return DMV_OK;
}

int dmv_ct_set_K(dmv_ct* c, int l, float fx, float fy, float cx, float cy) {
  if (!c || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad level");
  c->fx[l] = fx; c->fy[l] = fy; c->cx[l] = cx; c->cy[l] = cy; c->haveK[l] = true;
  return DMV_OK;
}
int dmv_ct_set_huber(dmv_ct* c, float huberTH) {
  if (!c) return set_error(DMV_ERR_INVALID, "null handle");
  c->huber = huberTH;
  return DMV_OK;
}

int dmv_ct_set_ref(dmv_ct* c, int l, int n, const float* u, const float* v, const float* id, const float* col) {
  if (!c || l < 0 || l >= c->cfg.levels || n < 0 || n > c->cfg.max_points) return set_error(DMV_ERR_INVALID, "bad level / count");
  if (n > 0 && (!u || !v || !id || !col)) return set_error(DMV_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  c->n[l] = n;
  if (n > 0) {
    CK(ct_wait_staging(c));
    float* s = c->h_scratch;
    std::memcpy(s, u, 4 * (size_t)n); std::memcpy(s + n, v, 4 * (size_t)n); std::memcpy(s + 2 * (size_t)n, id, 4 * (size_t)n);
    std::memcpy(s + 3 * (size_t)n, col, 4 * (size_t)n);
    CK(cudaMemcpyAsync(c->d_u[l], s, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_v[l], s + n, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_id[l], s + 2 * (size_t)n, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_col[l], s + 3 * (size_t)n, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  return DMV_OK;
}

int dmv_ct_upload_new(dmv_ct* c, int l, const float* dIp) {
  if (!c || !dIp || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad level / pointer");
  CK(cudaSetDevice(c->device));
  const size_t npx = (size_t)c->w[l] * c->h[l];
  CK(ct_wait_staging(c));
  std::memcpy(c->h_scratch, dIp, npx * 3 * sizeof(float));
  CK(cudaMemcpyAsync(c->d_stage, c->h_scratch, npx * 3 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  launch_repack(c->d_stage, c->d_img[l], (int)npx, c->stream);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return DMV_OK;
}

int dmv_ct_upload_new_image(dmv_ct* c, const float* image) {
  if (!c || !image) return set_error(DMV_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  const size_t npx = (size_t)c->w[0] * c->h[0];
  CK(ct_wait_staging(c));
  std::memcpy(c->h_scratch, image, npx * sizeof(float));
  CK(cudaMemcpyAsync(c->d_gray[0], c->h_scratch, npx * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  const int rc = ct_build_pyramid(c, 0);
  if (rc != DMV_OK) return rc;
  // no synchronisation: every consumer (dmv_ct_calc_res_gs / dmv_ct_track) runs on the same stream and synchronises itself; the image
  // was copied into the handle's pinned staging buffer above, so the caller's buffer is already free
  c->staging_busy = true;
  return DMV_OK;
}

int dmv_ct_download_frame(dmv_ct* c, int l, float* dIp) {
  if (!c || !dIp || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad level / pointer");
  CK(cudaSetDevice(c->device));
  const size_t npx = (size_t)c->w[l] * c->h[l];
  CK(ct_wait_staging(c));
  // float4 (I, dx, dy, 0) -> 3 floats per pixel into the pinned staging buffer (it holds w*h*3 floats of level 0)
  CK(cudaMemcpy2DAsync(c->h_scratch, 3 * sizeof(float), c->d_img[l], sizeof(float4), 3 * sizeof(float), npx, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  std::memcpy(dIp, c->h_scratch, npx * 3 * sizeof(float));
  return DMV_OK;
}

int dmv_ct_calc_res_gs(dmv_ct* c, int l, const float RKi[9], const float t[3], const float affLL[2], float b0, float cutoffTH, int want_gs,
                       double res6[6], double H[64], double b[8], int* n_warped) {
  if (!c || !RKi || !t || !affLL || !res6 || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad argument");
  if (!c->haveK[l]) return set_error(DMV_ERR_STATE, "dmv_ct_set_K(level) first");
  if (want_gs && (!H || !b)) return set_error(DMV_ERR_INVALID, "H/b required with want_gs");
  CK(cudaSetDevice(c->device));
  CTParams P;
  std::memcpy(P.RKi, RKi, sizeof(P.RKi));
  std::memcpy(P.t, t, sizeof(P.t));
  // Ki[lvl] = K^-1 (CoarseTracker.cpp:L126-133)
  {
    const float Kl[9] = {c->fx[l], 0.f, c->cx[l], 0.f, c->fy[l], c->cy[l], 0.f, 0.f, 1.f};
    inv3_cofactor(Kl, P.Ki);
  }
  P.fx = c->fx[l]; P.fy = c->fy[l]; P.cx = c->cx[l]; P.cy = c->cy[l];
  P.affa = affLL[0]; P.affb = affLL[1]; P.a_gs = affLL[0]; P.b0 = b0;
  P.cutoff = cutoffTH; P.huber = c->huber;
  P.maxEnergy = 2 * c->huber * cutoffTH - c->huber * c->huber;
  P.w = c->w[l]; P.h = c->h[l]; P.n = c->n[l]; P.lvl = l; P.want_gs = want_gs;
  const int nb = std::max(1, (c->n[l] + CT_THREADS - 1) / CT_THREADS);
  if (c->timing) CK(cudaEventRecord(c->ev[0], c->stream));
  // the last block writes the 53 reduced doubles straight into the pinned host buffer (zero-copy): no D2H copy node per evaluation
  ct_res_gs_kernel<<<nb, CT_THREADS, 0, c->stream>>>(P, c->d_u[l], c->d_v[l], c->d_id[l], c->d_col[l], c->d_img[l], c->d_partial, c->d_ticket,
                                                      c->h_out);
  c->launches++;
  if (c->timing) CK(cudaEventRecord(c->ev[1], c->stream));
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  c->staging_busy = false;
  if (c->timing) cudaEventElapsedTime(&c->last_ms[0], c->ev[0], c->ev[1]);
  const double* o = c->h_out;
  const double E = o[45], nE = o[46], nSat = o[47], nW = o[48];
  res6[0] = E;
  res6[1] = nE;
  res6[2] = (double)((float)o[49] / ((float)o[51] + 0.1f));
  res6[3] = 0;
  res6[4] = (double)((float)o[50] / ((float)o[51] + 0.1f));
  res6[5] = (double)((float)nSat / (float)nE);
  const int npad = ((int)nW + 3) & ~3;
  if (n_warped) *n_warped = npad;
  if (want_gs) {
    // acc.H (9x9) -> H_out = H[0:8,0:8] * (1/n), b_out = H[0:8,8] * (1/n), then SCALE_* (CoarseTracker.cpp:L341-355)
    double M[9][9];
    int e = 0;
    for (int r = 0; r < 9; r++)
      for (int cc = r; cc < 9; cc++) { M[r][cc] = M[cc][r] = o[e]; e++; }
    const double inv = (double)(1.0f / (float)npad);
    const double sc[8] = {1, 1, 1, 1, 1, 1, 10.0, 1000.0};  // SCALE_XI_ROT/TRANS = 1, SCALE_A, SCALE_B
    for (int r = 0; r < 8; r++) {
      for (int cc = 0; cc < 8; cc++) H[r * 8 + cc] = M[r][cc] * inv * sc[r] * sc[cc];
      b[r] = M[r][8] * inv * sc[r];
    }
  }
  return DMV_OK;
}

// TMA descriptors of the level planes: a w x h plane of float4 texels = a 2-D tensor of (2w) x h fp64 elements (the widest element type a
// tensor map knows; 16-byte texels = pairs), one box = the whole plane.  c->staged[l] records the levels encoded here; the cluster kernel
// stages exactly those (a plane that fits CTC_PLANE_BYTES but exceeds the 256-element box limit is gathered from L2).
static int ct_make_tensor_maps(dmv_ct* c) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                               CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn || qres != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return set_error(DMV_ERR_CUDA, "cuTensorMapEncodeTiled is not available");
  }
  if (!c->maps) c->maps.reset(new CTMaps());
  std::memset(c->maps.get(), 0, sizeof(CTMaps));
  for (int l = 0; l < DMV_MAX_PYR_LEVELS; l++) c->staged[l] = 0;
  for (int l = 0; l < c->cfg.levels; l++) {
    const size_t bytes = (size_t)c->w[l] * c->h[l] * sizeof(float4);
    if (bytes > (size_t)CTC_PLANE_BYTES || 2 * c->w[l] > 256 || c->h[l] > 256) continue;   // never staged (box limits: 256 elements per dimension)
    const cuuint64_t gdim[2] = {(cuuint64_t)(2 * c->w[l]), (cuuint64_t)c->h[l]};
    const cuuint64_t gstride[1] = {(cuuint64_t)c->w[l] * sizeof(float4)};
    const cuuint32_t box[2] = {(cuuint32_t)(2 * c->w[l]), (cuuint32_t)c->h[l]};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = reinterpret_cast<EncodeFn>(fn)(&c->maps->lvl[l], CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, c->d_img[l], gdim, gstride, box, estr,
                                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(DMV_ERR_CUDA, "cuTensorMapEncodeTiled failed for level %d (CUresult %d)", l, (int)r);
    c->staged[l] = 1;
  }
  return DMV_OK;
}

// a grid of `clusters` thread-block clusters of nc CTAs of the track kernels on stream s
struct CTClusterLaunch {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  CTClusterLaunch(int nc, int clusters, cudaStream_t s) {
    cfg.gridDim = dim3(nc * clusters); cfg.blockDim = dim3(CTC_THREADS); cfg.dynamicSmemBytes = sizeof(CTCSmem); cfg.stream = s;
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = nc; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
  }
};

static CTTrackOut* ct_track_out(const dmv_ct* c) { return reinterpret_cast<CTTrackOut*>(c->h_out.get()); }

// dmv_ct_track's argument checks and the launch parameters of one handle, all but staged[] (decided by the probe); no CUDA call
static int ct_track_params(dmv_ct* c, const dmv_ct_track_args* in, CTTrack& T) {
  if (in->coarsestLvl < 0 || in->coarsestLvl >= c->cfg.levels || in->coarsestLvl >= 5) return set_error(DMV_ERR_INVALID, "coarsestLvl out of range");
  std::memset(&T, 0, sizeof(T));
  T.levels = c->cfg.levels; T.coarsest = in->coarsestLvl;
  for (int l = 0; l < c->cfg.levels; l++) {
    if (!c->haveK[l]) return set_error(DMV_ERR_STATE, "dmv_ct_set_K(level) first");
    T.n[l] = c->n[l]; T.w[l] = c->w[l]; T.h[l] = c->h[l];
    T.fx[l] = c->fx[l]; T.fy[l] = c->fy[l]; T.cx[l] = c->cx[l]; T.cy[l] = c->cy[l];
    const float Kl[9] = {c->fx[l], 0.f, c->cx[l], 0.f, c->fy[l], c->cy[l], 0.f, 0.f, 1.f};
    inv3_cofactor(Kl, T.Ki[l]);
    T.u[l] = c->d_u[l]; T.v[l] = c->d_v[l]; T.id[l] = c->d_id[l]; T.col[l] = c->d_col[l]; T.img[l] = c->d_img[l];
  }
  for (int i = 0; i < 9; i++) T.R0[i] = in->R[i];
  for (int i = 0; i < 3; i++) T.t0[i] = in->t[i];
  T.a0 = in->a; T.b0 = in->b; T.ref_a = in->ref_a; T.ref_b = in->ref_b;
  T.ref_exposure = in->ref_exposure; T.new_exposure = in->new_exposure;
  T.huber = c->huber; T.cutoffTH = in->coarseCutoffTH; T.affModeA = in->affineOptModeA; T.affModeB = in->affineOptModeB;
  for (int i = 0; i < 5; i++) T.minRes[i] = in->minResForAbort[i];
  T.out = ct_track_out(c);
  return DMV_OK;
}

// the handle's cluster size, probed on its first track (on the handle's device): the largest cluster the device schedules for
// ct_track_cluster_kernel (16 needs the non-portable opt-in).  ct_track_many_kernel, ct_track_tries_kernel and ct_track_tries_many_kernel
// have the same block, shared memory and launch bounds, so the probed size holds for them too; the probe opts all four kernels in.
static int ct_probe_cluster(dmv_ct* c) {
  if (c->cluster_size == 0) {
    c->cluster_size = -1;
    // test hook: DMV_CT_CLUSTER=16|8|4 probes only that cluster size
    const char* env_nc = getenv("DMV_CT_CLUSTER");
    const int want_nc = env_nc ? atoi(env_nc) : 0;
    if (env_nc && want_nc != 16 && want_nc != 8 && want_nc != 4) {
      c->cluster_size = 0;
      return set_error(DMV_ERR_INVALID, "DMV_CT_CLUSTER=%s: expected 16, 8 or 4", env_nc);
    }
    if (ct_make_tensor_maps(c) == DMV_OK) {
      const void* const kernels[] = {(const void*)ct_track_cluster_kernel, (const void*)ct_track_many_kernel, (const void*)ct_track_tries_kernel,
                                     (const void*)ct_track_tries_many_kernel};
      for (const void* k : kernels) {
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CTCSmem)));
        cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);   // without it the probe finds at most 8
      }
      cudaGetLastError();
      for (int nc : {16, 8, 4}) {
        if (want_nc && nc != want_nc) continue;
        CTClusterLaunch q(nc, 1, c->stream);
        int ncl = 0;
        if (cudaOccupancyMaxActiveClusters(&ncl, ct_track_cluster_kernel, &q.cfg) == cudaSuccess && ncl >= 1) { c->cluster_size = nc; break; }
        cudaGetLastError();
      }
    }
    if (want_nc && c->cluster_size != want_nc) {
      c->cluster_size = 0;
      return set_error(DMV_ERR_INVALID, "DMV_CT_CLUSTER=%d: ct_track_cluster_kernel cannot be scheduled with that cluster size", want_nc);
    }
  }
  if (c->cluster_size < 0)
    return set_error(DMV_ERR_INVALID, "dmv_ct_track needs a thread-block cluster of 16, 8 or 4 CTAs and TMA tensor maps, which this device "
                                      "cannot provide: drive dmv_ct_calc_res_gs from the host LM loop instead");
  return DMV_OK;
}

// the result the kernel wrote into the handle's pinned output block
static void ct_read_result(const dmv_ct* c, dmv_ct_track_result* out) {
  const CTTrackOut* o = ct_track_out(c);
  for (int i = 0; i < 9; i++) out->R[i] = o->R[i];
  for (int i = 0; i < 3; i++) out->t[i] = o->t[i];
  out->a = o->a; out->b = o->b;
  for (int i = 0; i < 5; i++) out->lastResiduals[i] = o->lastResiduals[i];
  for (int i = 0; i < 3; i++) out->flowIndicators[i] = o->flow[i];
  out->trackingGood = (int)o->good; out->iterations = (int)o->iterations; out->evaluations = (int)o->evaluations; out->status = (int)o->status;
}

// the last checks of a track over hs[0..n), after every member's own: each member probed on hs[0]'s device, which this makes current
// (`many`: a member's error names it), and one cluster size among them.  Then each member's staged levels and tensor maps into its launch
// parameters T[i], maps[i].
static int ct_cluster_ready(dmv_ct* const* hs, int n, bool many, CTTrack* T, CTMaps* maps) {
  CK(cudaSetDevice(hs[0]->device));
  for (int i = 0; i < n; i++) {
    const int rc = ct_probe_cluster(hs[i]);
    if (rc != DMV_OK) return many ? ct_member_error(rc, i) : rc;
  }
  for (int i = 1; i < n; i++)
    if (hs[i]->cluster_size != hs[0]->cluster_size)
      return set_error(DMV_ERR_INVALID, "handles[0] tracks with clusters of %d CTAs, handles[%d] with %d: one launch needs one cluster size",
                       hs[0]->cluster_size, i, hs[i]->cluster_size);
  for (int i = 0; i < n; i++) {
    for (int l = 0; l < DMV_MAX_PYR_LEVELS; l++) T[i].staged[l] = hs[i]->staged[l];
    maps[i] = *hs[i]->maps;
  }
  return DMV_OK;
}

// kernel (args: pointers to its parameters) on one cluster per member, on hs[0]'s stream behind every other member's queued work; counted
// on every member and awaited
static int ct_cluster_launch(dmv_ct* const* hs, int n, const void* kernel, void** args) {
  const cudaStream_t s = hs[0]->stream;
  for (int i = 1; i < n; i++) CK(ct_order_behind(hs[i], s));
  CTClusterLaunch q(hs[0]->cluster_size, n, s);
  CK(cudaLaunchKernelExC(&q.cfg, kernel, args));
  for (int i = 0; i < n; i++) hs[i]->launches++;
  CK(cudaStreamSynchronize(s));
  for (int i = 0; i < n; i++) hs[i]->staging_busy = false;   // each member's uploads completed before the kernel started
  return DMV_OK;
}

// CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:L539-770, visual-only branch) for hs[0..n) in one launch, one cluster per handle.
// Every check precedes the launch; `many`: a member's error names it.  One handle launches ct_track_cluster_kernel, the same device function
// with a 1.7 KB instead of a 27 KB parameter block (through ct_track_many_kernel one 640x480, 5-level track took 0.360 ms against 0.336 ms,
// H100 80GB HBM3 at 700 W).
static int ct_track_run(dmv_ct* const* hs, int n, const dmv_ct_track_args* in, dmv_ct_track_result* out, bool many) {
  CTTrack T1;
  CTMaps M1;
  std::unique_ptr<CTTrackMany> B(n > 1 ? new CTTrackMany() : nullptr);
  CTTrack* T = n > 1 ? B->T : &T1;
  for (int i = 0; i < n; i++) {
    const int rc = ct_track_params(hs[i], &in[i], T[i]);
    if (rc != DMV_OK) return many ? ct_member_error(rc, i) : rc;
  }
  int rc = ct_cluster_ready(hs, n, many, T, n > 1 ? B->maps : &M1);
  if (rc != DMV_OK) return rc;
  if (n == 1) {
    void* args[] = {&T1, &M1};
    rc = ct_cluster_launch(hs, 1, (const void*)ct_track_cluster_kernel, args);
  } else {
    void* args[] = {B.get()};
    rc = ct_cluster_launch(hs, n, (const void*)ct_track_many_kernel, args);
  }
  if (rc != DMV_OK) return rc;
  for (int i = 0; i < n; i++) ct_read_result(hs[i], &out[i]);
  return DMV_OK;
}

int dmv_ct_track(dmv_ct* c, const dmv_ct_track_args* in, dmv_ct_track_result* out) {
  if (!c || !in || !out) return set_error(DMV_ERR_INVALID, "null argument");
  return ct_track_run(&c, 1, in, out, false);
}

int dmv_ct_track_many(dmv_ct* const* handles, int n, const dmv_ct_track_args* in, dmv_ct_track_result* out) {
  if (!handles || !in || !out) return set_error(DMV_ERR_INVALID, "null argument");
  const int rc = ct_check_members(handles, n, DMV_CT_TRACK_MANY_MAX);
  return rc != DMV_OK ? rc : ct_track_run(handles, n, in, out, true);
}

// dmv_ct_track_tries's argument checks and the launch parameters of one handle's loop, all but staged[] (decided by the probe) and the
// result pointer (allocated after every check); no CUDA call
static int ct_tries_params(dmv_ct* c, const dmv_ct_tries_args* in, CTTrack& T, CTTryLoop& L) {
  if (in->n < 1 || in->n > DMV_CT_MAX_TRIES) return set_error(DMV_ERR_INVALID, "n = %d: expected 1 to %d tries", in->n, DMV_CT_MAX_TRIES);
  if (!in->R || !in->t) return set_error(DMV_ERR_INVALID, "null R / t");
  dmv_ct_track_args a;   // try 0 with minResForAbort NaN: dmv_ct_track's checks and descriptors
  std::memcpy(a.R, in->R, sizeof(a.R));
  std::memcpy(a.t, in->t, sizeof(a.t));
  a.a = in->a; a.b = in->b; a.ref_a = in->ref_a; a.ref_b = in->ref_b;
  a.ref_exposure = in->ref_exposure; a.new_exposure = in->new_exposure;
  a.coarseCutoffTH = in->coarseCutoffTH; a.affineOptModeA = in->affineOptModeA; a.affineOptModeB = in->affineOptModeB;
  a.coarsestLvl = in->coarsestLvl;
  for (int i = 0; i < 5; i++) a.minResForAbort[i] = NAN;   // unused: each try aborts against the loop's achievedRes
  const int rc = ct_track_params(c, &a, T);
  if (rc != DMV_OK) return rc;
  L.n = in->n;
  L.reTrackThreshold = in->reTrackThreshold;
  L.lastCoarseRMSE0 = in->lastCoarseRMSE0;
  L.out = nullptr;
  return DMV_OK;
}

// lastF_2_fh_tries of in as the kernels' try table
static void ct_fill_tries(const dmv_ct_tries_args* in, CTPose* pose) {
  for (int k = 0; k < in->n; k++) {
    for (int i = 0; i < 9; i++) pose[k][i] = in->R[9 * k + i];
    for (int i = 0; i < 3; i++) pose[k][9 + i] = in->t[3 * k + i];
  }
}

// FullSystem::trackNewCoarse's try loop (FullSystem.cpp:L412-506, visual-only) for hs[0..n) in one launch, one cluster per handle: see
// ct_track_tries_kernel.  Every check precedes the first allocation and the launch; `many`: a member's error names it.  One handle launches
// ct_track_tries_kernel and its 4.8 KB parameter block, as ct_track_run launches ct_track_cluster_kernel.
static int ct_tries_run(dmv_ct* const* hs, int n, const dmv_ct_tries_args* in, dmv_ct_tries_result* out, bool many) {
  std::unique_ptr<CTTries> Q(n == 1 ? new CTTries() : nullptr);
  std::unique_ptr<CTTriesMany> B(n > 1 ? new CTTriesMany() : nullptr);
  CTTrack* T = n > 1 ? B->T : &Q->T;
  CTTryLoop* L = n > 1 ? B->L : &Q->L;
  for (int i = 0; i < n; i++) {
    const int rc = ct_tries_params(hs[i], &in[i], T[i], L[i]);
    if (rc != DMV_OK) return many ? ct_member_error(rc, i) : rc;
  }
  int rc = ct_cluster_ready(hs, n, many, T, n > 1 ? B->maps : &Q->maps);
  if (rc != DMV_OK) return rc;
  for (int i = 0; i < n; i++) {
    dmv_ct* c = hs[i];
    CK(c->h_tries.reserve(1));
    L[i].out = c->h_tries;
    if (n > 1) {   // the kernel reads the try table from pinned memory: no earlier call still reads it, every call synchronises before it returns
      CK(c->h_pose.reserve((size_t)DMV_CT_MAX_TRIES * 12));
      ct_fill_tries(&in[i], reinterpret_cast<CTPose*>(c->h_pose.get()));
      B->pose[i] = reinterpret_cast<const CTPose*>(c->h_pose.get());
    }
  }
  if (n == 1) {
    ct_fill_tries(&in[0], Q->pose);
    void* args[] = {Q.get()};
    rc = ct_cluster_launch(hs, 1, (const void*)ct_track_tries_kernel, args);
  } else {
    void* args[] = {B.get()};
    rc = ct_cluster_launch(hs, n, (const void*)ct_track_tries_many_kernel, args);
  }
  if (rc != DMV_OK) return rc;
  for (int i = 0; i < n; i++) out[i] = *hs[i]->h_tries;
  return DMV_OK;
}

int dmv_ct_track_tries(dmv_ct* c, const dmv_ct_tries_args* in, dmv_ct_tries_result* out) {
  if (!c || !in || !out) return set_error(DMV_ERR_INVALID, "null argument");
  return ct_tries_run(&c, 1, in, out, false);
}

int dmv_ct_track_tries_many(dmv_ct* const* handles, int n, const dmv_ct_tries_args* in, dmv_ct_tries_result* out) {
  if (!handles || !in || !out) return set_error(DMV_ERR_INVALID, "null argument");
  const int rc = ct_check_members(handles, n, DMV_CT_TRACK_MANY_MAX);
  return rc != DMV_OK ? rc : ct_tries_run(handles, n, in, out, true);
}

// library-internal: the resident level-0 float4 plane of the coarse-tracker handle (dmv_ba_adopt_frame copies it device-to-device)
__attribute__((visibility("hidden"))) int dmv_ct_level0_plane(dmv_ct* c, const void** plane, int* w, int* h, int* device, cudaStream_t* stream) {
  if (!c) return set_error(DMV_ERR_INVALID, "null handle");
  *plane = c->d_img[0]; *w = c->w[0]; *h = c->h[0]; *device = c->device; *stream = c->stream;
  return DMV_OK;
}

int dmv_ct_set_timing(dmv_ct* c, int enable) {
  if (!c) return set_error(DMV_ERR_INVALID, "null handle");
  c->timing = enable != 0;
  return DMV_OK;
}
int dmv_ct_last_timing(dmv_ct* c, float ms[4]) {
  if (!c || !ms) return set_error(DMV_ERR_INVALID, "null argument");
  for (int i = 0; i < 4; i++) ms[i] = c->last_ms[i];
  return DMV_OK;
}
// instrumentation: reference points evaluated by the last dmv_ct_track, summed over its calcRes / calcGSSSE evaluations.  After a
// dmv_ct_calc_res_gs it reads sum 26 of that call's 53, which share the pinned block.
int dmv_ct_last_point_evaluations(dmv_ct* c, double* n) {
  if (!c || !n) return set_error(DMV_ERR_INVALID, "null argument");
  *n = ct_track_out(c)->pevals;
  return DMV_OK;
}
int dmv_ct_kernel_launch_count(dmv_ct* c, long long* n) {
  if (!c || !n) return set_error(DMV_ERR_INVALID, "null argument");
  *n = c->launches;
  return DMV_OK;
}

}  // extern "C"
