// dmv_ba_select_activation — the selection half of FullSystem::activatePointsMT (reference FullSystem.cpp:L642-717): which immature points
// are deleted, kept, or handed to optimizeImmaturePoint, and in which order (toOptimize).
//
//   1. CoarseDistanceMap::makeDistanceMap (CoarseTracker.cpp:L931-967): every active point of the other frames is projected into the newest
//      frame at level 1 and its cell set to 0; growDistBFS (L979-1073) then writes step k into every unreached cell next to a cell of step
//      k-1, for k = 1..39.
//   2. The loop over the immature points of every other frame: delete (non-finite idepth_max, IPS_OUTLIER, not ready on a flagged host or with
//      IPS_OOB, projection outside), keep (not ready), or read the map at the projection; an accepted point runs addIntoDistFinal
//      (L1076-1082): its cell is set to 0 and growDistBFS floods from it alone, on top of the map as the earlier points left it.
//
// Where exactness is decided:
//   - The projection.  KRKi * (u, v, 1) + Kt * x is evaluated as ip_trace.cu / ct_depth.cu reproduce Eigen's order: ((K0*u + K1*v) + K2*1) +
//     Kt*x per row, then ptp[0] / ptp[2] + 0.5f.  The conversion to int truncates as x86's cvttss2si does: NaN, infinities and values outside
//     int's range become INT_MIN (CUDA's conversion saturates, or gives 0 for NaN); sel_cvtt states it explicitly.
//   - The map BFS.  At step k every write stores k and tests "> k", and the cells that expand at step k are exactly those written at step k-1,
//     so the set written at step k does not depend on the order in which the frontier is walked.  A level-synchronous pull (a cell looks for a
//     neighbour written at step k-1) therefore gives the reference's map exactly.  The reference's rules are kept: the 8-neighbourhood on odd k
//     and the 4-neighbourhood on even k (the `k%2==0` branch of growDistBFS), no expansion from a cell on the one-pixel border, k <= 39, 1000
//     where nothing reaches.  In the initial build the cells written at step k-1 are those holding k-1; in a flood they are tracked in a
//     window of step stamps around the seed, because the map already holds other cells of value k-1 that must not expand.
//   - The greedy selection.  A decision reads one cell of the map as all earlier accepted points left it.  A flood's result depends on the
//     map it runs on (blocking, and the parity of the step it arrives with), so the map after several overlapping floods is neither a
//     per-seed minimum nor independent of their order (tests/test_ref_pin_activation.py shows both against the reference's BFS): floods
//     that can meet run in loop order.  Three exact reductions split the rest:
//       * static decisions (sel_classify_kernel): the map never rises above its value before the loop (map0) and never falls below 0, and
//         float addition is monotone, so map0 + frac < thr keeps the point and 0 + frac >= thr accepts it, without waiting for any flood.
//         Only the others ("undecided") read the map in the chain.  With currentMinActDist = 0 every candidate is decided statically.
//       * reach (sel_reach_kernel): a flood writes a cell at distance d (Chebyshev) only at a step k >= d and only if the cell's value,
//         <= map0, exceeds k; the written cells are 8-connected around the seed.  So the first ring d with no cell of map0 > d bounds the
//         flood to the box of radius d-1 around its seed, whatever ran before it: a flood reads and writes the map inside its box only.
//         Two events whose boxes are disjoint commute, and a decision depends only on earlier floods whose box holds its cell.
//       * floods nobody reads: when the caller does not ask for the map, a flood after the last undecided candidate changes nothing that is
//         returned and is not run.
//     sel_chain_kernel (one CTA) keeps the remaining events (undecided candidates, and accepted points whose flood is needed) in loop order
//     and runs them in rounds: each pending event claims the tiles its box covers with an atomicMin of its position, an event that owns all
//     its tiles has no earlier pending event that can interact with it, and all such events run at once, one warp each (the decision, then
//     the flood, level-synchronously across the warp).  The earliest pending event always owns its tiles, so every round makes progress.
//     toOptimize is then the accepted points in loop order.  stats reports the undecided candidates, the floods run and the rounds.
//
// THIS TRANSLATION UNIT IS COMPILED WITH -fmad=false: no FMA contraction, IEEE division, so every float decision is the reference's.
#include "../../include/dmvio_b200.h"
#include "ba_handle.h"
#include "common_host.h"
#include "ip_store.h"
#include "ip_trace.h"
#include <algorithm>
#include <climits>
#include <cstring>
#include <cub/block/block_scan.cuh>
#include <cuda_runtime.h>
#include <math.h>

namespace dmv {
namespace {

constexpr int SEL_T = 1024;    // threads of the chain CTA
constexpr int SEL_R = 39;      // growDistBFS: for (k = 1; k < 40; k++)
constexpr int SEL_CAND = 3;    // provisional action: undecided, read from the map in the chain

struct SelArgs {
  int n, na, nf, newest, w1, h1;
  int want_map;                // the caller asked for the final map: every accepted point floods
  int tile;                    // side of the chain's ownership tiles (cells)
  float minActDist, minTraceQuality;
  const float* tab;            // nf * 12: KRKi | Kt
  const int* flagged;
  const int* off;
  const float *au, *av, *aid;
  const int* ah;
  const float *u, *v, *idmin, *idmax;
  const int* status;
  const float *interval, *quality, *type;
  int* action;
  int* opt;
  int* counters;               // [0] toOptimize size, [1] floods run, [2] rounds of the chain, [4] undecided candidates
  const int* last_undecided;   // &counters[3]: the last undecided candidate (-1: none)
  float* map;
  int* cell;
  float* frac;
  int* rad;                    // per point: reach of its flood (sel_reach_kernel), -1 = not an event of the chain
  int* stamp;                  // per cell: (flood id << 6) | step of the last flood that wrote it, -1 initially
};

// (int)f as x86-64 converts a float (cvttss2si): truncation, and INT_MIN for NaN, infinities and values outside int's range
__device__ __forceinline__ int sel_cvtt(float f) { return (f >= -2147483648.f && f < 2147483648.f) ? (int)f : INT_MIN; }

// Vec3f ptp = KRKi * Vec3f(u, v, 1) + Kt * x;  int u = ptp[0] / ptp[2] + 0.5f;  int v = ...;  (u > 0 && v > 0 && u < w1 && v < h1)
__device__ __forceinline__ bool sel_project(const float* __restrict__ T, float u, float v, float x, int w1, int h1, int& cu, int& cv, float& p0) {
  float ptp[3];
#pragma unroll
  for (int k = 0; k < 3; k++) ptp[k] = ((T[3 * k] * u + T[3 * k + 1] * v) + T[3 * k + 2] * 1.0f) + T[9 + k] * x;
  cu = sel_cvtt(ptp[0] / ptp[2] + 0.5f);
  cv = sel_cvtt(ptp[1] / ptp[2] + 0.5f);
  p0 = ptp[0];
  return cu > 0 && cv > 0 && cu < w1 && cv < h1;
}

// the neighbours a cell expands to at step k: growDistBFS's `k%2==0` branch has 4, the other 8
__device__ __constant__ int c_sel_nb[8][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}, {1, 1}, {-1, 1}, {-1, -1}, {1, -1}};

__device__ __forceinline__ bool sel_inner(int x, int y, int w1, int h1) { return x > 0 && y > 0 && x < w1 - 1 && y < h1 - 1; }

__global__ void sel_map_init_kernel(float* __restrict__ map, int ncell) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ncell) map[i] = 1000.f;
}

// makeDistanceMap's projection loop: every in-bounds active point of another frame seeds its cell with 0 (duplicates write the same value)
__global__ void sel_seed_kernel(const SelArgs A) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.na) return;
  const int h = A.ah[p];
  if (h == A.newest) return;
  int cu, cv;
  float p0;
  if (sel_project(A.tab + 12 * h, A.au[p], A.av[p], A.aid[p], A.w1, A.h1, cu, cv, p0)) A.map[cu + A.w1 * cv] = 0.f;
}

// growDistBFS step k on the whole map, pulled: an unreached cell (> k) takes k if a neighbour of the step's neighbourhood holds k-1 (= was
// written at step k-1) and is not on the border.  Cells written in this step hold k, which no other cell of the step reads as k-1.
__global__ void sel_bfs_step_kernel(float* __restrict__ map, int w1, int h1, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w1 * h1) return;
  if (!(map[i] > (float)k)) return;
  const int x = i % w1, y = i / w1;
  const int nn = (k % 2 == 0) ? 4 : 8;
  const float prev = (float)(k - 1);
  for (int d = 0; d < nn; d++) {
    const int nx = x + c_sel_nb[d][0], ny = y + c_sel_nb[d][1];
    if (sel_inner(nx, ny, w1, h1) && map[nx + w1 * ny] == prev) { map[i] = (float)k; return; }
  }
}

// the loop body up to the map read: delete / keep / candidate (with its cell and ptp[0] - floorf(ptp[0]))
__global__ void sel_classify_kernel(const SelArgs A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  int h = 0;
  while (A.off[h + 1] <= i) h++;
  int act = DMV_ACT_KEEP;
  if (h != A.newest) {
    const int st = A.status[i];
    const float imin = A.idmin[i], imax = A.idmax[i];
    if (!isfinite(imax) || st == 2) {   // IPS_OUTLIER
      act = DMV_ACT_DELETE;
    } else {
      const bool canActivate = (st == 0 || st == 3 || st == 4 || st == 1) && A.interval[i] < 8 && A.quality[i] > A.minTraceQuality && (imax + imin) > 0;
      if (!canActivate) {
        if (A.flagged[h] || st == 1) act = DMV_ACT_DELETE;   // IPS_OOB
      } else {
        int cu, cv;
        float p0;
        if (sel_project(A.tab + 12 * h, A.u[i], A.v[i], 0.5f * (imax + imin), A.w1, A.h1, cu, cv, p0)) {
          // The map only decreases below its value before the loop (map0, what A.map holds now) and never below 0, and float addition is
          // monotone: a point whose distance on map0 fails is kept whatever the floods do, and one whose distance on a 0 passes is accepted.
          const int c = cu + A.w1 * cv;
          const float frac = p0 - floorf((float)(p0)), thr = A.minActDist * A.type[i];
          A.cell[i] = c;
          A.frac[i] = frac;
          if (!(A.map[c] + frac >= thr)) act = DMV_ACT_KEEP;
          else if (0.f + frac >= thr) act = DMV_ACT_OPTIMIZE;
          else { act = SEL_CAND; atomicMax(A.counters + 3, i); atomicAdd(A.counters + 4, 1); }
        } else {
          act = DMV_ACT_DELETE;
        }
      }
    }
  }
  A.action[i] = act;
}

// How far a flood from cell c can write, bounded by the map before the loop (map0): the cells a flood writes form an 8-connected set around
// its seed, a cell x at Chebyshev distance d is written at a step k >= d and only if its current value, which is <= map0(x), exceeds k.  So
// if no cell of ring d has map0 > d, nothing at distance >= d is written, whatever other floods did before.  One warp per event; rad = -1
// for a point that is not an event of the chain.
__global__ void sel_reach_kernel(const SelArgs A) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= A.n) return;
  const int act = A.action[i];
  const bool ev = act == SEL_CAND || (act == DMV_ACT_OPTIMIZE && (A.want_map || i < *A.last_undecided));
  if (!ev) { if (lane == 0) A.rad[i] = -1; return; }
  const int w1 = A.w1, h1 = A.h1, cx = A.cell[i] % w1, cy = A.cell[i] / w1;
  int r = SEL_R;
  for (int d = 1; d <= SEL_R; d++) {
    bool open = false;
    for (int j = lane; j < 8 * d; j += 32) {   // ring d: 8d cells
      const int side = j / (2 * d), o = j % (2 * d);
      const int x = side == 0 ? cx - d + o : side == 1 ? cx + d : side == 2 ? cx + d - o : cx - d;
      const int y = side == 0 ? cy - d : side == 1 ? cy - d + o : side == 2 ? cy + d : cy + d - o;
      if (x >= 0 && y >= 0 && x < w1 && y < h1 && A.map[x + w1 * y] > (float)d) open = true;
    }
    if (!__any_sync(0xffffffffu, open)) { r = d - 1; break; }
  }
  if (lane == 0) A.rad[i] = r;
}

// addIntoDistFinal(c) by one warp, all 39 steps but only over the cells within rad of the seed (nothing further can be written, see
// sel_reach_kernel); it stops at the first step that writes nothing, as growDistBFS's frontier empties.
// stamp[x] = (fid << 6) | k marks the cells this flood wrote at step k: the map already holds other cells of value k-1 that must not expand.
__device__ void sel_flood_warp(const SelArgs& A, int c, int rad, int fid) {
  const int lane = threadIdx.x & 31, w1 = A.w1, h1 = A.h1, sx = c % w1, sy = c / w1;
  if (lane == 0) { A.map[c] = 0.f; A.stamp[c] = fid << 6; }
  __syncwarp();
  for (int k = 1; k <= SEL_R; k++) {   // rad bounds where the flood can write, not when: a cell inside can still be reached late
    const int r = min(k, rad);
    const int x0 = max(sx - r, 0), x1 = min(sx + r, w1 - 1), y0 = max(sy - r, 0), y1 = min(sy + r, h1 - 1);
    const int W = x1 - x0 + 1, cnt = W * (y1 - y0 + 1);
    const int nn = (k % 2 == 0) ? 4 : 8, want = (fid << 6) | (k - 1);
    bool any = false;
    for (int j = lane; j < cnt; j += 32) {
      const int x = x0 + j % W, y = y0 + j / W, idx = x + w1 * y;
      if (!(A.map[idx] > (float)k)) continue;
      for (int d = 0; d < nn; d++) {
        const int nx = x + c_sel_nb[d][0], ny = y + c_sel_nb[d][1];
        if (sel_inner(nx, ny, w1, h1) && A.stamp[nx + w1 * ny] == want) {
          A.map[idx] = (float)k;
          A.stamp[idx] = (fid << 6) | k;
          any = true;
          break;
        }
      }
    }
    if (!__any_sync(0xffffffffu, any)) break;   // also orders this step's writes before the next step's reads
  }
}

constexpr int SEL_P = 2048;          // pending events held by the chain
constexpr int SEL_TILES = 4096;      // tile-owner slots

// The loop over the candidates, decomposed exactly (see the file header).  One CTA: pending events are kept in loop order; every round,
// each pending event claims the tiles its reach box covers (atomicMin of its pending slot), and an event that owns all its tiles has no
// earlier pending event whose box meets its own.  Those events are independent of each other and of everything still pending before them:
// each is run by one warp (the decision, then the flood).  Afterwards toOptimize is the accepted points in loop order.
__global__ void __launch_bounds__(SEL_T) sel_chain_kernel(const SelArgs A) {
  using Scan = cub::BlockScan<int, SEL_T>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int owner[SEL_TILES];
  __shared__ int pend[2][SEL_P];
  __shared__ int ready[SEL_P];
  __shared__ int s_n, s_nready, s_fid, s_total;
  const int tid = threadIdx.x, warp = tid >> 5, T = A.tile, tw = (A.w1 + T - 1) / T, th = (A.h1 + T - 1) / T, ntiles = tw * th;
  int cur = 0, next = 0, rounds = 0;
  if (tid == 0) { s_n = 0; s_fid = 0; }
  __syncthreads();
  while (true) {
    // refill in loop order, SEL_T points at a time, while a whole chunk of events fits
    while (next < A.n && s_n <= SEL_P - SEL_T) {
      const int i = next + tid;
      const int ev = (i < A.n && A.rad[i] >= 0) ? 1 : 0;
      int pos, tot;
      Scan(scan_tmp).ExclusiveSum(ev, pos, tot);
      if (ev) pend[cur][s_n + pos] = i;
      __syncthreads();
      if (tid == 0) s_n += tot;
      next += SEL_T;
      __syncthreads();
    }
    const int np = s_n;
    if (np == 0) break;
    rounds++;
    for (int t = tid; t < ntiles; t += SEL_T) owner[t] = INT_MAX;
    if (tid == 0) s_nready = 0;
    __syncthreads();
    for (int s = tid; s < np; s += SEL_T) {
      const int i = pend[cur][s], r = A.rad[i], c = A.cell[i], cx = c % A.w1, cy = c / A.w1;
      const int tx0 = max(cx - r, 0) / T, tx1 = min(cx + r, A.w1 - 1) / T, ty0 = max(cy - r, 0) / T, ty1 = min(cy + r, A.h1 - 1) / T;
      for (int ty = ty0; ty <= ty1; ty++)
        for (int tx = tx0; tx <= tx1; tx++) atomicMin(&owner[tx + tw * ty], s);
    }
    __syncthreads();
    for (int s = tid; s < np; s += SEL_T) {
      const int i = pend[cur][s], r = A.rad[i], c = A.cell[i], cx = c % A.w1, cy = c / A.w1;
      const int tx0 = max(cx - r, 0) / T, tx1 = min(cx + r, A.w1 - 1) / T, ty0 = max(cy - r, 0) / T, ty1 = min(cy + r, A.h1 - 1) / T;
      bool mine = true;
      for (int ty = ty0; ty <= ty1 && mine; ty++)
        for (int tx = tx0; tx <= tx1; tx++)
          if (owner[tx + tw * ty] != s) { mine = false; break; }
      if (mine) ready[atomicAdd(&s_nready, 1)] = s;
    }
    __syncthreads();
    const int nr = s_nready;
    for (int q = warp; q < nr; q += SEL_T / 32) {
      const int i = pend[cur][ready[q]];
      bool flood = A.action[i] == DMV_ACT_OPTIMIZE;
      if (!flood) {   // undecided: the map at its cell as every earlier accepted point that can reach it left it
        flood = A.map[A.cell[i]] + A.frac[i] >= A.minActDist * A.type[i];
        __syncwarp();
        if ((threadIdx.x & 31) == 0) A.action[i] = flood ? DMV_ACT_OPTIMIZE : DMV_ACT_KEEP;
        flood = flood && (A.want_map || i < *A.last_undecided);
      }
      if (flood) {
        int fid = 0;
        if ((threadIdx.x & 31) == 0) fid = atomicAdd(&s_fid, 1);
        sel_flood_warp(A, A.cell[i], A.rad[i], __shfl_sync(0xffffffffu, fid, 0));
      }
      __syncwarp();
      if ((threadIdx.x & 31) == 0) pend[cur][ready[q]] = -1;   // done
    }
    __syncthreads();
    // drop the finished events, keeping loop order
    int keep[SEL_P / SEL_T], cnt = 0;
#pragma unroll
    for (int u = 0; u < SEL_P / SEL_T; u++) { const int s = tid * (SEL_P / SEL_T) + u; keep[u] = (s < np && pend[cur][s] >= 0); cnt += keep[u]; }
    int pos, tot;
    Scan(scan_tmp).ExclusiveSum(cnt, pos, tot);
#pragma unroll
    for (int u = 0; u < SEL_P / SEL_T; u++) {
      const int s = tid * (SEL_P / SEL_T) + u;
      if (keep[u]) pend[cur ^ 1][pos++] = pend[cur][s];
    }
    __syncthreads();
    if (tid == 0) s_n = tot;
    cur ^= 1;
    __syncthreads();
  }
  // toOptimize: the accepted points in loop order
  if (tid == 0) s_total = 0;
  __syncthreads();
  for (int base = 0; base < A.n; base += SEL_T) {
    const int i = base + tid;
    const int acc = (i < A.n && A.action[i] == DMV_ACT_OPTIMIZE) ? 1 : 0;
    int pos, tot;
    Scan(scan_tmp).ExclusiveSum(acc, pos, tot);
    if (acc) A.opt[s_total + pos] = i;
    __syncthreads();
    if (tid == 0) s_total += tot;
    __syncthreads();
  }
  if (tid == 0) { A.counters[0] = s_total; A.counters[1] = s_fid; A.counters[2] = rounds; }
}

// Staging layout (4-byte words): tab 96 | flagged 8 | off 9 (header 128) | active u v idepth host | immature u v idmin idmax status interval
// quality type | action | opt | counters 8 | map | cell | frac | rad | stamp.  [0, act) goes up, [act, map (+ ncell)) comes back.
struct SelLayout {
  size_t au, av, aid, ah, iu, iv, imin, imax, ist, iint, iq, ity, act, opt, cnt, map, cell, frac, rad, stamp, words;
  SelLayout(size_t n, size_t na, size_t ncell) {
    au = 128; av = au + na; aid = av + na; ah = aid + na; iu = ah + na; iv = iu + n; imin = iv + n; imax = imin + n; ist = imax + n; iint = ist + n;
    iq = iint + n; ity = iq + n; act = ity + n; opt = act + n; cnt = opt + n; map = cnt + 8; cell = map + ncell; frac = cell + n; rad = frac + n;
    stamp = rad + n; words = stamp + ncell;
  }
};

// The selection's immature-point rows fed from a store: row i of group f = row src[f] + i - off[f] of the store's buffer (capacity scap).
// Copies the 7 words the selection reads from the store (u, v, idepth_min, idepth_max, status, interval, quality) into the staging arrays.
struct SelGatherArgs {
  int n, nf, scap;
  int off[MAXF + 1], src[MAXF];
  const unsigned* pts;
  unsigned* dst;      // the staging's u (the 7 arrays follow it at stride n)
};
__global__ void __launch_bounds__(128) sel_gather_kernel(const __grid_constant__ SelGatherArgs G) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G.n) return;
  int f = 0;
  while (G.off[f + 1] <= i) f++;
  const size_t r = G.src[f] + (i - G.off[f]), cap = G.scap, n = G.n;
  G.dst[i] = G.pts[ipw::u * cap + r];
  G.dst[n + i] = G.pts[ipw::v * cap + r];
  G.dst[2 * n + i] = G.pts[ipw::idepth_min * cap + r];
  G.dst[3 * n + i] = G.pts[ipw::idepth_max * cap + r];
  G.dst[4 * n + i] = G.pts[ipw::status * cap + r];
  G.dst[5 * n + i] = G.pts[ipw::interval * cap + r];
  G.dst[6 * n + i] = G.pts[ipw::quality * cap + r];
}

}  // namespace

int sel_check(const dmv_ba* b, const dmv_ba_select_args* a, bool from_store) {
  const int nf = a->nf;
  if (nf < 1 || nf > DMV_MAX_FRAMES || a->newest < 0 || a->newest >= nf) return set_error(DMV_ERR_INVALID, "nf %d / newest %d out of range", nf, a->newest);
  if (!a->tables12 || !a->flagged || !a->imm_offset || !a->n_opt || a->n_active < 0 || a->cap < 0)
    return set_error(DMV_ERR_INVALID, "incomplete dmv_ba_select_args");
  if (a->n_active > 0 && (!a->act_u || !a->act_v || !a->act_idepth_scaled || !a->act_host)) return set_error(DMV_ERR_INVALID, "incomplete active points");
  if (a->imm_offset[0] != 0) return set_error(DMV_ERR_INVALID, "imm_offset[0] must be 0");
  for (int f = 0; f < nf; f++)
    if (a->imm_offset[f + 1] < a->imm_offset[f]) return set_error(DMV_ERR_INVALID, "imm_offset decreases at frame %d", f);
  const int n = a->imm_offset[nf], na = a->n_active;
  if (!from_store && n > 0 && (!a->u || !a->v || !a->idepth_min || !a->idepth_max || !a->lastTraceStatus || !a->lastTracePixelInterval || !a->quality ||
                               !a->my_type || !a->action || (a->cap > 0 && !a->opt_idx)))
    return set_error(DMV_ERR_INVALID, "incomplete immature points");
  for (int p = 0; p < na; p++)
    if (a->act_host[p] < 0 || a->act_host[p] >= nf) return set_error(DMV_ERR_INVALID, "active point %d: host %d out of range", p, a->act_host[p]);
  if ((b->cfg.w >> 1) < 3 || (b->cfg.h >> 1) < 3) return set_error(DMV_ERR_INVALID, "image too small for a level-1 distance map");
  return DMV_OK;
}

// the header and the active points into h_sel, d_sel and h_sel grown to the layout
static int sel_stage(dmv_ba* b, const dmv_ba_select_args* a, const SelLayout& o) {
  const int nf = a->nf, na = a->n_active;
  CK(cudaSetDevice(b->device));
  CK(b->d_sel.reserve(o.words));
  CK(b->h_sel.reserve(o.words));
  float* hb = b->h_sel;
  int* hi = reinterpret_cast<int*>(hb);
  std::memcpy(hb, a->tables12, sizeof(float) * 12 * nf);
  for (int f = 0; f < nf; f++) hi[96 + f] = a->flagged[f] != 0;
  std::memcpy(hi + 104, a->imm_offset, sizeof(int) * (nf + 1));
  if (na > 0) {
    std::memcpy(hb + o.au, a->act_u, 4 * (size_t)na); std::memcpy(hb + o.av, a->act_v, 4 * (size_t)na);
    std::memcpy(hb + o.aid, a->act_idepth_scaled, 4 * (size_t)na); std::memcpy(hi + o.ah, a->act_host, 4 * (size_t)na);
  }
  return DMV_OK;
}

// The selection on the staged d_sel (map init, seed, the 39 BFS steps, classify, reach, chain), its read-back and one synchronisation;
// then a's outputs.  Returns DMV_ERR_INVALID when toOptimize exceeds cap (*n_opt, action, map and stats written).
static int sel_launch(dmv_ba* b, const dmv_ba_select_args* a, const SelLayout& o) {
  const int n = a->imm_offset[a->nf], na = a->n_active, w1 = b->cfg.w >> 1, h1 = b->cfg.h >> 1, ncell = w1 * h1;
  float* hb = b->h_sel;
  int* hi = reinterpret_cast<int*>(hb);
  float* d = b->d_sel;
  int* di = reinterpret_cast<int*>(d);
  SelArgs A;
  A.n = n; A.na = na; A.nf = a->nf; A.newest = a->newest; A.w1 = w1; A.h1 = h1; A.want_map = a->map != nullptr;
  A.tile = 8;
  while (((w1 + A.tile - 1) / A.tile) * ((h1 + A.tile - 1) / A.tile) > SEL_TILES) A.tile *= 2;
  A.minActDist = a->currentMinActDist; A.minTraceQuality = a->minTraceQuality;
  A.tab = d; A.flagged = di + 96; A.off = di + 104;
  A.au = d + o.au; A.av = d + o.av; A.aid = d + o.aid; A.ah = di + o.ah;
  A.u = d + o.iu; A.v = d + o.iv; A.idmin = d + o.imin; A.idmax = d + o.imax; A.status = di + o.ist; A.interval = d + o.iint; A.quality = d + o.iq;
  A.type = d + o.ity; A.action = di + o.act; A.opt = di + o.opt; A.counters = di + o.cnt; A.map = d + o.map; A.cell = di + o.cell; A.frac = d + o.frac;
  A.last_undecided = di + o.cnt + 3; A.rad = di + o.rad; A.stamp = di + o.stamp;
  const cudaStream_t s = b->stream;
  CK(cudaMemsetAsync(di + o.cnt, 0, 4 * 8, s));
  CK(cudaMemsetAsync(di + o.cnt + 3, 0xFF, 4, s));
  CK(cudaMemsetAsync(A.stamp, 0xFF, 4 * (size_t)ncell, s));
  sel_map_init_kernel<<<(ncell + 255) / 256, 256, 0, s>>>(A.map, ncell);
  if (na > 0) sel_seed_kernel<<<(na + 255) / 256, 256, 0, s>>>(A);
  for (int k = 1; k <= SEL_R; k++) sel_bfs_step_kernel<<<(ncell + 255) / 256, 256, 0, s>>>(A.map, w1, h1, k);
  if (n > 0) {
    sel_classify_kernel<<<(n + 255) / 256, 256, 0, s>>>(A);
    sel_reach_kernel<<<(n + 7) / 8, 256, 0, s>>>(A);
  }
  sel_chain_kernel<<<1, SEL_T, 0, s>>>(A);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(hb + o.act, d + o.act, 4 * (o.map - o.act + (a->map ? (size_t)ncell : 0)), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const int nopt = hi[o.cnt];
  if (n > 0) std::memcpy(a->action, hi + o.act, 4 * (size_t)n);
  if (a->map) std::memcpy(a->map, hb + o.map, 4 * (size_t)ncell);
  if (a->stats) { a->stats[0] = hi[o.cnt + 4]; a->stats[1] = hi[o.cnt + 1]; a->stats[2] = hi[o.cnt + 2]; }
  *a->n_opt = nopt;
  if (nopt > a->cap) return set_error(DMV_ERR_INVALID, "%d points to optimise exceed cap %d", nopt, a->cap);
  if (nopt > 0) std::memcpy(a->opt_idx, hi + o.opt, 4 * (size_t)nopt);
  return DMV_OK;
}

int ip_select_from_store(dmv_ba* b, const dmv_ba_select_args* a, const dmv_ip_store* s, const int* slot, const float* const* my_type, const int** d_opt) {
  const int nf = a->nf, n = a->imm_offset[nf];
  const SelLayout o(n, a->n_active, (size_t)(b->cfg.w >> 1) * (b->cfg.h >> 1));
  int rc = sel_stage(b, a, o);
  if (rc != DMV_OK) return rc;
  float* hb = b->h_sel;
  float* d = b->d_sel;
  SelGatherArgs G;
  G.n = n; G.nf = nf; G.scap = s->cap[s->cur];
  for (int f = 0; f < nf; f++) {
    G.off[f] = a->imm_offset[f];
    G.src[f] = slot[f] >= 0 ? ip_store_first(s, slot[f]) : 0;
    const int m = a->imm_offset[f + 1] - a->imm_offset[f];
    if (m > 0) std::memcpy(hb + o.ity + a->imm_offset[f], my_type[f], 4 * (size_t)m);
  }
  G.off[nf] = n;
  G.pts = reinterpret_cast<const unsigned*>(s->d_pts[s->cur].get());
  G.dst = reinterpret_cast<unsigned*>(d + o.iu);
  CK(cudaMemcpyAsync(d, hb, 4 * o.iu, cudaMemcpyHostToDevice, b->stream));
  if (n > 0) {
    CK(cudaMemcpyAsync(d + o.ity, hb + o.ity, 4 * (size_t)n, cudaMemcpyHostToDevice, b->stream));
    sel_gather_kernel<<<(n + 127) / 128, 128, 0, b->stream>>>(G);
  }
  rc = sel_launch(b, a, o);
  *d_opt = reinterpret_cast<const int*>(d + o.opt);
  return rc;
}

}  // namespace dmv

using namespace dmv;

extern "C" int dmv_ba_select_activation(dmv_ba* b, const dmv_ba_select_args* a) {
  if (!b || !a) return set_error(DMV_ERR_INVALID, "null argument");
  int rc = sel_check(b, a, false);
  if (rc != DMV_OK) return rc;
  const int n = a->imm_offset[a->nf];
  const SelLayout o(n, a->n_active, (size_t)(b->cfg.w >> 1) * (b->cfg.h >> 1));
  rc = sel_stage(b, a, o);
  if (rc != DMV_OK) return rc;
  float* hb = b->h_sel;
  int* hi = reinterpret_cast<int*>(hb);
  if (n > 0) {
    std::memcpy(hb + o.iu, a->u, 4 * (size_t)n); std::memcpy(hb + o.iv, a->v, 4 * (size_t)n);
    std::memcpy(hb + o.imin, a->idepth_min, 4 * (size_t)n); std::memcpy(hb + o.imax, a->idepth_max, 4 * (size_t)n);
    std::memcpy(hi + o.ist, a->lastTraceStatus, 4 * (size_t)n); std::memcpy(hb + o.iint, a->lastTracePixelInterval, 4 * (size_t)n);
    std::memcpy(hb + o.iq, a->quality, 4 * (size_t)n); std::memcpy(hb + o.ity, a->my_type, 4 * (size_t)n);
  }
  CK(cudaMemcpyAsync(b->d_sel, hb, 4 * o.act, cudaMemcpyHostToDevice, b->stream));
  return sel_launch(b, a, o);
}
