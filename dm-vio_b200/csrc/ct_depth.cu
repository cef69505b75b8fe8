// Coarse-tracking reference construction on the device (SURVEY.md §8a-B1 / §8f-3): CoarseTracker::makeCoarseDepthL0
// (reference FullSystem/CoarseTracker.cpp:L138-295) — weighted splat of the keyframe's IN residuals, 2x2 sum pooling to the coarser
// levels, one dilation step per level (diagonal neighbours on levels 0-1, 4-neighbourhood above), normalisation and ORDER-PRESERVING
// compaction into the pc_u / pc_v / pc_idepth / pc_color lists that calcRes reads.  Bit-identical to the CPU code:
//   * the splat is the only order-dependent float sum (points that hit the same pixel): the host folds colliding points in input order
//     (exactly the reference's sequential +=) and the device scatters collision-free entries;
//   * dilation reads only originally-valid pixels and writes only originally-empty ones, so the in-place sweep of the reference is
//     order-independent; pooling / dilation keep the reference's operand order; there is no multiply-add to contract;
//   * compaction = per-row counts, an exclusive scan over the rows, ballot-prefix writes: row-major order like the reference's loops.
// Fed from a BA handle (dmv_ct_set_ref_from_ba) the fold runs here too: a stable radix sort of (pixel, point index) puts the points that
// hit one pixel next to each other in input order, and one thread per pixel adds its run in that order — the reference's sequential +=.
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include "ct_depth.h"
#include <cub/device/device_radix_sort.cuh>

namespace dmv {

__global__ void cd_scatter_kernel(int n, const int* __restrict__ pix, const float* __restrict__ idw, const float* __restrict__ wsum, float* idepth0, float* ws0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { idepth0[pix[i]] = idw[i]; ws0[pix[i]] = wsum[i]; }
}

__global__ void cd_pool_kernel(const float* __restrict__ id_lm, const float* __restrict__ ws_lm, float* id_l, float* ws_l, int wl, int hl, int wlm1) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= wl || y >= hl) return;
  const int b = 2 * x + 2 * y * wlm1;
  id_l[x + y * wl] = id_lm[b] + id_lm[b + 1] + id_lm[b + wlm1] + id_lm[b + wlm1 + 1];
  ws_l[x + y * wl] = ws_lm[b] + ws_lm[b + 1] + ws_lm[b + wlm1] + ws_lm[b + wlm1 + 1];
}

// ws_bak = weights before the sweep (read only), ws_out = weights after it, idl updated in place (see the file header)
__global__ void cd_dilate_kernel(const float* __restrict__ ws_bak, float* __restrict__ ws_out, float* idl, int wl, int hl, int diagonal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int npx = wl * hl;
  if (i >= npx) return;
  float wv = ws_bak[i];
  const int wh = npx - wl;
  if (i >= wl + 1 && i < wh - 1 && wv <= 0) {
    const int o0 = diagonal ? 1 + wl : 1, o1 = diagonal ? -1 - wl : -1, o2 = diagonal ? wl - 1 : wl, o3 = diagonal ? -wl + 1 : -wl;
    float sum = 0, num = 0, numn = 0;
    if (ws_bak[i + o0] > 0) { sum += idl[i + o0]; num += ws_bak[i + o0]; numn++; }
    if (ws_bak[i + o1] > 0) { sum += idl[i + o1]; num += ws_bak[i + o1]; numn++; }
    if (ws_bak[i + o2] > 0) { sum += idl[i + o2]; num += ws_bak[i + o2]; numn++; }
    if (ws_bak[i + o3] > 0) { sum += idl[i + o3]; num += ws_bak[i + o3]; numn++; }
    if (numn > 0) { idl[i] = sum / numn; wv = num / numn; }
  }
  ws_out[i] = wv;
}

__device__ __forceinline__ bool cd_valid(const float* ws, const float* idl, const float4* img, int i, float& q, float& col) {
  const float w = ws[i];
  if (!(w > 0)) return false;
  q = idl[i] / w;
  col = img[i].x;
  return isfinite(col) && (q > 0);
}

// one warp per row y in [2, hl-2): number of list entries of the row
__global__ void cd_rowcount_kernel(const float* __restrict__ ws, const float* __restrict__ idl, const float4* __restrict__ img, int wl, int hl, int* rowcnt) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int y = row + 2;
  if (y >= hl - 2) return;
  int cnt = 0;
  for (int x0 = 2; x0 < wl - 2; x0 += 32) {
    const int x = x0 + lane;
    float q, col;
    const bool v = (x < wl - 2) && cd_valid(ws, idl, img, x + y * wl, q, col);
    cnt += __popc(__ballot_sync(0xffffffffu, v));
  }
  if (lane == 0) rowcnt[row] = cnt;
}

// exclusive scan of the row counts by one block; total -> *total
__global__ void cd_scan_kernel(const int* __restrict__ rowcnt, int* __restrict__ rowoff, int nrows, int* total) {
  __shared__ int s[1024];
  const int tid = threadIdx.x;
  int carry = 0;
  for (int base = 0; base < nrows; base += 1024) {
    const int v = (base + tid < nrows) ? rowcnt[base + tid] : 0;
    s[tid] = v;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
      const int t = (tid >= d) ? s[tid - d] : 0;
      __syncthreads();
      s[tid] += t;
      __syncthreads();
    }
    if (base + tid < nrows) rowoff[base + tid] = carry + s[tid] - v;
    carry += s[1023];
    __syncthreads();
  }
  if (tid == 0) *total = carry;
}

__global__ void cd_write_kernel(const float* __restrict__ ws, const float* __restrict__ idl, const float4* __restrict__ img, int wl, int hl,
                                const int* __restrict__ rowoff, int cap, float* pc_u, float* pc_v, float* pc_id, float* pc_col) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int y = row + 2;
  if (y >= hl - 2) return;
  int off = rowoff[row];
  for (int x0 = 2; x0 < wl - 2; x0 += 32) {
    const int x = x0 + lane;
    float q = 0, col = 0;
    const bool v = (x < wl - 2) && cd_valid(ws, idl, img, x + y * wl, q, col);
    const unsigned m = __ballot_sync(0xffffffffu, v);
    if (v) {
      const int o = off + __popc(m & ((1u << lane) - 1u));
      if (o < cap) { pc_u[o] = (float)x; pc_v[o] = (float)y; pc_id[o] = q; pc_col[o] = col; }
    }
    off += __popc(m);
  }
}

static void cd_clear(const CDLevels& L, cudaStream_t s) {
  cudaMemsetAsync(L.idepth[0], 0, sizeof(float) * L.w[0] * L.h[0], s);
  cudaMemsetAsync(L.ws[0], 0, sizeof(float) * L.w[0] * L.h[0], s);
}

// everything after the level-0 splat: pooling, dilation, compaction
static int cd_reduce(const CDLevels& L, cudaStream_t s) {
  int k = 0;
  for (int l = 1; l < L.levels; l++) {
    dim3 grid((L.w[l] + 127) / 128, L.h[l]);
    cd_pool_kernel<<<grid, 128, 0, s>>>(L.idepth[l - 1], L.ws[l - 1], L.idepth[l], L.ws[l], L.w[l], L.h[l], L.w[l - 1]);
    k++;
  }
  for (int l = 0; l < L.levels; l++) {
    const int npx = L.w[l] * L.h[l];
    cd_dilate_kernel<<<(npx + 255) / 256, 256, 0, s>>>(L.ws[l], L.ws2[l], L.idepth[l], L.w[l], L.h[l], l < 2 ? 1 : 0);
    k++;
    const int nrows = L.h[l] - 4;
    if (nrows > 0) {
      cd_rowcount_kernel<<<(nrows + 7) / 8, 256, 0, s>>>(L.ws2[l], L.idepth[l], L.img[l], L.w[l], L.h[l], L.rowcnt);
      cd_scan_kernel<<<1, 1024, 0, s>>>(L.rowcnt, L.rowoff, nrows, L.totals + l);
      cd_write_kernel<<<(nrows + 7) / 8, 256, 0, s>>>(L.ws2[l], L.idepth[l], L.img[l], L.w[l], L.h[l], L.rowoff, L.cap, L.pc_u[l], L.pc_v[l], L.pc_id[l], L.pc_col[l]);
      k += 3;
    } else {
      cudaMemsetAsync(L.totals + l, 0, sizeof(int), s);
    }
  }
  return k;
}

void cd_launch(const CDLevels& L, int n_unique, const int* d_pix, const float* d_idw, const float* d_wsum, cudaStream_t s) {
  cd_clear(L, s);
  if (n_unique > 0) cd_scatter_kernel<<<(n_unique + 255) / 256, 256, 0, s>>>(n_unique, d_pix, d_idw, d_wsum, L.idepth[0], L.ws[0]);
  cd_reduce(L, s);
}

// one entry per window point: key = the level-0 pixel u + w0 * v of its IN residual into the reference frame (CoarseTracker.cpp:L148-153),
// npx0 for a point without one.  A projection outside the image is an error of the call: *bad = the lowest such point.
__global__ void cd_key_kernel(int npts, const uint8_t* __restrict__ st, const float* __restrict__ cu, const float* __restrict__ cv, int w0, int h0,
                              unsigned* __restrict__ key, int* __restrict__ ord, int* bad) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npts) return;
  unsigned k = (unsigned)(w0 * h0);
  if (st[p] == 0) {
    // int u = Ku + 0.5f truncates: 0 <= u < w0 exactly when -1 < Ku + 0.5f < w0 (NaN fails both tests, as the host's conversion does)
    const float x = cu[p] + 0.5f, y = cv[p] + 0.5f;
    if (x > -1.f && x < (float)w0 && y > -1.f && y < (float)h0) k = (unsigned)((int)x + w0 * (int)y);
    else atomicMin(bad, p);
  }
  key[p] = k;
  ord[p] = p;
}

// FullSystem::removeOutliers' reorder: point moves[2k] takes position moves[2k+1] of the fold order (a point without residuals, so its key is
// empty); the position it leaves becomes empty.  Sources and targets are distinct points, so the pairs are independent.
__global__ void cd_move_kernel(int n, const int* __restrict__ moves, unsigned empty, unsigned* key, int* ord) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int from = moves[2 * k], to = moves[2 * k + 1];
  key[to] = key[from];
  ord[to] = from;
  key[from] = empty;
}

// one thread per run of equal keys (the sort kept input order inside a run): the reference's idepth[0][i] += new_idepth * weight and
// weightSums[0][i] += weight over the points of pixel i, starting from the memset's +0 (so a -0 first term becomes +0 as there)
__global__ void cd_fold_kernel(int n, const unsigned* __restrict__ key, const int* __restrict__ ord, const float* __restrict__ cid,
                               const float* __restrict__ hdi, unsigned npx, float* idepth0, float* ws0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = key[i];
  if (k >= npx || (i > 0 && key[i - 1] == k)) return;
  float idw = 0.f, ws = 0.f;
  for (int j = i; j < n && key[j] == k; j++) {
    const int p = ord[j];
    const float weight = sqrtf((float)(1e-3 / ((double)hdi[p] + 1e-12)));   // CoarseTracker.cpp:L154, float HdiF promoted to double
    idw += cid[p] * weight;
    ws += weight;
  }
  idepth0[k] = idw;
  ws0[k] = ws;
}

size_t cd_sort_temp_bytes(int cap) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, cap, 0, 32);
  return bytes;
}

cudaError_t cd_launch_from_ba(const CDLevels& L, const CDFromBA& B, const CDSortScratch& S, cudaStream_t s, int* kernels) {
  const unsigned npx = (unsigned)(L.w[0] * L.h[0]);
  int end_bit = 1;
  while (end_bit < 32 && (npx >> end_bit) != 0) end_bit++;   // keys are <= npx
  int k = 0;
  cd_clear(L, s);
  cudaMemsetAsync(S.bad, 0x7f, sizeof(int), s);   // 0x7f7f7f7f: above any point index
  if (B.npts > 0) {
    const int g = (B.npts + 255) / 256;
    cd_key_kernel<<<g, 256, 0, s>>>(B.npts, B.st, B.cu, B.cv, L.w[0], L.h[0], S.key[0], S.ord[0], S.bad);
    k++;
    if (B.n_moves > 0) {
      cd_move_kernel<<<(B.n_moves + 255) / 256, 256, 0, s>>>(B.n_moves, B.moves, npx, S.key[0], S.ord[0]);
      k++;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t tb = S.temp_bytes;
    // LSD radix sort: stable, so the points of one pixel stay in fold order (array position)
    e = cub::DeviceRadixSort::SortPairs(S.temp, tb, S.key[0], S.key[1], S.ord[0], S.ord[1], B.npts, 0, end_bit, s);
    if (e != cudaSuccess) return e;
    cd_fold_kernel<<<g, 256, 0, s>>>(B.npts, S.key[1], S.ord[1], B.cid, B.hdi, npx, L.idepth[0], L.ws[0]);
    k++;
  }
  k += cd_reduce(L, s);
  *kernels = k;
  return cudaGetLastError();
}

}  // namespace dmv
