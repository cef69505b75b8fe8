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
#include "ct_handle.h"
#include "ct_depth.h"
#include <cub/device/device_radix_sort.cuh>
#include <cstring>
#include <unordered_map>

namespace dmv {

// the handle's share (dmv_ct::cd), allocated on first use
struct CDScratch {
  DevBuf<float> idepth[DMV_MAX_PYR_LEVELS], ws[DMV_MAX_PYR_LEVELS], ws2[DMV_MAX_PYR_LEVELS];
  DevBuf<int> rowcnt, rowoff;   // scratch rows of the compaction
  PinnedBuf<int> totals;        // device-visible: pc_n of every level, then [DMV_MAX_PYR_LEVELS] = bad
  // the device fold of dmv_ct_set_ref_from_ba, for up to sort_cap points: radix-sort keys / ordinals (double-buffered) and CUB's temporary
  // storage, the moves, and the event that orders the tracker's stream behind the BA's
  DevBuf<unsigned> key[2];
  DevBuf<int> ord[2];
  DevBuf<uint8_t> temp;
  size_t temp_bytes = 0;
  DevBuf<int> bad;          // lowest point index whose projection leaves the image (>= npts: none)
  DevBuf<int> moves;        // device copy of CDFromBA::moves_host (2 * sort_cap ints)
  PinnedBuf<int> h_moves;   // its pinned staging
  int sort_cap = 0;
  Event ev_ba;
};

void CTPartDelete::operator()(CDScratch* p) const { delete p; }

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

static void cd_clear(const dmv_ct* c) {
  cudaMemsetAsync(c->cd->idepth[0], 0, sizeof(float) * c->w[0] * c->h[0], c->stream);
  cudaMemsetAsync(c->cd->ws[0], 0, sizeof(float) * c->w[0] * c->h[0], c->stream);
}

// everything after the level-0 splat: pooling, dilation, compaction into the handle's pc_* lists
static int cd_reduce(dmv_ct* c) {
  const CDScratch& S = *c->cd;
  const cudaStream_t s = c->stream;
  int k = 0;
  for (int l = 1; l < c->cfg.levels; l++) {
    dim3 grid((c->w[l] + 127) / 128, c->h[l]);
    cd_pool_kernel<<<grid, 128, 0, s>>>(S.idepth[l - 1], S.ws[l - 1], S.idepth[l], S.ws[l], c->w[l], c->h[l], c->w[l - 1]);
    k++;
  }
  for (int l = 0; l < c->cfg.levels; l++) {
    const int npx = c->w[l] * c->h[l];
    cd_dilate_kernel<<<(npx + 255) / 256, 256, 0, s>>>(S.ws[l], S.ws2[l], S.idepth[l], c->w[l], c->h[l], l < 2 ? 1 : 0);
    k++;
    const int nrows = c->h[l] - 4;
    if (nrows > 0) {
      cd_rowcount_kernel<<<(nrows + 7) / 8, 256, 0, s>>>(S.ws2[l], S.idepth[l], c->d_img[l], c->w[l], c->h[l], S.rowcnt);
      cd_scan_kernel<<<1, 1024, 0, s>>>(S.rowcnt, S.rowoff, nrows, S.totals + l);
      cd_write_kernel<<<(nrows + 7) / 8, 256, 0, s>>>(S.ws2[l], S.idepth[l], c->d_img[l], c->w[l], c->h[l], S.rowoff, c->cfg.max_points, c->d_u[l],
                                                      c->d_v[l], c->d_id[l], c->d_col[l]);
      k += 3;
    } else {
      cudaMemsetAsync(S.totals + l, 0, sizeof(int), s);
    }
  }
  return k;
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

static size_t cd_sort_temp_bytes(int cap) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, cap, 0, 32);
  return bytes;
}

// the same lists as dmv_ct_make_coarse_depth fed with the host fold of the IN residuals, built without leaving the device.  *kernels = the
// kernels it launches itself (the radix sort's own launches are not counted); returns the first error of the sort or a launch.
static cudaError_t cd_launch_from_ba(dmv_ct* c, const CDFromBA& B, int* kernels) {
  const CDScratch& S = *c->cd;
  const cudaStream_t s = c->stream;
  const unsigned npx = (unsigned)(c->w[0] * c->h[0]);
  int end_bit = 1;
  while (end_bit < 32 && (npx >> end_bit) != 0) end_bit++;   // keys are <= npx
  int k = 0;
  cd_clear(c);
  cudaMemsetAsync(S.bad, 0x7f, sizeof(int), s);   // 0x7f7f7f7f: above any point index
  if (B.npts > 0) {
    const int g = (B.npts + 255) / 256;
    cd_key_kernel<<<g, 256, 0, s>>>(B.npts, B.st, B.cu, B.cv, c->w[0], c->h[0], S.key[0], S.ord[0], S.bad);
    k++;
    if (B.n_moves > 0) {
      cd_move_kernel<<<(B.n_moves + 255) / 256, 256, 0, s>>>(B.n_moves, B.moves, npx, S.key[0], S.ord[0]);
      k++;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t tb = S.temp_bytes;
    // LSD radix sort: stable, so the points of one pixel stay in fold order (array position)
    e = cub::DeviceRadixSort::SortPairs(S.temp, tb, S.key[0].get(), S.key[1].get(), S.ord[0].get(), S.ord[1].get(), B.npts, 0, end_bit, s);
    if (e != cudaSuccess) return e;
    cd_fold_kernel<<<g, 256, 0, s>>>(B.npts, S.key[1], S.ord[1], B.cid, B.hdi, npx, S.idepth[0], S.ws[0]);
    k++;
  }
  k += cd_reduce(c);
  *kernels = k;
  return cudaGetLastError();
}

}  // namespace dmv

using namespace dmv;

// working planes of the device makeCoarseDepthL0, allocated on first use; totals, the last of them, is set only once all of them are
static int ct_cd_allocate(dmv_ct* c) {
  if (!c->cd) c->cd.reset(new CDScratch());
  CDScratch& S = *c->cd;
  if (S.totals) return DMV_OK;
  for (int l = 0; l < c->cfg.levels; l++) {
    const size_t npx = (size_t)c->w[l] * c->h[l];
    CK(S.idepth[l].alloc(npx));
    CK(S.ws[l].alloc(npx));
    CK(S.ws2[l].alloc(npx));
  }
  CK(S.rowcnt.alloc(c->h[0]));
  CK(S.rowoff.alloc(c->h[0]));
  CK(S.totals.alloc(DMV_MAX_PYR_LEVELS + 1));
  return DMV_OK;
}
// pc_n of every level from the compaction's totals (after the stream synchronisation); a level over capacity is an error
static int ct_cd_take_counts(dmv_ct* c, int32_t* pc_n_out) {
  const int* totals = c->cd->totals;
  for (int l = 0; l < c->cfg.levels; l++) {
    if (totals[l] > c->cfg.max_points) return set_error(DMV_ERR_INVALID, "level %d: %d reference points exceed max_points %d", l, totals[l], c->cfg.max_points);
    c->n[l] = totals[l];
    if (pc_n_out) pc_n_out[l] = c->n[l];
  }
  return DMV_OK;
}

// CoarseTracker::setCoarseTrackingRef -> makeCoarseDepthL0 (CoarseTracker.cpp:L138-295) on the device; the reference frame is
// the one resident in the handle (last dmv_ct_upload_new_image / dmv_ct_upload_new of every level)
int dmv_ct_make_coarse_depth(dmv_ct* c, int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, int32_t* pc_n_out) {
  if (!c || n < 0 || (n > 0 && (!Ku || !Kv || !new_idepth || !HdiF))) return set_error(DMV_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  const int L = c->cfg.levels, w0 = c->w[0], h0 = c->h[0];
  int rc = ct_cd_allocate(c);
  if (rc != DMV_OK) return rc;
  // ---- the splat's only order-dependent part on the host: points hitting the same pixel are folded in input order (L144-160)
  CK(ct_reserve_ip(c, n));
  CK(ct_wait_staging(c));
  const size_t cap = c->ip_cap;
  int* h_pix = reinterpret_cast<int*>(c->h_ip.get());
  float* h_idw = c->h_ip + cap;
  float* h_ws = c->h_ip + 2 * cap;
  int nu = 0;
  {
    std::unordered_map<int, int> slot;
    slot.reserve((size_t)n * 2);
    for (int i = 0; i < n; i++) {
      const int u = Ku[i] + 0.5f, v = Kv[i] + 0.5f;
      if (u < 0 || v < 0 || u >= w0 || v >= h0) return set_error(DMV_ERR_INVALID, "residual %d projects to (%d,%d) outside the image", i, u, v);
      const float weight = sqrtf(1e-3 / (HdiF[i] + 1e-12));
      const int pix = u + w0 * v;
      auto it = slot.find(pix);
      if (it == slot.end()) { slot.emplace(pix, nu); h_pix[nu] = pix; h_idw[nu] = 0.f + new_idepth[i] * weight; h_ws[nu] = 0.f + weight; nu++; }
      else { h_idw[it->second] += new_idepth[i] * weight; h_ws[it->second] += weight; }
    }
  }
  CK(cudaMemcpyAsync(c->d_ip, c->h_ip, sizeof(float) * 3 * cap, cudaMemcpyHostToDevice, c->stream));
  cd_clear(c);
  if (nu > 0) cd_scatter_kernel<<<(nu + 255) / 256, 256, 0, c->stream>>>(nu, reinterpret_cast<const int*>(c->d_ip.get()), c->d_ip + cap, c->d_ip + 2 * cap, c->cd->idepth[0], c->cd->ws[0]);
  cd_reduce(c);
  c->launches += 2 + 4 * L;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return ct_cd_take_counts(c, pc_n_out);
}

// CoarseTracker::setCoarseTrackingRef fed straight from a BA handle on the same device (cd_launch_from_ba).  The points' IN
// residuals into the window's newest frame are folded on the device; the frame's level-0 plane is copied from the BA slot and the coarser levels
// are built as dmv_ct_upload_new_image builds them.  Ordered behind the BA stream by an event; one synchronisation at the end (pc_n).
extern "C" __attribute__((visibility("hidden"))) int dmv_ba_ref_source(dmv_ba* b, CDFromBA* out);
int dmv_ct_set_ref_from_ba(dmv_ct* c, dmv_ba* ba, int32_t* pc_n_out) {
  if (!c || !ba) return set_error(DMV_ERR_INVALID, "null argument");
  CDFromBA B;
  int rc = dmv_ba_ref_source(ba, &B);
  if (rc != DMV_OK) return rc;
  if (B.device != c->device) return set_error(DMV_ERR_INVALID, "the BA handle lives on device %d, the tracker handle on %d", B.device, c->device);
  if (B.w != c->w[0] || B.h != c->h[0]) return set_error(DMV_ERR_INVALID, "image size mismatch (BA %dx%d vs tracker %dx%d)", B.w, B.h, c->w[0], c->h[0]);
  CK(cudaSetDevice(c->device));
  if ((rc = ct_cd_allocate(c)) != DMV_OK) return rc;
  CDScratch& S = *c->cd;
  if (!S.ev_ba) CK(cudaEventCreateWithFlags(S.ev_ba.put(), cudaEventDisableTiming));
  if (B.npts > S.sort_cap) {
    CK(cudaStreamSynchronize(c->stream));   // kernels in flight may still use the old scratch
    S.sort_cap = 0;
    const int cap = std::max(B.npts, 2048);
    for (int k = 0; k < 2; k++) { CK(S.key[k].reserve(cap)); CK(S.ord[k].reserve(cap)); }
    CK(S.moves.reserve((size_t)2 * cap));
    CK(S.h_moves.reserve((size_t)2 * cap));
    S.temp_bytes = cd_sort_temp_bytes(cap);
    CK(S.temp.reserve(std::max<size_t>(S.temp_bytes, 16)));
    CK(S.bad.reserve(1));
    S.sort_cap = cap;
  }
  CK(cudaEventRecord(S.ev_ba, B.stream));         // the BA's last linearisation / accumulate / frame upload
  CK(cudaStreamWaitEvent(c->stream, S.ev_ba, 0));
  CK(cudaMemcpyAsync(c->d_img[0], B.img, sizeof(float4) * (size_t)c->w[0] * c->h[0], cudaMemcpyDeviceToDevice, c->stream));
  if ((rc = ct_build_pyramid(c, 1)) != DMV_OK) return rc;
  if (B.n_moves > 0) {   // the previous call ended in a synchronisation: the pinned staging is free
    std::memcpy(S.h_moves, B.moves_host, sizeof(int) * 2 * (size_t)B.n_moves);
    CK(cudaMemcpyAsync(S.moves, S.h_moves, sizeof(int) * 2 * (size_t)B.n_moves, cudaMemcpyHostToDevice, c->stream));
    B.moves = S.moves;
  }
  int kernels = 0;
  CK(cd_launch_from_ba(c, B, &kernels));
  c->launches += kernels;   // the pyramid counted itself; the radix sort's own launches are not counted
  CK(cudaMemcpyAsync(S.totals + DMV_MAX_PYR_LEVELS, S.bad, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  const int bad = S.totals[DMV_MAX_PYR_LEVELS];
  if (bad < B.npts) {  // the lists were rebuilt from an inconsistent window: leave no reference to track against
    for (int l = 0; l < c->cfg.levels; l++) c->n[l] = 0;
    return set_error(DMV_ERR_INVALID, "point %d: its IN residual into the newest frame projects outside the image", bad);
  }
  return ct_cd_take_counts(c, pc_n_out);
}

// pc_u / pc_v / pc_idepth / pc_color of a level as they sit on the device (tests; any pointer may be NULL); returns pc_n[level] in *n
int dmv_ct_get_ref(dmv_ct* c, int l, int* n, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color) {
  if (!c || !n || l < 0 || l >= c->cfg.levels) return set_error(DMV_ERR_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  *n = c->n[l];
  const size_t bytes = sizeof(float) * c->n[l];
  if (pc_u) CK(cudaMemcpy(pc_u, c->d_u[l], bytes, cudaMemcpyDeviceToHost));
  if (pc_v) CK(cudaMemcpy(pc_v, c->d_v[l], bytes, cudaMemcpyDeviceToHost));
  if (pc_idepth) CK(cudaMemcpy(pc_idepth, c->d_id[l], bytes, cudaMemcpyDeviceToHost));
  if (pc_color) CK(cudaMemcpy(pc_color, c->d_col[l], bytes, cudaMemcpyDeviceToHost));
  return DMV_OK;
}
