// dmv_ba_edit_window (include/dmvio_b200.h): one change of the window's membership — FullSystem::makeKeyFrame's makeIDX points — made on the
// window already on the device, bit-identical to a download and a re-upload through dmv_ba_set_window + dmv_ba_set_points +
// dmv_ba_set_residuals.  The caller names the new point order (point_src: a current point, or an entry of the last activation) and the new
// frames (frame_src), so the host keeps every index its read-backs use.  One copy-only kernel gathers the new point arrays and the new
// [target][point] input grids from the current ones and the activation staging into the spare buffers, which then swap with the handle's.
// The host mirrors (res_slot, host_of_point, h_st_in, h_en_in) are rebuilt from what the host already knows; only the carried residuals'
// states of a committed linearisation live on the device alone, and they come back compacted in the call's one synchronisation.
#include "ba_handle.h"
#include <algorithm>
#include <cstring>
#include <utility>
#include <vector>

using namespace dmv;

struct BAEditArgs {
  int npts, mp, nf, act_nf, new_res_target;
  int fsrc[MAXF];             // new frame -> current frame, or -1
  const int* src;             // [npts] point_src, then [npts] each carried point's first entry in the compacted read-back
  const float2* uv;           // current point arrays
  const float *idepth, *idepth_zero, *color, *weights, *priorF;   // idepth_zero NULL: aliased to idepth (and so in the new window)
  const uint8_t* st;          // the states the next linearisation would read (committed outputs, else the inputs)
  const float* en;
  const float* act;           // activation staging (d_act) and its layout
  ActLayout o;
  float2* uv_out;
  float *idepth_out, *idepth_zero_out, *color_out, *weights_out, *priorF_out;
  uint8_t* st_out;            // [MAXF][mp] new input grids, every slot written (as dmv_ba_set_residuals uploads them)
  float* en_out;
  uint8_t* cst;               // carried residuals' states and energies, compacted (NULL: not needed, the host mirrors hold them)
  float* cen;
};

// one thread per point slot of the new window
__global__ void __launch_bounds__(128) ba_edit_gather_kernel(const __grid_constant__ BAEditArgs A) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.mp) return;
  const size_t mp = A.mp;
  if (j >= A.npts) {
    for (int t = 0; t < MAXF; t++) { A.st_out[t * mp + j] = RES_NONE; A.en_out[t * mp + j] = 0.f; }
    return;
  }
  const int s = A.src[j];
  if (s >= 0) {   // carried point
    A.uv_out[j] = A.uv[s];
    const float id = A.idepth[s];
    A.idepth_out[j] = id;
    if (A.idepth_zero_out) A.idepth_zero_out[j] = A.idepth_zero[s];
#pragma unroll
    for (int k = 0; k < 8; k++) { A.color_out[8 * j + k] = A.color[8 * s + k]; A.weights_out[8 * j + k] = A.weights[8 * s + k]; }
    A.priorF_out[j] = A.priorF[s];
    int c = A.src[A.npts + j];
    for (int t = 0; t < MAXF; t++) {
      uint8_t st = RES_NONE;
      float en = 0.f;
      const int to = t < A.nf ? A.fsrc[t] : -1;
      if (t == A.new_res_target) {
        st = RES_IN;
      } else if (to >= 0) {
        const size_t q = (size_t)to * mp + s;
        st = A.st[q];
        if (st != RES_NONE) {
          en = A.en[q];
          if (A.cst) { A.cst[c] = st; A.cen[c] = en; c++; }
        }
      }
      A.st_out[t * mp + j] = st;
      A.en_out[t * mp + j] = en;
    }
  } else {        // entry k of the last activation
    const int k = -1 - s;
    const ActLayout& o = A.o;
    A.uv_out[j] = make_float2(A.act[o.u + k], A.act[o.v + k]);
    const float id = A.act[o.id + k];
    A.idepth_out[j] = id;
    if (A.idepth_zero_out) A.idepth_zero_out[j] = id;
#pragma unroll
    for (int c = 0; c < 8; c++) { A.color_out[8 * j + c] = A.act[o.col + 8 * k + c]; A.weights_out[8 * j + c] = A.act[o.wgt + 8 * k + c]; }
    A.priorF_out[j] = 0.f;
    const int* rs = reinterpret_cast<const int*>(A.act + o.rs) + (size_t)k * A.act_nf;
    for (int t = 0; t < MAXF; t++) {
      const int to = t < A.nf ? A.fsrc[t] : -1;
      A.st_out[t * mp + j] = (to >= 0 && rs[to] == 0) ? (uint8_t)RES_IN : (uint8_t)RES_NONE;
      A.en_out[t * mp + j] = 0.f;
    }
  }
}

extern "C" int dmv_ba_edit_window(dmv_ba* b, const dmv_ba_edit_args* a) {
  if (!b || !a || !a->frame_src || !a->point_src) return set_error(DMV_ERR_INVALID, "null argument");
  if (b->nranks > 1) return set_error(DMV_ERR_STATE, "sharded BA handle (%d ranks): its points are one rank's share; re-upload the window", b->nranks);
  if (b->nf < 2 || b->npts < 1 || !b->res_valid)
    return set_error(DMV_ERR_STATE, "dmv_ba_set_window + dmv_ba_set_points + dmv_ba_set_residuals first");
  const int nf0 = b->nf, np0 = b->npts, nf = a->nf, npts = a->npts, mp = b->mp, nrt = a->new_res_target;
  if (nf < 2 || nf > b->cfg.max_frames) return set_error(DMV_ERR_INVALID, "nf out of range");
  for (int f = 0; f < nf; f++) {
    const int s = a->slots ? a->slots[f] : f;
    if (s < 0 || s >= b->cfg.max_frames) return set_error(DMV_ERR_INVALID, "slot out of range");
  }
  int fnew[MAXF];   // current frame -> new frame, or -1 (leaves)
  for (int f = 0; f < MAXF; f++) fnew[f] = -1;
  for (int f = 0; f < nf; f++) {
    const int s = a->frame_src[f];
    if (s < -1 || s >= nf0) return set_error(DMV_ERR_INVALID, "frame_src[%d] = %d: expected -1 to %d", f, s, nf0 - 1);
    if (s >= 0 && fnew[s] >= 0) return set_error(DMV_ERR_INVALID, "frame_src[%d] and frame_src[%d] are both %d", fnew[s], f, s);
    if (s >= 0) fnew[s] = f;
  }
  if (npts < 1 || npts > b->cfg.max_points) return set_error(DMV_ERR_INVALID, "npts = %d: expected 1 to %d", npts, b->cfg.max_points);
  if (nrt < -1 || nrt >= nf) return set_error(DMV_ERR_INVALID, "new_res_target = %d: expected -1 to %d", nrt, nf - 1);
  const ActLayout o = act_layout(b->act_cap);
  const int act_n = b->act_n;
  const int32_t* act_host = act_n > 0 ? reinterpret_cast<const int32_t*>(b->h_act.get() + o.host) : nullptr;
  const int32_t* act_status = act_n > 0 ? reinterpret_cast<const int32_t*>(b->h_act.get() + o.st) : nullptr;
  const int32_t* act_rs = act_n > 0 ? reinterpret_cast<const int32_t*>(b->h_act.get() + o.rs) : nullptr;
  std::vector<int32_t> host(npts);
  std::vector<int> pnew(np0, -1), anew(std::max(act_n, 0), -1);
  for (int j = 0; j < npts; j++) {
    const int s = a->point_src[j];
    int h0;
    if (s >= 0) {
      if (s >= np0) return set_error(DMV_ERR_INVALID, "point_src[%d] = %d: the window has %d points", j, s, np0);
      if (pnew[s] >= 0) return set_error(DMV_ERR_INVALID, "point_src[%d] and point_src[%d] are both %d", pnew[s], j, s);
      pnew[s] = j;
      h0 = b->host_of_point[s];
    } else {
      const int k = -1 - s;
      if (act_n < 0) return set_error(DMV_ERR_INVALID, "point_src[%d] = %d: no activation ran on this window", j, s);
      if (k >= act_n) return set_error(DMV_ERR_INVALID, "point_src[%d] = %d: the last activation has %d entries", j, s, act_n);
      if (anew[k] >= 0) return set_error(DMV_ERR_INVALID, "point_src[%d] and point_src[%d] are both %d", anew[k], j, s);
      if (act_status[k] != 1) return set_error(DMV_ERR_INVALID, "point_src[%d] = %d: activation entry %d has status %d, not 1", j, s, k, act_status[k]);
      anew[k] = j;
      h0 = act_host[k];
    }
    host[j] = fnew[h0];
    if (host[j] < 0) return set_error(DMV_ERR_INVALID, "point %d: its host frame %d leaves the window", j, h0);
    if (j > 0 && host[j] < host[j - 1]) return set_error(DMV_ERR_INVALID, "points must be ordered by host frame (EnergyFunctional::allPoints order)");
  }
  const std::vector<uint8_t>& st0 = b->h_st_in;
  if (nrt >= 0)
    for (int j = 0; j < npts; j++) {
      const int s = a->point_src[j];
      if (s < 0) continue;
      if (host[j] == nrt) return set_error(DMV_ERR_INVALID, "new_res_target %d is the host frame of point %d", nrt, j);
      if (a->frame_src[nrt] >= 0 && st0[(size_t)a->frame_src[nrt] * mp + s] != RES_NONE)
        return set_error(DMV_ERR_INVALID, "new_res_target %d: point %d already has a residual into it", nrt, j);
    }
  BAShape shape;
  dmv_ba_window_shape(b, npts, host.data(), &shape);
  if (shape.nchunks > b->max_chunks) return set_error(DMV_ERR_INVALID, "too many chunks");

  // the new residual list and input mirrors: carried (current order), new_res_target (point order), activated (point order, target ascending)
  const size_t ns = (size_t)MAXF * mp;
  const bool committed = b->have_committed;
  std::vector<int> slot;
  slot.reserve(b->nres + npts * (nf - 1));
  std::vector<uint8_t> st1(ns, (uint8_t)RES_NONE);
  std::vector<float> en1(ns, 0.f);
  for (int i = 0; i < b->nres; i++) {
    const int q = b->res_slot[i], p = pnew[q % mp], t = fnew[q / mp];
    if (p < 0 || t < 0) continue;
    const int s = t * mp + p;
    slot.push_back(s);
    st1[s] = st0[q];
    en1[s] = b->h_en_in[q];
  }
  if (nrt >= 0)
    for (int j = 0; j < npts; j++)
      if (a->point_src[j] >= 0) { slot.push_back(nrt * mp + j); st1[(size_t)nrt * mp + j] = RES_IN; }
  for (int j = 0; j < npts; j++) {
    const int k = -1 - a->point_src[j];
    if (k < 0) continue;
    for (int t = 0; t < nf; t++)
      if (a->frame_src[t] >= 0 && act_rs[(size_t)k * nf0 + a->frame_src[t]] == 0) { slot.push_back(t * mp + j); st1[(size_t)t * mp + j] = RES_IN; }
  }
  // each carried point's first entry in the compacted read-back: its carried residuals, target ascending, points in new order
  std::vector<int32_t> first(npts, 0);
  int ncarry = 0;
  for (int j = 0; j < npts; j++) {
    first[j] = ncarry;
    const int s = a->point_src[j];
    if (s < 0) continue;
    for (int t = 0; t < nf; t++)
      if (t != nrt && a->frame_src[t] >= 0 && st0[(size_t)a->frame_src[t] * mp + s] != RES_NONE) ncarry++;
  }

  // everything checked: allocate, upload, gather, read back
  CK(cudaSetDevice(b->device));
  if (!b->e_src) {   // the last of the group: set only once all of it is
    CK(b->e_uv.alloc(mp));
    CK(b->e_idepth_zero.alloc(mp));
    CK(b->e_color.alloc((size_t)mp * 8));
    CK(b->e_weights.alloc((size_t)mp * 8));
    CK(b->e_priorF.alloc(mp));
    CK(b->e_st_in.alloc(ns));
    CK(b->e_en_in.alloc(ns));
    CK(b->e_cst.alloc(ns));
    CK(b->e_cen.alloc(ns));
    CK(b->e_src.alloc((size_t)2 * mp));
  }
  int32_t* h_src = reinterpret_cast<int32_t*>(b->h_scratch.get());   // [npts] point_src | [npts] first | carried energies | carried states
  float* h_cen = b->h_scratch + 2 * (size_t)npts;
  uint8_t* h_cst = reinterpret_cast<uint8_t*>(h_cen + ncarry);
  std::memcpy(h_src, a->point_src, sizeof(int32_t) * npts);
  std::memcpy(h_src + npts, first.data(), sizeof(int32_t) * npts);
  CK(cudaMemcpyAsync(b->e_src, h_src, sizeof(int32_t) * 2 * npts, cudaMemcpyHostToDevice, b->stream));
  BAEditArgs A;
  std::memset(&A, 0, sizeof(A));
  A.npts = npts; A.mp = mp; A.nf = nf; A.act_nf = nf0; A.new_res_target = nrt;
  for (int f = 0; f < MAXF; f++) A.fsrc[f] = f < nf ? a->frame_src[f] : -1;
  A.src = b->e_src;
  A.uv = b->d_uv; A.idepth = b->d_idepth[b->id_cur]; A.idepth_zero = b->zero_alias ? nullptr : b->d_idepth_zero.get();
  A.color = b->d_color; A.weights = b->d_weights; A.priorF = b->d_priorF;
  A.st = committed ? b->d_st_new[1 - b->tent] : b->d_st_in;
  A.en = committed ? b->d_en_new[1 - b->tent] : b->d_en_in;
  A.act = b->d_act; A.o = o;
  A.uv_out = b->e_uv; A.idepth_out = b->d_idepth[1 - b->id_cur]; A.idepth_zero_out = b->zero_alias ? nullptr : b->e_idepth_zero.get();
  A.color_out = b->e_color; A.weights_out = b->e_weights; A.priorF_out = b->e_priorF;
  A.st_out = b->e_st_in; A.en_out = b->e_en_in;
  A.cst = committed ? b->e_cst.get() : nullptr; A.cen = b->e_cen;
  ba_edit_gather_kernel<<<(mp + 127) / 128, 128, 0, b->stream>>>(A);
  b->launches++;
  CK(cudaGetLastError());
  for (int k = 0; k < 2; k++) CK(cudaMemsetAsync(b->d_st_new[k], 0xff, ns, b->stream));
  if (committed && ncarry > 0) {
    CK(cudaMemcpyAsync(h_cen, b->e_cen, sizeof(float) * ncarry, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(h_cst, b->e_cst, ncarry, cudaMemcpyDeviceToHost, b->stream));
  }
  // the new window: set_window's descriptor (which also drops adjoints, state, linearisations and the activation), then the shape
  const int id_new = 1 - b->id_cur;
  int rc = dmv_ba_set_window(b, nf, a->slots);
  if (rc != DMV_OK) return rc;
  b->npts = npts;
  b->host_of_point.assign(host.begin(), host.end());
  rc = dmv_ba_take_shape(b, &shape);
  if (rc != DMV_OK) return rc;
  std::swap(b->d_uv, b->e_uv);
  if (!b->zero_alias) std::swap(b->d_idepth_zero, b->e_idepth_zero);
  std::swap(b->d_color, b->e_color);
  std::swap(b->d_weights, b->e_weights);
  std::swap(b->d_priorF, b->e_priorF);
  std::swap(b->d_st_in, b->e_st_in);
  std::swap(b->d_en_in, b->e_en_in);
  b->id_cur = b->id_bak = id_new;
  CK(cudaStreamSynchronize(b->stream));
  if (committed)
    for (int j = 0, c = 0; j < npts; j++) {
      const int s = a->point_src[j];
      if (s < 0) continue;
      for (int t = 0; t < nf; t++)
        if (t != nrt && a->frame_src[t] >= 0 && st0[(size_t)a->frame_src[t] * mp + s] != RES_NONE) {
          st1[(size_t)t * mp + j] = h_cst[c];
          en1[(size_t)t * mp + j] = h_cen[c];
          c++;
        }
    }
  b->h_st_in.swap(st1);
  b->h_en_in.swap(en1);
  b->res_slot.swap(slot);
  b->nres = (int)b->res_slot.size();
  b->st_in_clean = true;
  for (int i = 0; i < b->nres; i++)
    if (b->h_st_in[b->res_slot[i]] != RES_IN || b->h_en_in[b->res_slot[i]] != 0.f) { b->st_in_clean = false; break; }
  b->res_valid = true;
  b->hdi_solve_n = 0;
  b->en_newest_valid = false;
  return DMV_OK;
}
