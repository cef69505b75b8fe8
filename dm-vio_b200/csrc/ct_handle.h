// Internal layout of the coarse-tracker handle, shared by ct_kernels.cu (tracking, uploads, create/destroy) and the files of the features
// built on its resident frame: ct_ingest.cu, ct_depth.cu, ip_trace.cu and ps_select.cu.
#pragma once
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include <algorithm>
#include <memory>

namespace dmv {
struct CTMaps;      // TMA descriptors of the level planes (ct_kernels.cu)
struct CDScratch;   // makeCoarseDepthL0's working planes and sort scratch (ct_depth.cu), allocated on first use
struct PSScratch;   // pixel selection's scratch (ps_select.cu), allocated on first use
// deletes the handle's share of a feature: each operator() is defined in the feature's file, where the type is complete
struct CTPartDelete {
  void operator()(CTMaps* p) const;
  void operator()(CDScratch* p) const;
  void operator()(PSScratch* p) const;
};
template <typename T> using CTPart = std::unique_ptr<T, CTPartDelete>;
}  // namespace dmv

struct dmv_ct {
  dmv_ct_config cfg;
  int device = 0;
  dmv::Stream stream;
  dmv::Event ev[2];
  dmv::Event ev_order;              // orders a dmv_ct_track_many / _tries_many / dmv_ct_trace_many launch on another member's stream behind this handle's queued work
  bool staging_busy = false;  // an asynchronous upload from h_scratch may be in flight
  bool timing = false;  // CUDA-event timing of every evaluation (dmv_ct_set_timing); off by default: two event records per launch
  int w[DMV_MAX_PYR_LEVELS], h[DMV_MAX_PYR_LEVELS];
  float fx[DMV_MAX_PYR_LEVELS], fy[DMV_MAX_PYR_LEVELS], cx[DMV_MAX_PYR_LEVELS], cy[DMV_MAX_PYR_LEVELS];
  bool haveK[DMV_MAX_PYR_LEVELS];
  dmv::DevBuf<float4> d_img[DMV_MAX_PYR_LEVELS];
  dmv::DevBuf<float> d_gray[DMV_MAX_PYR_LEVELS];
  dmv::DevBuf<float> d_stage;
  dmv::DevBuf<float> d_u[DMV_MAX_PYR_LEVELS], d_v[DMV_MAX_PYR_LEVELS], d_id[DMV_MAX_PYR_LEVELS], d_col[DMV_MAX_PYR_LEVELS];
  int n[DMV_MAX_PYR_LEVELS];
  dmv::DevBuf<double> d_partial;
  dmv::DevBuf<unsigned int> d_ticket;
  dmv::PinnedBuf<double> h_out;
  dmv::PinnedBuf<float> h_scratch;
  dmv::CTPart<dmv::CDScratch> cd;   // dmv_ct_make_coarse_depth / dmv_ct_set_ref_from_ba
  dmv::DevBuf<float> d_ip;   // per-point staging of dmv_ct_make_coarse_depth, dmv_ct_init_points and dmv_ct_trace_points (ct_reserve_ip)
  dmv::PinnedBuf<float> h_ip;
  int ip_cap = 0;            // points the staging layout holds (0 while d_ip / h_ip may be short of it)
  float huber = 9.f;
  int cluster_size = 0;        // CTAs of ct_track_cluster_kernel's cluster (0 = not probed yet, -1 = none schedulable: dmv_ct_track fails)
  dmv::CTPart<dmv::CTMaps> maps;  // TMA descriptors of the level planes (host copy; passed as a kernel parameter)
  int staged[DMV_MAX_PYR_LEVELS] = {0};   // levels whose map ct_make_tensor_maps encoded: the only ones the cluster kernel stages
  dmv::PinnedBuf<dmv_ct_tries_result> h_tries;   // dmv_ct_track_tries's pinned result, allocated on first use
  dmv::PinnedBuf<double> h_pose;   // dmv_ct_track_tries_many's try table (DMV_CT_MAX_TRIES x 12: R row-major, t), allocated on first use
  long long launches = 0;
  float last_ms[4] = {0, 0, 0, 0};
  // raw-frame ingest (dmv_ct_set_undistort / dmv_ct_upload_raw_image)
  bool have_undistort = false;
  int wOrg = 0, hOrg = 0, nG = 0, pmode = 0;
  dmv::DevBuf<float2> d_remap;                 // (remapX, remapY) per level-0 pixel; empty = passthrough
  dmv::DevBuf<float> d_G, d_vigInv;            // response map; vignetteMapInv (wOrg*hOrg, photometric mode 2)
  dmv::DevBuf<uint8_t> d_raw;
  dmv::CTPart<dmv::PSScratch> ps;   // dmv_ct_make_new_traces
};

namespace dmv {

// the pyramid of the frame whose level-0 intensities are in d_gray[0] (first_level 0), or whose level-0 plane d_img[0] is already in place
// (first_level 1: dmv_ct_set_ref_from_ba copies it from the BA handle); counts its launches
int ct_build_pyramid(dmv_ct* c, int first_level);

// a previous asynchronous upload may still read the pinned staging buffer h_scratch
inline cudaError_t ct_wait_staging(dmv_ct* c) {
  if (!c->staging_busy) return cudaSuccess;
  const cudaError_t e = cudaStreamSynchronize(c->stream);
  if (e == cudaSuccess) c->staging_busy = false;
  return e;
}

// the error a check of member i of a call over several handles just set, prefixed with the member's index
inline int ct_member_error(int rc, int i) {
  char msg[512];
  snprintf(msg, sizeof(msg), "%s", dmv_last_error());
  return set_error(rc, "handles[%d]: %s", i, msg);
}

// the member list of a call over several handles: 1..max handles, none NULL, none twice, all on one device
inline int ct_check_members(dmv_ct* const* handles, int n, int max) {
  if (n < 1 || n > max) return set_error(DMV_ERR_INVALID, "n = %d: expected 1 to %d handles", n, max);
  for (int i = 0; i < n; i++) {
    if (!handles[i]) return set_error(DMV_ERR_INVALID, "handles[%d] is NULL", i);
    for (int j = 0; j < i; j++)
      if (handles[j] == handles[i]) return set_error(DMV_ERR_INVALID, "handles[%d] and handles[%d] are the same handle", j, i);
    if (handles[i]->device != handles[0]->device)
      return set_error(DMV_ERR_INVALID, "handles[%d] is on device %d, handles[0] on device %d: one launch runs on one device", i, handles[i]->device,
                       handles[0]->device);
  }
  return DMV_OK;
}

// work enqueued on stream s from now on runs behind the work queued on member c's stream so far: a launch over several handles goes on one
// member's stream, behind every other member's uploads (dmv_ct_upload_new_image does not synchronise)
inline cudaError_t ct_order_behind(dmv_ct* c, cudaStream_t s) {
  const cudaError_t e = cudaEventRecord(c->ev_order, c->stream);
  return e == cudaSuccess ? cudaStreamWaitEvent(s, c->ev_order, 0) : e;
}

// d_ip / h_ip hold at least n points: 31 words per point (dmv_ct_trace_points' layout, the widest) and 14 words of tables for each of up
// to 64 host frames
inline cudaError_t ct_reserve_ip(dmv_ct* c, int n) {
  if (n <= c->ip_cap) return cudaSuccess;
  c->ip_cap = 0;
  const int cap = std::max(n, 2048);
  const size_t words = (size_t)31 * cap + 14 * 64;
  cudaError_t e = c->d_ip.reserve(words);
  if (e == cudaSuccess) e = c->h_ip.reserve(words);
  if (e == cudaSuccess) c->ip_cap = cap;
  return e;
}

}  // namespace dmv
