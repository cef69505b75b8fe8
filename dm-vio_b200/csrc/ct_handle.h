// Internal layout of the coarse-tracker handle, shared by ct_kernels.cu (tracking, uploads, create/destroy) and the files of the features
// built on its resident frame: ct_ingest.cu, ct_depth.cu, ip_trace.cu and ps_select.cu.
#pragma once
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include <algorithm>

namespace dmv {
struct CTMaps;      // TMA descriptors of the level planes (ct_kernels.cu)
struct CDScratch;   // makeCoarseDepthL0's working planes and sort scratch (ct_depth.cu), allocated on first use
struct PSScratch;   // pixel selection's scratch (ps_select.cu), allocated on first use
void cd_free(CDScratch* s);
void ps_free(PSScratch* s);
}  // namespace dmv

struct dmv_ct {
  dmv_ct_config cfg;
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  cudaEvent_t ev_order = nullptr;   // orders a dmv_ct_track_many / dmv_ct_trace_many launch on another member's stream behind this handle's queued work
  bool staging_busy = false;  // an asynchronous upload from h_scratch may be in flight
  bool timing = false;  // CUDA-event timing of every evaluation (dmv_ct_set_timing); off by default: two event records per launch
  int w[DMV_MAX_PYR_LEVELS], h[DMV_MAX_PYR_LEVELS];
  float fx[DMV_MAX_PYR_LEVELS], fy[DMV_MAX_PYR_LEVELS], cx[DMV_MAX_PYR_LEVELS], cy[DMV_MAX_PYR_LEVELS];
  bool haveK[DMV_MAX_PYR_LEVELS];
  float4* d_img[DMV_MAX_PYR_LEVELS] = {nullptr};
  float* d_gray[DMV_MAX_PYR_LEVELS] = {nullptr};
  float* d_stage = nullptr;
  float *d_u[DMV_MAX_PYR_LEVELS] = {nullptr}, *d_v[DMV_MAX_PYR_LEVELS] = {nullptr}, *d_id[DMV_MAX_PYR_LEVELS] = {nullptr},
        *d_col[DMV_MAX_PYR_LEVELS] = {nullptr};
  int n[DMV_MAX_PYR_LEVELS];
  double* d_partial = nullptr;
  unsigned int* d_ticket = nullptr;
  double* d_out = nullptr;
  double* h_out = nullptr;
  float* h_scratch = nullptr;
  dmv::CDScratch* cd = nullptr;   // dmv_ct_make_coarse_depth / dmv_ct_set_ref_from_ba
  float* d_ip = nullptr;   // per-point staging of dmv_ct_make_coarse_depth, dmv_ct_init_points and dmv_ct_trace_points (ct_reserve_ip)
  float* h_ip = nullptr;
  int ip_cap = 0;
  float huber = 9.f;
  int cluster_size = 0;        // CTAs of ct_track_cluster_kernel's cluster (0 = not probed yet, -1 = none schedulable: dmv_ct_track fails)
  dmv::CTMaps* maps = nullptr; // TMA descriptors of the level planes (host copy; passed as a kernel parameter)
  int staged[DMV_MAX_PYR_LEVELS] = {0};   // levels whose map ct_make_tensor_maps encoded: the only ones the cluster kernel stages
  dmv_ct_tries_result* h_tries = nullptr;   // dmv_ct_track_tries's pinned result, allocated on first use
  long long launches = 0;
  float last_ms[4] = {0, 0, 0, 0};
  size_t scratch_bytes = 0;    // capacity of h_scratch
  // raw-frame ingest (dmv_ct_set_undistort / dmv_ct_upload_raw_image)
  bool have_undistort = false;
  int wOrg = 0, hOrg = 0, nG = 0, pmode = 0;
  float2* d_remap = nullptr;                   // (remapX, remapY) per level-0 pixel; nullptr = passthrough
  float *d_G = nullptr, *d_vigInv = nullptr;   // response map; vignetteMapInv (wOrg*hOrg, photometric mode 2)
  void* d_raw = nullptr;
  dmv::PSScratch* ps = nullptr;   // dmv_ct_make_new_traces
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

// d_ip / h_ip hold at least n points: 31 words per point (dmv_ct_trace_points' layout, the widest) and 14 words of tables for each of up
// to 64 host frames
inline cudaError_t ct_reserve_ip(dmv_ct* c, int n) {
  if (n <= c->ip_cap) return cudaSuccess;
  cudaFree(c->d_ip); cudaFreeHost(c->h_ip);
  c->d_ip = nullptr; c->h_ip = nullptr; c->ip_cap = 0;
  const int cap = std::max(n, 2048);
  const size_t words = (size_t)31 * cap + 14 * 64;
  cudaError_t e = cudaMalloc(&c->d_ip, sizeof(float) * words);
  if (e == cudaSuccess) e = cudaMallocHost(&c->h_ip, sizeof(float) * words);
  if (e == cudaSuccess) c->ip_cap = cap;
  return e;
}

}  // namespace dmv
