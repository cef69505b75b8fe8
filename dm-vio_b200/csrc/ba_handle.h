// Internal layout of the BA handle (shared by ba_api.cu, the entry points beside their kernels in ip_trace.cu and ip_select.cu, and the
// measurement-only entry points in ba_bench.cu).
#pragma once
#include "../../include/dmvio_b200.h"
#include "ba_device.cuh"
#include "common_host.h"
#include <cstdint>
#include <vector>

namespace dmv {
cudaError_t launch_fused_kernel(BAWinDev& W, const BAIter& it, bool marg, cudaStream_t s, unsigned* bar_count);
cudaError_t launch_fused_kernel_clocked(BAWinDev& W, const BAIter& it, cudaStream_t s, unsigned* bar_count, unsigned long long* clk, int* grid);
cudaError_t launch_fused_batch_kernel(int P, const BAWinDev* gW, const BAIter* gIt, BABatchHdr& hdr, int max_nf, cudaStream_t s, unsigned* bar_count);
void launch_resub_kernel(const BAWinDev& W, const BAIter& it, int apply, double* sums, cudaStream_t s);
void launch_l2_flush(float4* buf, size_t n, cudaStream_t s);
}  // namespace dmv

struct HostUpload {  // descriptor + per-iteration tables: passed BY VALUE as __grid_constant__ kernel parameters (no H2D copy)
  dmv::BAWinDev win;
  dmv::BAIter it;
};

using dmv::MAXF; using dmv::XCHG_MAXR; using dmv::BAAdj; using dmv::BAMarg;

struct dmv_ba {
  dmv_ba_config cfg;
  dmv_ba_params prm;
  int device = 0;
  dmv::Stream stream;
  dmv::Event ev[4];
  int P = 16;            // points per chunk of the CURRENT window (16 or 32)
  bool P_auto = true;    // dmv_ba_config::chunk_points == 0: chosen per window in dmv_ba_set_points
  int sms = 132;
  int mp = 0;  // point capacity (slot pitch)
  int nf = 0, npts = 0, nres = 0, nchunks = 0, max_chunks = 0;
  int N = 0, NW = 0, T = 0, ntiles = 0;
  int slots[MAXF];
  // device buffers
  dmv::DevBuf<float4> d_img[MAXF];
  dmv::DevBuf<float> d_stage_img;
  dmv::DevBuf<BAAdj> d_adj;
  dmv::DevBuf<float2> d_uv;
  dmv::DevBuf<float> d_idepth[2];           // ping-pong: [cur] current depths, [bak] FullSystem::backupState copy
  int id_cur = 0, id_bak = 0;
  bool zero_alias = false;                  // idepth_zero == idepth (true after any step / restore)
  dmv::DevBuf<float> d_idepth_zero, d_color, d_weights, d_priorF;
  dmv::DevBuf<uint8_t> d_st_in;
  dmv::DevBuf<float> d_en_in;
  dmv::DevBuf<uint8_t> d_st_new[2];
  dmv::DevBuf<float> d_en_new[2], d_en_wo[2], d_cpt[2], d_jpjd[2], d_pout[2];
  dmv::DevBuf<double> d_result[2];
  dmv::DevBuf<float> d_step;
  dmv::DevBuf<double> d_part;      // [max_chunks][PART_STRIDE] per-chunk partial blobs (scratch of one launch)
  dmv::DevBuf<int4> d_dtab;        // phase D items [DITEMS_MAX][2] of the current window shape (dmv_ba_set_points)
  std::vector<int4> h_dtab;
  int nditems = 0;
  dmv::DevBuf<float4> d_wg;        // [WG_GROUPS][mp] Schur vectors, transposed (scratch)
  dmv::DevBuf<float> d_hdig;       // [mp] HdiF (scratch)
  dmv::DevBuf<float> d_hdi_solve;  // [mp] HdiF of the linearisation the last dmv_ba_accumulate returned (PointHessian::idepth_hessian)
  int hdi_solve_n = 0;
  dmv::DevBuf<unsigned int> d_bar; // grid-barrier arrival counter
  unsigned int bar_count = 0;      // arrivals issued so far (monotonic, wraps)
  dmv::DevBuf<double> d_resub_sums;
  dmv::DevBuf<float4> d_flush;     // L2 scrub of the benches, allocated on first use
  // pinned host
  dmv::PinnedBuf<HostUpload> h_up;
  dmv::PinnedBuf<BAAdj> h_adj;
  dmv::PinnedBuf<double> h_result[2];
  dmv::PinnedBuf<float> h_scratch;  // max(mp*8, w*h*3) floats
  dmv::PinnedBuf<float> h_en_newest; // [mp] en_wo of the residuals targeting the newest frame, written by the kernel itself (zero-copy)
  bool en_newest_valid = false; // h_en_newest belongs to the linearisation the getters read (tentative if any, else committed)
  // host bookkeeping
  int host_start[MAXF + 1];
  int chunk_beg[MAXF + 1];
  std::vector<int> host_of_point;
  std::vector<int> res_slot;   // residual index -> slot (t*mp+p)
  std::vector<uint8_t> h_st_in;
  std::vector<float> h_en_in;
  std::vector<int> ref_moves;  // dmv_ba_ref_source: FullSystem::removeOutliers' reorder as (from, to) point pairs
  bool st_in_clean = false;    // every existing residual's INPUT state on the device is IN with zero energy (dmv_ba_reset_oob becomes a flag flip)
  bool no_zero_copy = false;   // DMV_NO_ZERO_COPY=1: D2H copy node instead of in-kernel writes to the pinned result (A/B experiment)
  bool timing = false;         // record CUDA events around the kernels of every call (dmv_ba_set_timing)
  int tent = 0;                // index of the tentative buffer set; committed = 1 - tent
  bool have_tentative = false, have_committed = false, have_adj = false, have_state = false;
  long long launches = 0;
  float last_ms[4] = {0, 0, 0, 0};
  // NCCL
  void* nccl_comm = nullptr;
  int nranks = 1, rank = 0;
  // marginalisation launch (dmv_ba_marginalize_points): allocated on first use, as a whole
  dmv::DevBuf<BAMarg> d_marg;
  dmv::DevBuf<uint8_t> d_marg_mask;
  dmv::DevBuf<float> d_marg_rtz;
  dmv::DevBuf<double> d_marg_result;
  dmv::PinnedBuf<double> h_marg_result;
  dmv::DevBuf<float> d_act;    // point-activation staging (dmv_ba_activate_points)
  dmv::PinnedBuf<float> h_act;
  int act_cap = 0;             // points the staging layout holds (0 while d_act / h_act may be short of it)
  int act_n = -1;              // entries of the last activation on this window, whose host, status and res_state h_act holds (-1: none)
  // window edit (dmv_ba_edit_window, ba_edit.cu): the gather's destinations, swapped with the point arrays and input grids above; its
  // per-point upload and the carried residuals' compacted states.  Allocated on first use, as a whole
  dmv::DevBuf<float2> e_uv;
  dmv::DevBuf<float> e_idepth_zero, e_color, e_weights, e_priorF, e_en_in, e_cen;
  dmv::DevBuf<uint8_t> e_st_in, e_cst;
  dmv::DevBuf<int> e_src;
  bool res_valid = false;      // h_st_in / h_en_in / res_slot describe the current points (dmv_ba_set_residuals or an edit since set_points)
  dmv::DevBuf<float> d_sel;    // activation-selection staging and scratch (dmv_ba_select_activation, ip_select.cu)
  dmv::PinnedBuf<float> h_sel;
  // peer-memory exchange (inside ba_fused_kernel)
  dmv::DevBuf<uint4> xchg_own;              // this rank's inbox (exported through CUDA IPC)
  void* xchg_map[XCHG_MAXR] = {nullptr};    // every rank's inbox as mapped here ([rank] == xchg_own)
  int xchg_pitch = 0;
  bool xchg_on = false;
  unsigned int xchg_seq = 0;
};

// dmv_ba_activate_points' staging (words): RT[64*12] | aff[64*2] | host | u | v | color*8 | weights*8 | energyTH | idmin | idmax | status | idepth |
// res_state*MAXF | lastTraceStatus (dmv_ba_activate_store only), cap points per array.  [0, st) goes up, status .. res_state come back.
struct ActLayout {
  size_t rt, aff, host, u, v, col, wgt, eth, min, max, st, id, rs, ts, words;
};
inline ActLayout act_layout(size_t cap) {
  ActLayout o;
  o.rt = 0; o.aff = (size_t)MAXF * MAXF * 12; o.host = (size_t)MAXF * MAXF * 14; o.u = o.host + cap; o.v = o.u + cap; o.col = o.v + cap;
  o.wgt = o.col + 8 * cap; o.eth = o.wgt + 8 * cap; o.min = o.eth + cap; o.max = o.min + cap; o.st = o.max + cap; o.id = o.st + cap; o.rs = o.id + cap;
  o.ts = o.rs + MAXF * cap; o.words = o.ts + cap;
  return o;
}

// chunk shape of a window of points ordered by host frame: P, each host's first point and first chunk (dmv_ba_set_points, dmv_ba_edit_window)
struct BAShape {
  int P, nchunks;
  int host_start[MAXF + 1], chunk_beg[MAXF + 1];
};

// shared by the product path and the benches (library-internal: hidden from the dynamic symbol table)
#define DMV_INTERNAL extern "C" __attribute__((visibility("hidden")))
DMV_INTERNAL int dmv_ba_fill_descriptor(dmv_ba* b);
DMV_INTERNAL void dmv_ba_next_exchange(dmv_ba* b);
DMV_INTERNAL int dmv_ba_enqueue_exchange(dmv_ba* b);
DMV_INTERNAL void dmv_ba_stage_x(dmv_ba* b, const double* x);
DMV_INTERNAL int dmv_ba_check_ready(dmv_ba* b);
DMV_INTERNAL int dmv_ba_stage_state(dmv_ba* b, const dmv_ba_state* st);
DMV_INTERNAL int dmv_ba_finish_linearize(dmv_ba* b, dmv_ba_lin_result* out, double sums[3]);
DMV_INTERNAL void dmv_ba_window_shape(const dmv_ba* b, int npts, const int32_t* host, BAShape* s);
DMV_INTERNAL int dmv_ba_take_shape(dmv_ba* b, const BAShape* s);
