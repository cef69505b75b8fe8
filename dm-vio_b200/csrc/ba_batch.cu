// Batched windows (SURVEY.md §8d "batched variant"): B independent sliding windows — each an ordinary BA handle with its own keyframes,
// points and state — linearised by ONE launch of ba_fused_batch_kernel.  One window is a latency-bound chain on an L2-sized working set;
// a batch keeps all SMs busy and streams B x 34 MB of level-0 planes, which is the regime the HBM roofline describes.
// No reference counterpart (the reference optimises one window at a time, FullSystem::optimize): this is the throughput mode of the
// same hot path (offline re-optimisation / several sessions per GPU); per window the results are bit-identical to its own launch.
#include "ba_handle.h"
#include <cstring>
#include <memory>

using namespace dmv;

struct BatchUpload {
  BAWinDev win[BATCH_MAX];
  BAIter it[BATCH_MAX];
};

struct dmv_ba_batch {
  std::vector<dmv_ba*> h;
  int device = 0, P = 16, max_nf = 2;
  cudaStream_t stream = nullptr;   // = the first handle's stream
  PinnedBuf<BatchUpload> h_up;     // pinned staging
  DevBuf<BAWinDev> d_win;
  DevBuf<BAIter> d_it;
  DevBuf<unsigned int> d_bar;
  unsigned int bar_count = 0;
  Event ev[2];
  float last_ms = 0.f;
  bool timing = false;
};

extern "C" {

int dmv_ba_batch_create(dmv_ba* const* handles, int n, dmv_ba_batch** out) {
  if (!handles || !out || n < 1 || n > BATCH_MAX) return set_error(DMV_ERR_INVALID, "1..%d handles", BATCH_MAX);
  for (int i = 0; i < n; i++) {
    if (!handles[i]) return set_error(DMV_ERR_INVALID, "handle %d is null", i);
    for (int j = 0; j < i; j++)  // one launch would run both members on the same buffers
      if (handles[j] == handles[i]) return set_error(DMV_ERR_INVALID, "handles[%d] and handles[%d] are the same handle", j, i);
    if (handles[i]->device != handles[0]->device || handles[i]->P != handles[0]->P) return set_error(DMV_ERR_INVALID, "all handles of a batch must share the device and chunk_points");
    if (handles[i]->nranks > 1) return set_error(DMV_ERR_INVALID, "sharded handles cannot be batched");
  }
  std::unique_ptr<dmv_ba_batch> B(new dmv_ba_batch());   // a failed call below releases what was allocated
  B->h.assign(handles, handles + n);
  B->device = handles[0]->device;
  B->P = handles[0]->P;
  B->stream = handles[0]->stream;
  CK(cudaSetDevice(B->device));
  CK(B->h_up.alloc(1));
  CK(B->d_win.alloc(BATCH_MAX));
  CK(B->d_it.alloc(BATCH_MAX));
  CK(B->d_bar.alloc(1));
  CK(cudaMemset(B->d_bar, 0, sizeof(unsigned int)));
  for (int i = 0; i < 2; i++) CK(cudaEventCreate(B->ev[i].put()));
  *out = B.release();
  return DMV_OK;
}

int dmv_ba_batch_destroy(dmv_ba_batch* B) {
  if (!B) return DMV_OK;
  cudaSetDevice(B->device);
  cudaStreamSynchronize(B->stream);
  delete B;
  return DMV_OK;
}

// dmv_ba_gn_step on every handle of the batch, ONE kernel launch: x[i] (may be NULL) = the solved increment whose point half is fused in,
// st[i] = the window's per-iteration tables.  Afterwards every handle is exactly as after its own dmv_ba_gn_step (tentative linearisation
// present, result blob in its pinned mirror): dmv_ba_apply_res / dmv_ba_accumulate / ... per handle as usual.
int dmv_ba_batch_gn_step(dmv_ba_batch* B, const double* const* x, const dmv_ba_state* const* st, dmv_ba_lin_result* out, double* sums3) {
  if (!B || !st) return set_error(DMV_ERR_INVALID, "null argument");
  CK(cudaSetDevice(B->device));
  const int n = (int)B->h.size();
  B->P = B->h[0]->P;   // with chunk_points = 0 a handle picks its shape per window: the batch needs ONE shape
  // every check precedes the first upload: a refused call leaves every member as it was
  for (int i = 0; i < n; i++) {
    const dmv_ba* b = B->h[i];
    if (b->P != B->P) return set_error(DMV_ERR_STATE, "window %d uses %d-point chunks, window 0 %d: create the handles of a batch with an explicit chunk_points", i, b->P, B->P);
    if (!st[i]) return set_error(DMV_ERR_INVALID, "state %d is null", i);
    if (!st[i]->precalc || !st[i]->frameEnergyTH) return set_error(DMV_ERR_INVALID, "state %d: precalc / frameEnergyTH required", i);
    if (b->xchg_on) return set_error(DMV_ERR_STATE, "window %d is sharded with the in-kernel peer exchange: the batched kernel has none", i);
    if (b->npts < 1) return set_error(DMV_ERR_STATE, "window %d: points not set", i);
    if (!b->have_adj) return set_error(DMV_ERR_STATE, "window %d: dmv_ba_set_adjoints first", i);
    if (x && x[i] && !b->have_committed) return set_error(DMV_ERR_STATE, "window %d: no committed linearisation to resubstitute", i);
  }
  BABatchHdr hdr;
  std::memset(&hdr, 0, sizeof(hdr));
  hdr.B = n;
  B->max_nf = 2;
  for (int i = 0; i < n; i++) {
    dmv_ba* b = B->h[i];
    const double* xi = x ? x[i] : nullptr;
    if (b->stream != B->stream) CK(cudaStreamSynchronize(b->stream));  // uploads issued on the handle's own stream
    int rc = dmv_ba_stage_state(b, st[i]);   // (idepth uploads, if any, go to the handle's stream: synchronised below)
    if (rc != DMV_OK) return rc;
    if (st[i]->idepth || st[i]->idepth_zero) CK(cudaStreamSynchronize(b->stream));
    if (xi) dmv_ba_stage_x(b, xi); else b->h_up->it.have_x = 0;
    dmv_ba_fill_descriptor(b);
    double* hres = b->h_result[b->tent];
    hres[(size_t)b->N * b->N + b->N + (size_t)b->ntiles * 16 + (ACC_MISC - 1)] = 0.0;
    b->h_up->win.result_host = hres;
    B->h_up->win[i] = b->h_up->win;
    B->h_up->it[i] = b->h_up->it;
    hdr.prefix[i] = hdr.total;
    hdr.total += b->nchunks;
    B->max_nf = std::max(B->max_nf, b->nf);
  }
  hdr.prefix[n] = hdr.total;
  hdr.bar = B->d_bar;
  CK(cudaMemcpyAsync(B->d_win, B->h_up->win, sizeof(BAWinDev) * n, cudaMemcpyHostToDevice, B->stream));
  CK(cudaMemcpyAsync(B->d_it, B->h_up->it, sizeof(BAIter) * n, cudaMemcpyHostToDevice, B->stream));
  if (B->timing) CK(cudaEventRecord(B->ev[0], B->stream));
  CK(launch_fused_batch_kernel(B->P, B->d_win, B->d_it, hdr, B->max_nf, B->stream, &B->bar_count));
  if (B->timing) CK(cudaEventRecord(B->ev[1], B->stream));
  CK(cudaStreamSynchronize(B->stream));
  if (B->timing) cudaEventElapsedTime(&B->last_ms, B->ev[0], B->ev[1]);
  for (int i = 0; i < n; i++) {
    dmv_ba* b = B->h[i];
    b->launches += (i == 0);
    b->en_newest_valid = true;
    int rc = dmv_ba_finish_linearize(b, out ? out + i : nullptr, sums3 ? sums3 + 3 * i : nullptr);
    b->h_up->it.have_x = 0;
    if (rc != DMV_OK) return rc;
  }
  return DMV_OK;
}

int dmv_ba_batch_set_timing(dmv_ba_batch* B, int enable) {
  if (!B) return set_error(DMV_ERR_INVALID, "null handle");
  B->timing = enable != 0;
  return DMV_OK;
}
int dmv_ba_batch_last_kernel_ms(dmv_ba_batch* B, float* ms) {
  if (!B || !ms) return set_error(DMV_ERR_INVALID, "null argument");
  *ms = B->last_ms;
  return DMV_OK;
}

}  // extern "C"
