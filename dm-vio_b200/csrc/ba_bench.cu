// Measurement-only entry points (include/dmvio_b200_bench.h): used by bench.py and tools/, never by a DM-VIO host.
// Built into the library only with BENCH=1 (the Makefile default; `make BENCH=0` ships the product surface alone).
#include "../../include/dmvio_b200_bench.h"
#include "ba_handle.h"
#include <chrono>

using namespace dmv;

extern "C" {

// iters x { [L2 scrub] ; ba_fused_kernel ; [NCCL all-reduce] } with everything resident in HBM; CUDA events on the handle's stream
// bracket every launch: ms[i] = kernel + exchange, ms_k[i] = ba_fused_kernel alone.  clk != nullptr: the clocked instantiation of the
// kernel writes its phase stamps to clk + i * clk_rows * FUSED_NCLK (the caller checked clk_rows >= the window's chunks >= the grid),
// the grid goes to *grid.
static int bench_loop(dmv_ba* b, const double* x, int iters, int flush_l2, std::vector<float>& ms, std::vector<float>& ms_k,
                      unsigned long long* clk, int clk_rows, int* grid) {
  int rc = dmv_ba_check_ready(b);
  if (rc != DMV_OK) return rc;
  if (iters < 1 || iters > 4096) return set_error(DMV_ERR_INVALID, "iters out of range");
  if (x && !b->have_committed) return set_error(DMV_ERR_STATE, "no committed linearisation to resubstitute");
  CK(cudaSetDevice(b->device));
  if (flush_l2 && !b->d_flush) {
    b->flush_n = (size_t)256 * 1024 * 1024 / sizeof(float4);  // 256 MiB > 50 MB L2
    CK(cudaMalloc(&b->d_flush, b->flush_n * sizeof(float4)));
    CK(cudaMemset(b->d_flush, 0, b->flush_n * sizeof(float4)));
  }
  if (x) dmv_ba_stage_x(b, x); else b->h_up->it.have_x = 0;
  std::vector<cudaEvent_t> e(3 * (size_t)iters);
  for (auto& ev : e) CK(cudaEventCreate(&ev));
  for (int i = 0; i < iters; i++) {
    if (flush_l2) launch_l2_flush(b->d_flush, b->flush_n, b->stream);
    dmv_ba_fill_descriptor(b);
    dmv_ba_next_exchange(b);
    HostUpload& U = *b->h_up;
    CK(cudaEventRecord(e[3 * i], b->stream));
    if (clk) CK(launch_fused_kernel_clocked(U.win, U.it, b->stream, &b->bar_count, clk + (size_t)i * clk_rows * FUSED_NCLK, grid));
    else CK(launch_fused_kernel(U.win, U.it, false, b->stream, &b->bar_count));
    CK(cudaEventRecord(e[3 * i + 1], b->stream));
    if (b->nccl_comm && !b->xchg_on) {  // a separate all-reduce follows the kernel: the step ends behind it
      rc = dmv_ba_enqueue_exchange(b);
      if (rc != DMV_OK) return rc;
      CK(cudaEventRecord(e[3 * i + 2], b->stream));
    }
    b->launches += 1;
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(b->stream));
  ms.assign(iters, 0.f);
  ms_k.assign(iters, 0.f);
  for (int i = 0; i < iters; i++) {
    cudaEventElapsedTime(&ms_k[i], e[3 * i], e[3 * i + 1]);
    if (b->nccl_comm && !b->xchg_on) cudaEventElapsedTime(&ms[i], e[3 * i], e[3 * i + 2]);
    else ms[i] = ms_k[i];  // the step IS the kernel (the peer exchange, if any, happens inside it)
  }
  for (auto& ev : e) cudaEventDestroy(ev);
  b->h_up->it.have_x = 0;
  b->have_tentative = true;
  return DMV_OK;
}

int dmv_ba_bench_device(dmv_ba* b, const double* x, int iters, int flush_l2, float* ms_per_iter, float* ms_kernel) {
  std::vector<float> ms, ms_k;
  const int rc = bench_loop(b, x, iters, flush_l2, ms, ms_k, nullptr, 0, nullptr);
  if (rc != DMV_OK) return rc;
  double tot = 0, pk = 0;
  for (int i = 0; i < iters; i++) { tot += ms[i]; pk += ms_k[i]; }
  if (ms_per_iter) *ms_per_iter = (float)(tot / iters);
  if (ms_kernel) *ms_kernel = (float)(pk / iters);
  return DMV_OK;
}

int dmv_ba_bench_phases(dmv_ba* b, const double* x, int iters, int flush_l2, int max_ctas, unsigned long long* stamps, int* n_ctas, float* ms_kernel) {
  if (!b || !stamps || !n_ctas || !ms_kernel || max_ctas < 1) return set_error(DMV_ERR_INVALID, "bad argument");
  if (iters < 1 || iters > 4096) return set_error(DMV_ERR_INVALID, "iters out of range");
  int rc = dmv_ba_check_ready(b);
  if (rc != DMV_OK) return rc;
  if (b->nccl_comm) return set_error(DMV_ERR_STATE, "the phase clock times the launch alone: no NCCL communicator");
  rc = dmv_ba_fill_descriptor(b);
  if (rc != DMV_OK) return rc;
  if (b->h_up->win.nchunks > max_ctas) return set_error(DMV_ERR_INVALID, "max_ctas below the window's chunk count");
  const size_t n = (size_t)iters * max_ctas * FUSED_NCLK;
  CK(cudaSetDevice(b->device));
  unsigned long long* d_clk = nullptr;
  CK(cudaMalloc(&d_clk, n * sizeof(unsigned long long)));
  if (cudaMemset(d_clk, 0, n * sizeof(unsigned long long)) != cudaSuccess) rc = set_error(DMV_ERR_CUDA, "cudaMemset failed");
  std::vector<float> ms, ms_k;
  int grid = 0;
  if (rc == DMV_OK) rc = bench_loop(b, x, iters, flush_l2, ms, ms_k, d_clk, max_ctas, &grid);
  if (rc == DMV_OK && cudaMemcpy(stamps, d_clk, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess)
    rc = set_error(DMV_ERR_CUDA, "cudaMemcpy failed");
  cudaFree(d_clk);
  if (rc != DMV_OK) return rc;
  *n_ctas = grid;
  for (int i = 0; i < iters; i++) ms_kernel[i] = ms_k[i];
  return DMV_OK;
}

// End-to-end timing of the public call sequence a DM-VIO host makes per GN iteration, from C (no interpreter in the loop):
// iters x { dmv_ba_gn_step(x, st) ; dmv_ba_apply_res() } with host buffers in and H/b out, wall clock (steady_clock).
int dmv_ba_bench_e2e(dmv_ba* b, const double* x, const dmv_ba_state* st, int iters, double* ms_per_iter) {
  if (!b || !st || !ms_per_iter || iters < 1) return set_error(DMV_ERR_INVALID, "bad argument");
  dmv_ba_lin_result r;
  double sums[3];
  CK(cudaSetDevice(b->device));
  CK(cudaStreamSynchronize(b->stream));
  const auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < iters; i++) {
    int rc = dmv_ba_gn_step(b, x, st, &r, sums);
    if (rc != DMV_OK) return rc;
    rc = dmv_ba_apply_res(b);
    if (rc != DMV_OK) return rc;
  }
  const auto t1 = std::chrono::steady_clock::now();
  *ms_per_iter = std::chrono::duration<double, std::milli>(t1 - t0).count() / iters;
  return DMV_OK;
}

// batched windows: `iters` x dmv_ba_batch_gn_step (+ apply_res on every handle), wall clock per call and CUDA-event time of the launch alone
int dmv_ba_batch_bench(dmv_ba_batch* B, dmv_ba* const* handles, int n, const double* const* x, const dmv_ba_state* const* st, int iters, double* e2e_ms_per_iter,
                       double* kernel_ms_per_iter) {
  if (!B || !handles || !st || iters < 1) return set_error(DMV_ERR_INVALID, "bad argument");
  int rc = dmv_ba_batch_set_timing(B, 1);
  if (rc != DMV_OK) return rc;
  double ksum = 0;
  const auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < iters; i++) {
    rc = dmv_ba_batch_gn_step(B, x, st, nullptr, nullptr);
    if (rc != DMV_OK) return rc;
    for (int k = 0; k < n; k++) {
      rc = dmv_ba_apply_res(handles[k]);
      if (rc != DMV_OK) return rc;
    }
    float ms = 0.f;
    dmv_ba_batch_last_kernel_ms(B, &ms);
    ksum += ms;
  }
  const auto t1 = std::chrono::steady_clock::now();
  if (e2e_ms_per_iter) *e2e_ms_per_iter = std::chrono::duration<double, std::milli>(t1 - t0).count() / iters;
  if (kernel_ms_per_iter) *kernel_ms_per_iter = ksum / iters;
  return dmv_ba_batch_set_timing(B, 0);
}

}  // extern "C"
