/* dmvio_b200_bench.h — measurement-only entry points of libdmvio_b200.so (bench.py, tools/).  Not part of the drop-in surface:
 * a DM-VIO host never calls these; they exist so that the timed regions run without an interpreter in the loop.
 * Compiled into the library with BENCH=1 (Makefile default). */
#ifndef DMVIO_B200_BENCH_H
#define DMVIO_B200_BENCH_H
#include "dmvio_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Device-resident throughput: runs the device part of one GN iteration (fused resubstitute + step if x != NULL, ba_fused_kernel, the
 * NCCL all-reduce if a communicator is attached) `iters` times on the handle's stream with all inputs resident in HBM, each iteration
 * bracketed by CUDA events and optionally preceded by an untimed larger-than-L2 scrub; returns the average device milliseconds per
 * iteration and of ba_fused_kernel alone. */
int dmv_ba_bench_device(dmv_ba* ba, const double* x, int iters, int flush_l2, float* ms_per_iter, float* ms_kernel);
/* Phase clock of the same loop (one window, no NCCL communicator: DMV_ERR_STATE): `iters` x { [L2 scrub] ; the clocked instantiation of ba_fused_kernel }, in which
 * thread 0 of every CTA records %globaltimer (ns) at 9 points: kernel entry, chunk decoded, first loads returned, taps returned, end of phase
 * A, end of phase C, grid barrier released, end of phase D, end of phase E.  stamps: iters x max_ctas x 9, iteration i's CTA c at
 * stamps[(i * max_ctas + c) * 9 + k] (0 = not reached); *n_ctas = the grid; ms_kernel[i] = CUDA-event time of launch i.  max_ctas
 * must be >= the window's chunk count.  Stamps 1-5 are per chunk: a CTA that runs several chunks keeps those of its last one, so the
 * segments are exact only for a window of at most one chunk per CTA (the headline).  The product kernels carry no clock. */
int dmv_ba_bench_phases(dmv_ba* ba, const double* x, int iters, int flush_l2, int max_ctas, unsigned long long* stamps, int* n_ctas, float* ms_kernel);
/* wall-clock time of `iters` x { dmv_ba_gn_step(x, st) ; dmv_ba_apply_res() } issued from C, milliseconds per iteration */
int dmv_ba_bench_e2e(dmv_ba* ba, const double* x, const dmv_ba_state* st, int iters, double* ms_per_iter);

/* `iters` x { dmv_ba_batch_gn_step(x, st) ; dmv_ba_apply_res on each of the n handles }: wall clock per iteration (host tables in, B result
 * blobs out, sync inside) and the CUDA-event time of the batched launch alone */
int dmv_ba_batch_bench(dmv_ba_batch* batch, dmv_ba* const* handles, int n, const double* const* x, const dmv_ba_state* const* st, int iters,
                       double* e2e_ms_per_iter, double* kernel_ms_per_iter);

#ifdef __cplusplus
}
#endif
#endif
