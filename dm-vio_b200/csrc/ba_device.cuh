// Device-side data layout of one sliding window (DESIGN.md §3).
// The window descriptor (BAWinDev, ~0.5 KB) and the per-iteration tables (BAIter, ~10.6 KB) travel as
// __grid_constant__ kernel parameters: no H2D copy node, no dependent global load before the first useful load.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dmv {

constexpr int MAXF = 8;             // DMV_MAX_FRAMES
constexpr int TOP_ROWS = 10;        // geometric rows [C4 | xi6] of the 13x13 pair block
constexpr int TOP_COLS = 13;
// One (host,target) pair block = the 91 distinct entries of the symmetric 13x13 AccumulatorApprox (MatrixAccumulators.h:L595-972):
// rows 0..9 packed upper-triangular (row r holds columns r..12), then the 6 bottom-right (a,b,r) entries, padded to 92 (16-byte rows).
constexpr int TOP_TRI = 85;                        // sum_{r=0}^{9} (13 - r)
constexpr int TOP_USED = TOP_TRI + 6;              // 91
constexpr int TOP_PART = 92;
__host__ __device__ constexpr int top_off(int r) { return r * TOP_COLS - (r * (r - 1)) / 2; }  // offset of entry (r, r); entry (r, c>=r) = top_off(r) + c - r
constexpr int RES_NONE = 255, RES_IN = 0, RES_OOB = 1, RES_OUTLIER = 2;
constexpr int FUSED_NCLK = 9;      // phase-clock stamps per CTA of the measurement-only clocked launch (ba_fused.cu: clk_stamp)
constexpr int ACC_MISC = 8;         // energy, n_in, n_oob, n_outlier, sum step^2, sum |idepth_backup|, npts, error flag (barrier / peer timeout)
// Partial blob of one chunk (P points of host frame h), fp64, written by phase C of ba_fused_kernel with plain stores and summed in a
// fixed order by phase D.  Per frame slot t: [O 64 | D 64 | C 32 | b 8]: t != h: O = contribution to H[h,t], D to H[t,t], C to H[t,C],
// b to b[t]; t == h: D to H[h,h], C to H[h,C], b to b[h] (O unused).  Then H[C,C] (16), b[C] (4), the ACC_MISC counters.
constexpr int PART_SLOT = 168;
constexpr int PART_CC = MAXF * PART_SLOT;
constexpr int PART_MISC = PART_CC + 20;
constexpr int PART_STRIDE = PART_MISC + ACC_MISC;

// per-iteration parameter block
struct BAIter {
  float calib[8];                 // fxl fyl cxl cyl fxli fyli cxli cyli
  float TH[MAXF];                 // frameEnergyTH
  float precalc[MAXF * MAXF][32]; // [h*nf + t] : KRKi[9] Kt[3] R0[9] t0[3] aff[2] b0
  float xAd[MAXF * MAXF][8];      // [h*nf + t] : x_h^T adHostF + x_t^T adTargetF   (resubstitute)
  float xc[4];                    // x.head<4>() as float
  int have_x;                     // 0: skip the resubstitute/step prologue
  int pad[3];
};

// adjoints (host -> device once per linearisation point)
struct BAAdj {
  float adHostF[MAXF * MAXF][64];   // [h*nf + t] row-major 8x8
  float adTdiagF[MAXF * MAXF][8];   // [h*nf + t] diagonal of adTarget
  double adHost[MAXF * MAXF][64];   // [h*nf + t]
  double adTdiag[MAXF * MAXF][8];
};

// peer-memory exchange inside ba_fused_kernel (DESIGN.md §7).  Inbox of one rank (cudaMalloc + CUDA IPC):
// [2 parities][XCHG_MAXR source ranks][pitch] 16-byte packets {value.lo, seq, value.hi, seq}  ("LL" packets: flag travels with the data)
constexpr int XCHG_MAXR = 8;
struct BAXchg {
  int nranks, rank, pitch;            // pitch = packets per (parity, source) slot >= result_doubles
  unsigned int seq;                   // exchange number 1, 2, ... (identical on every rank); 0 never appears as a flag of a live packet
  uint4* inbox[XCHG_MAXR];            // rank r's inbox as mapped in THIS process ([rank] = own)
};

// tables of a marginalisation launch (dmv_ba_marginalize_points -> ba_fused_kernel<.., MARG = true>); device memory, never read in production
struct BAMarg {
  float adHTdelta[MAXF * MAXF][8];  // [h*nf + t]: (state - state_zero)_h^T adHostF + (..)_t^T adTargetF  (EnergyFunctional.cpp:L175-198)
  float cDelta[4];                  // calibration value - value_zero (scaled), as float
  float priorFac;                   // setting_idepthFixPriorMargFac (EnergyFunctional.cpp:L693)
  int pad[3];
};

struct BAWinDev {
  int nf, npts, nchunks, w, h, N, NW, T, ntiles, mp, P;  // mp = capacity (row pitch of the [target][point] slot arrays)
  float huberTH, outlierTHSum;
  int zeroA, zeroB;
  int host_start[MAXF + 1];  // points of host h are [host_start[h], host_start[h+1])
  int chunk_beg[MAXF + 1];   // chunks (CTAs) of host h are [chunk_beg[h], chunk_beg[h+1]); chunk c covers P consecutive points
  const float4* img[MAXF];   // per window frame index: level-0 texels (I, dx, dy, 0)
  const BAAdj* adj;
  // points
  const float2* uv;
  const float* idepth;        // current inverse depths (read when no step is fused)
  const float* idepth_zero;   // FEJ inverse depths (aliases idepth after the first step / restore: DM-VIO keeps them equal)
  const float* idepth_backup; // FullSystem::backupState copy: ping-pong buffer, no copy kernel
  float* idepth_out;          // where a fused / stand-alone step writes idepth_backup + step
  const float* color;        // [p][8]
  const float* weights;      // [p][8]
  const float* priorF;
  // residual slots, [t*mp + p]
  const uint8_t* st_in;      // state_state
  const float* en_in;        // state_energy
  uint8_t* st_new;           // tentative outputs of this linearisation
  float* en_new;
  float* en_wo;
  float* en_wo_newest_host;  // pinned host mirror of en_wo for target frame nf-1 (setNewFrameEnergyTH's percentile input), or nullptr
  float* cpt;                // 3 planes [k][slot]
  float* jpjd;               // [slot][8]
  float* pout;               // [p][8]: Hdd bd Hcd[4] HdiF bdSum
  // committed copies (read by resubstitute)
  const uint8_t* c_st;
  const float* c_jpjd;
  const float* c_pout;
  float* step;               // [p]
  // scratch of one launch (never read by the host)
  double* part;              // [chunk][PART_STRIDE] partial blobs
  float4* wg;                // [4-column group][mp] Schur vectors w_p, transposed
  float* hdig;               // [p] HdiF
  unsigned int* bar;         // grid-barrier arrival counter (monotonic)
  unsigned int bar_target;   // arrivals expected once every CTA of THIS launch has arrived
  double* result;            // H_top N*N | b_top N | Schur tiles ntiles*16 | ACC_MISC tail
  double* result_host;       // pinned host mirror of the result blob written by the kernel itself (zero-copy), or nullptr
  BAXchg xc;                 // nranks <= 1: no exchange
  // marginalisation launch only (nullptr otherwise)
  const BAMarg* marg;
  const uint8_t* marg_mask;  // [p] 1 = point is being marginalised
  float* marg_rtz;           // [slot][8] EFResidual::res_toZeroF of the residuals linearised by the launch
};

// header of a batched launch (ba_fused_batch_kernel): B windows, work items = (window, chunk)
constexpr int BATCH_MAX = 64;
struct BABatchHdr {
  int B, total;                  // windows, sum of their chunk counts
  int prefix[BATCH_MAX + 1];     // first work item of window w
  unsigned int* bar;             // grid-barrier arrival counter of the batch
  unsigned int bar_target;
};

// result blob: H_top N*N | b_top N | raw Schur Gram tiles ntiles*16 | ACC_MISC counters
inline __host__ __device__ int result_doubles(int N, int ntiles) { return N * N + N + ntiles * 16 + ACC_MISC; }

}  // namespace dmv
