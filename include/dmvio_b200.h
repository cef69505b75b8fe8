/* dmvio_b200.h — C ABI of the H100-native DM-VIO photometric hot path.
 *
 * Drop-in boundary (SURVEY.md §8b).  Plain C, opaque handles, int status codes, caller-owned host
 * buffers, one CUDA stream per handle, no global mutable state: a BA handle (mapper thread) and a
 * coarse-tracker handle (tracker thread) never share anything.  Every entry point names the reference
 * interface it replaces (paths relative to the reference's src/dso/).
 *
 * Conventions shared with the reference:
 *   - state vector order  [C(4) | frame0: trans3 rot3 a b | frame1 ...],  N = 8*nf + 4
 *     (OptimizationBackend/EnergyFunctional.cpp:L1019-1024)
 *   - pair index of adjoint-like tables:  h + t*nf   (AccumulatedTopHessian.cpp:L71)
 *   - pair index of precalc tables:       h*nf + t   (host->targetPrecalc[target], FullSystem.cpp:L1670-1680)
 *   - x returned by the solve is -step               (EnergyFunctional.cpp:L975)
 *   - residual states: 0 = IN, 1 = OOB, 2 = OUTLIER  (FullSystem/Residuals.h:L43); 255 = "no residual in this slot"
 *
 * All functions return DMV_OK (0) or a negative dmv_status.  dmv_last_error() gives a message for the
 * calling thread.  There is NO CPU fallback: without a CUDA device every create() fails with DMV_ERR_NO_DEVICE.
 */
#ifndef DMVIO_B200_H
#define DMVIO_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMV_MAX_FRAMES 8      /* setting_maxFrames = 7 (+1 while the new keyframe is being optimised), util/settings.cpp:L100 */
#define DMV_PATTERN 8         /* patternNum, util/settings.h:L227 */
#define DMV_PRECALC_FLOATS 32 /* KRKi[9] Kt[3] R0[9] t0[3] aff[2] b0 pad[5] */
#define DMV_MAX_PYR_LEVELS 6  /* PYR_LEVELS, util/settings.h:L52 */

typedef enum dmv_status {
  DMV_OK = 0,
  DMV_ERR_INVALID = -1,   /* bad argument / inconsistent sizes */
  DMV_ERR_NO_DEVICE = -2, /* no usable CUDA device: the product has no CPU path */
  DMV_ERR_CUDA = -3,      /* a CUDA runtime call failed (see dmv_last_error) */
  DMV_ERR_STATE = -4,     /* call order violated (e.g. accumulate before linearize+apply) */
  DMV_ERR_NCCL = -5,
  DMV_ERR_TIMEOUT = -6    /* a grid barrier or the peer exchange inside a kernel gave up waiting (lost rank / CTA) */
} dmv_status;

const char* dmv_last_error(void);
const char* dmv_version(void);
int dmv_device_count(void);

/* ------------------------------------------------------------------------------------------------
 * Bundle-adjustment handle  ==  the GPU side of EnergyFunctional + FullSystem::linearizeAll
 * ------------------------------------------------------------------------------------------------ */
typedef struct dmv_ba dmv_ba;

typedef struct dmv_ba_config {
  int w, h;           /* level-0 image size (wG[0], hG[0]) */
  int max_frames;     /* <= DMV_MAX_FRAMES */
  int max_points;     /* capacity of the active point set */
  int device;         /* CUDA device ordinal */
  int chunk_points;   /* points per thread block: 16 or 32; 0 = chosen per window (16 up to 16 x #SMs points, i.e. one wave; 32 beyond) */
} dmv_ba_config;

/* util/settings.cpp values read by the kernels (constant during a run) */
typedef struct dmv_ba_params {
  float huberTH;                /* setting_huberTH = 9 */
  float outlierTHSumComponent;  /* setting_outlierTHSumComponent = 50*50 */
  float affineOptModeA;         /* <0: JabF[0] is zeroed (Residuals.cpp:L229-242) */
  float affineOptModeB;
} dmv_ba_params;

int dmv_ba_create(const dmv_ba_config* cfg, dmv_ba** out);
int dmv_ba_destroy(dmv_ba* ba);
int dmv_ba_set_params(dmv_ba* ba, const dmv_ba_params* p);
void dmv_ba_default_params(dmv_ba_params* p);

/* FrameHessian::dI (HessianBlocks.h:L122): level-0 [I,dx,dy] AoS, w*h*3 floats, into image slot `slot`
 * (0 <= slot < max_frames).  Slots let frames stay resident across keyframes while window indices shift. */
int dmv_ba_upload_frame(dmv_ba* ba, int slot, const float* dI_aos3);
/* Same, but builds [I,dx,dy] on the device from the raw float image (FrameHessian::makeImages, HessianBlocks.cpp:L128-191, level 0). */
int dmv_ba_upload_image(dmv_ba* ba, int slot, const float* image_wh);
/* Same frame, no second upload: the level-0 [I,dx,dy] plane is copied device-to-device from the coarse-tracker handle in which the frame is
 * resident (dmv_ct_upload_new_image when it arrived; same device).  The reference shares one FrameHessian::dIp between tracker and mapper
 * (HessianBlocks.h:L122-123); here the frame crosses PCIe once and makeImages runs once. */
struct dmv_ct;
int dmv_ba_adopt_frame(dmv_ba* ba, int slot, struct dmv_ct* ct);

/* EnergyFunctional::makeIDX (EnergyFunctional.cpp:L998-1016): window frame index -> image slot */
int dmv_ba_set_window(dmv_ba* ba, int nf, const int* slots);

/* EFPoint/PointHessian fields read on the path (HessianBlocks.h:L413-508, EnergyFunctionalStructs.h:L104-137).
 * Points must be ordered by host frame index (that is EnergyFunctional::allPoints' order).
 * color8/weights8: npts*8.  priorF/deltaF may be NULL (zeros). */
int dmv_ba_set_points(dmv_ba* ba, int npts, const int32_t* host, const float* u, const float* v, const float* idepth,
                      const float* idepth_zero, const float* color8, const float* weights8, const float* priorF);

/* The active (non-linearised) PointFrameResiduals of the window: (point, target) pairs, at most one per pair,
 * with PointFrameResidual::state_state / state_energy (Residuals.h:L64-84).  state_state/state_energy may be NULL (all IN / 0). */
int dmv_ba_set_residuals(dmv_ba* ba, int nres, const int32_t* point, const int32_t* target, const int32_t* state_state,
                         const float* state_energy);

/* EnergyFunctional::setAdjointsF (EnergyFunctional.cpp:L48-108): adHost/adTarget, nf*nf 8x8 row-major doubles, index h + t*nf */
int dmv_ba_set_adjoints(dmv_ba* ba, const double* adHost, const double* adTarget);

/* Per-iteration state == FullSystem::setPrecalcValues (FrameFramePrecalc::set, HessianBlocks.cpp:L193-223) + CalibHessian values +
 * FrameHessian::frameEnergyTH.  idepth (npts) may be NULL: keep the device copy (e.g. after dmv_ba_resubstitute(apply=1)).
 * idepth_zero likewise.  deltaF (npts) = idepth - idepth_zero for the prior shift (EnergyFunctional.cpp:L194); NULL => recomputed on device. */
typedef struct dmv_ba_state {
  float calib[8];          /* fxl fyl cxl cyl fxli fyli cxli cyli (CalibHessian::value_scaledf / value_scaledi) */
  const float* precalc;    /* nf*nf*DMV_PRECALC_FLOATS, index h*nf + t */
  const float* frameEnergyTH; /* nf */
  const float* idepth;     /* npts or NULL */
  const float* idepth_zero;/* npts or NULL */
} dmv_ba_state;
int dmv_ba_set_state(dmv_ba* ba, const dmv_ba_state* st);

/* FullSystem::linearizeAll(false) (FullSystemOptimize.cpp:L150-218) fused with the *tentative* accumulateAF/SCF of the
 * next solveSystemF: evaluates every active residual at the current state, reduces the per-pair 13x13 blocks, the
 * per-point Hdd/bd/Hcd and the Schur complement, and assembles the dense system on the device (one launch).
 * Nothing becomes visible to dmv_ba_accumulate / dmv_ba_resubstitute until dmv_ba_apply_res().
 * out: energy = sum of PointFrameResidual::linearize() return values (stats[0]); n_in = #residuals with state_NewState==IN. */
typedef struct dmv_ba_lin_result {
  double energy;
  int n_in, n_oob, n_outlier;
} dmv_ba_lin_result;
int dmv_ba_linearize(dmv_ba* ba, dmv_ba_lin_result* out);

/* Per-residual outputs of the last linearize, in the order given to dmv_ba_set_residuals
 * (state_NewState, state_NewEnergy, state_NewEnergyWithOutlier, centerProjectedTo; Residuals.h:L64-84) and JpJdF, which is defined for
 * residuals with state_NewState == IN only (EFResidual::takeDataF runs on active residuals). Any pointer may be NULL. */
int dmv_ba_get_residual_outputs(dmv_ba* ba, int32_t* newState, float* newEnergy, float* newEnergyWithOutlier, float* centerProjectedTo3,
                                float* JpJdF8);

/* state_NewEnergyWithOutlier of the residuals whose target is frame `target` (input of FullSystem::setNewFrameEnergyTH,
 * FullSystemOptimize.cpp:L96-149): writes at most cap floats, returns the count in *n. Entries < 0 (not evaluated) are skipped.
 * Every target, the newest frame included, reports the linearisation dmv_ba_get_residual_outputs reports: the tentative one if there is one,
 * else the committed one (after dmv_ba_marginalize_points: the committed one), in point order. */
int dmv_ba_get_target_energies(dmv_ba* ba, int target, float* out, int cap, int* n);

/* PointFrameResidual::applyRes(true) + EFResidual::takeDataF for all active residuals (FullSystemOptimize.cpp:L90-94):
 * commits the tentative linearisation (buffer swap; no kernel). */
int dmv_ba_apply_res(dmv_ba* ba);

/* The accumulate half of EnergyFunctional::solveSystemF (EnergyFunctional.cpp:L853-860): accumulateAF_MT + accumulateSCF_MT of the
 * committed linearisation.  H_A/H_sc: N*N row-major doubles, b_A/b_sc: N.  (accumulateLF_MT's priors are host data; the host adapter adds them.)
 * resInA = AccumulatedTopHessianSSE::nres[0]. */
int dmv_ba_accumulate(dmv_ba* ba, double* H_A, double* b_A, double* H_sc, double* b_sc, int* resInA);

/* Per-point results of the committed accumulation: EFPoint::{Hdd_accAF, bd_accAF, Hcd_accAF, HdiF, bdSumF} (EnergyFunctionalStructs.h:L117-135).
 * Any pointer may be NULL. */
int dmv_ba_get_point_outputs(dmv_ba* ba, float* Hdd_accAF, float* bd_accAF, float* Hcd_accAF4, float* HdiF, float* bdSumF);
/* EFPoint::HdiF as AccumulatedSCHessian::addPoint left it during the last solveSystemF (AccumulatedSCHessian.cpp:L42-50; idepth_hessian =
 * 1 / HdiF): the values of the linearisation the last dmv_ba_accumulate() returned, kept on the device while later linearisations
 * (rejected steps, the tail's linearizeAll(true)) overwrite the per-point outputs.  FullSystem::flagPointsForRemoval reads it (FullSystem.cpp:L840-850). */
int dmv_ba_get_solve_HdiF(dmv_ba* ba, float* HdiF);

/* EnergyFunctional::resubstituteF_MT (EnergyFunctional.cpp:L267-321): x = N doubles (= -step).  step_out (npts) may be NULL.
 * apply != 0 additionally performs the point part of FullSystem::doStepFromBackup (FullSystemOptimize.cpp:L264-272):
 * idepth = idepth_backup + step, idepth_zero likewise (DM-VIO), on the device copy; sums[0] = sum step^2, sums[1] = sum |idepth_backup|, sums[2] = npts. */
int dmv_ba_resubstitute(dmv_ba* ba, const double* x, float* step_out, int apply, double sums[3]);
/* FullSystem::backupState / loadSateBackup for the point depths held on the device (FullSystemOptimize.cpp:L322-388) */
int dmv_ba_backup_points(dmv_ba* ba);
int dmv_ba_restore_points(dmv_ba* ba);
int dmv_ba_get_idepth(dmv_ba* ba, float* idepth, float* idepth_zero);

/* Fused GN iteration (one host<->device round trip): resubstitute(x) + point step + set_state + linearize.
 * x may be NULL (first linearisation).  Equivalent to dmv_ba_resubstitute(x, apply=1) ; dmv_ba_set_state(st) ; dmv_ba_linearize(). */
int dmv_ba_gn_step(dmv_ba* ba, const double* x, const dmv_ba_state* st, dmv_ba_lin_result* out, double sums[3]);

/* Point activation: FullSystem::optimizeImmaturePoint (FullSystem/FullSystemOptPoint.cpp:L51-205) with ImmaturePoint::linearizeResidual
 * (FullSystem/ImmaturePoint.cpp:L498-565) for n immature points against every other keyframe of the window, as
 * FullSystem::activatePointsMT_Reductor does (FullSystem.cpp:L586-602).  Uses the frames, calibration and PRE_aff_mode of the last
 * dmv_ba_set_state / dmv_ba_gn_step.  RT: nf*nf*12 floats, index h*nf+t: PRE_RTll (row-major) | PRE_tTll of FrameFramePrecalc (current state).
 * out: status 1 = activate (the caller creates the PointHessian with idepth and one residual per res_state == 0), 0 = not well
 * constrained (keep as immature point), -1 = outlier (delete); idepth = optimised inverse depth; res_state[i*nf+f]: 0 IN, 1 OOB, 2 OUTLIER,
 * 255 = no residual.  Bit-identical to the CPU code (see dmv_ct_trace_points). */
typedef struct dmv_ba_activate_args {
  int n;
  const int32_t* host;
  const float *u, *v, *color8, *weights8, *energyTH, *idepth_min, *idepth_max;
  const float* RT;
  int minObs;               /* 1 in activatePointsMT_Reductor */
  int32_t* status;
  float* idepth;
  int32_t* res_state;
} dmv_ba_activate_args;
int dmv_ba_activate_points(dmv_ba* ba, const dmv_ba_activate_args* a);

/* Which immature points to activate: the part of FullSystem::activatePointsMT (FullSystem.cpp:L642-717) from coarseDistanceMap->makeK up to,
 * not including, activatePointsMT_Reductor.  CoarseDistanceMap::makeDistanceMap (CoarseTracker.cpp:L931-967) projects the active points into
 * the newest frame at pyramid level 1 and grows the distance map over (w/2) x (h/2) cells (growDistBFS, L979-1073); then the immature points of
 * every other frame are deleted, kept, or accepted by the map, each accepted point flooding the map again (addIntoDistFinal, L1076-1082).
 * All arrays are the caller's host memory.  Active points: any order; those hosted by the newest frame are skipped, as the reference skips
 * that frame.  Immature points: grouped by host frame in frame order, host->immaturePoints order inside a group (imm_offset[f] .. imm_offset[f+1]);
 * the newest frame's group is skipped (action keep).  tables12: per frame [KRKi 9 row-major | Kt 3], computed in float as the reference does:
 * K[1] * R * Ki[0] and K[1] * t of newest->PRE_worldToCam * host->PRE_camToWorld.  lastTraceStatus: ImmaturePointStatus (dmv_ip_points).
 * Results are BIT-IDENTICAL to the reference's CPU code.  No BA state is read or changed; only the handle's device, stream and image size
 * are used.  Scratch (8 bytes per level-1 cell, 52 per immature point and 16 per active point, on the device and again in pinned host
 * memory) is allocated on first use and grown when a call needs more.  Returns after one synchronisation.
 * Errors: DMV_ERR_INVALID for bad arguments, or more accepted points than cap (*n_opt = the count needed; action is still written);
 * DMV_ERR_CUDA. */
enum { DMV_ACT_KEEP = 0, DMV_ACT_DELETE = 1, DMV_ACT_OPTIMIZE = 2 };
typedef struct dmv_ba_select_args {
  int nf;                       /* frames of the window (1 .. DMV_MAX_FRAMES) */
  int newest;                   /* index of frameHessians.back() */
  const float* tables12;        /* nf * 12 */
  const uint8_t* flagged;       /* nf: FrameHessian::flaggedForMarginalization */
  int n_active;
  const float *act_u, *act_v, *act_idepth_scaled;
  const int32_t* act_host;
  const int32_t* imm_offset;    /* nf + 1, imm_offset[0] = 0 */
  const float *u, *v, *idepth_min, *idepth_max;
  const int32_t* lastTraceStatus;
  const float *lastTracePixelInterval, *quality, *my_type;
  float currentMinActDist;      /* as FullSystem::activatePointsMT leaves it after its update from ef->nPoints (L607-629) */
  float minTraceQuality;        /* setting_minTraceQuality = 3 */
  int cap;                      /* capacity of opt_idx */
  int* n_opt;                   /* out: size of toOptimize (on overflow the count needed) */
  int32_t* action;              /* out, imm_offset[nf] entries: DMV_ACT_KEEP / DMV_ACT_DELETE / DMV_ACT_OPTIMIZE */
  int32_t* opt_idx;             /* out: indexes of the accepted points in toOptimize order */
  float* map;                   /* optional ((w/2)*(h/2)): fwdWarpedIDDistFinal after the loop */
  int* stats;                   /* optional out [3]: candidates the map before the loop could not decide (the only ones whose decision
                                   waits for earlier floods), floods run (floods no later decision needs are skipped unless map is
                                   requested), rounds of the chain (its serial depth) */
} dmv_ba_select_args;
int dmv_ba_select_activation(dmv_ba* ba, const dmv_ba_select_args* a);

/* PointFrameResidual::resetOOB for every residual of the window, as FullSystem::optimize does when it collects activeResiduals
 * (FullSystem/FullSystemOptimize.cpp:L431-448; FullSystem/Residuals.h:L91-98): state IN, energy 0.  Discards the tentative and the committed
 * linearisation (the next dmv_ba_linearize / dmv_ba_gn_step starts from these states). */
int dmv_ba_reset_oob(dmv_ba* ba);

/* Residuals leave the window: the deletion loop of FullSystem::linearizeAll(fixLinearization = true) (FullSystem/FullSystemOptimize.cpp:L196-214 ->
 * EnergyFunctional::dropResidual, OptimizationBackend/EnergyFunctional.cpp:L500-520) for residuals that did not end up IN.  res_idx: indices in
 * the current dmv_ba_set_residuals order; the remaining residuals keep their relative order (per-residual outputs shrink accordingly).  The
 * committed linearisation stays valid (a non-active residual contributes nothing to it). */
int dmv_ba_drop_residuals(dmv_ba* ba, int n, const int32_t* res_idx);

/* Point marginalisation at keyframe creation, one launch pair for the whole flagged set:
 *   - the compute of FullSystem::flagPointsForRemoval for each flagged point (FullSystem/FullSystem.cpp:L826-838): PointFrameResidual::resetOOB,
 *     linearize, applyRes(true), EFResidual::fixLinearizationF (OptimizationBackend/EnergyFunctionalStructs.cpp:L88-114) -> res_toZeroF;
 *   - EnergyFunctional::marginalizePointsF (OptimizationBackend/EnergyFunctional.cpp:L678-742): priorF *= idepthFixPriorMargFac,
 *     AccumulatedTopHessian::addPoint<2>, AccumulatedSCHessian::addPoint(p, shiftPriorToZero = false), stitch without priors.
 * The caller decides WHICH points (PointHessian::isOOB / isInlierNew / idepth_hessian > setting_minIdepthH_marg are host bookkeeping) and finishes
 * with HM += setting_margWeightFac * (M - Msc), bM += setting_margWeightFac * (Mb - Mbsc), then re-uploads the window without the points.
 * Uses the frames / calibration / depths of the last dmv_ba_set_state or dmv_ba_gn_step.  adHTdeltaF: nf*nf*8 floats, entry [h + t*nf]
 * (EnergyFunctional::setDeltaF, EnergyFunctional.cpp:L175-198); cDeltaF: calibration value - value_zero.  Any output may be NULL.
 * M/Msc: N*N row-major, N = 8 nf + 4.  res_toZeroF [nres*8] / isLinearized [nres] follow the dmv_ba_set_residuals order (zero for residuals
 * that were not linearised); ngoodRes [n] follows `point`.  Invalidates the tentative linearisation; the committed one is untouched.
 * Sharded handles (dmv_ba_comm_init / dmv_ba_p2p_import): not supported, returns DMV_ERR_STATE (marginalise per rank and sum on the host). */
typedef struct dmv_ba_marg_args {
  int32_t n;
  const int32_t* point;          /* [n] indices in dmv_ba_set_points order */
  const float* adHTdeltaF;
  float cDeltaF[4];
  float idepthFixPriorMargFac;   /* 600*600 (util/settings.cpp:L68) */
  double *M, *Mb, *Msc, *Mbsc;
  int32_t* resInM;
  int32_t* ngoodRes;
  float* res_toZeroF;
  uint8_t* isLinearized;
} dmv_ba_marg_args;
int dmv_ba_marginalize_points(dmv_ba* ba, const dmv_ba_marg_args* a);

/* Multi-GPU (SURVEY.md §8e): points are sharded over ranks, images/tables replicated.  After dmv_ba_comm_init every
 * dmv_ba_linearize / dmv_ba_gn_step / dmv_ba_marginalize_points all-reduces the system (and energy / counters) over NCCL so that all ranks
 * hold identical H,b; every rank must make the same sequence of these calls (dmv_ba_marginalize_points with its own flagged points, possibly none).
 * nccl_unique_id: 128 bytes from ncclGetUniqueId() on rank 0, distributed by the caller. */
int dmv_nccl_unique_id(void* id128);
int dmv_ba_comm_init(dmv_ba* ba, int nranks, int rank, const void* nccl_unique_id);

/* The same exchange without NCCL, over NVLink/NVSwitch peer memory (CUDA IPC, one process per GPU of one node, <= 8 ranks):
 * every rank exports its inbox (64-byte cudaIpcMemHandle_t), the caller all-gathers the handles (any transport: MPI,
 * torch.distributed, a file) and every rank imports all of them.  From then on the all-reduce happens INSIDE THE LINEARISATION KERNEL:
 * the lanes that produce a result entry push it to every peer as a 16-byte flag-carrying packet, later wait (bounded: DMV_ERR_TIMEOUT) for the
 * peers' packets of the same entry and add them in rank order (bit-identical H,b on all ranks; no extra launch, no fence round trip).
 * Takes precedence over a NCCL communicator if both are set; nranks = 1 in dmv_ba_p2p_import switches it off again.
 * No reference counterpart (the reference is single-node CPU). */
int dmv_ba_p2p_export(dmv_ba* ba, void* ipc_handle64);
int dmv_ba_p2p_import(dmv_ba* ba, int nranks, int rank, const void* ipc_handles /* nranks*64 bytes, rank order */);

/* ---- batched windows (SURVEY.md section 8d "batched variant"): B independent windows, each an ordinary BA handle on the same device with
 * the same chunk_points, linearised by ONE launch.  No reference counterpart (FullSystem::optimize handles one window); per window the
 * results are bit-identical to dmv_ba_gn_step on that handle. */
typedef struct dmv_ba_batch dmv_ba_batch;
int dmv_ba_batch_create(dmv_ba* const* handles, int n, dmv_ba_batch** out);   /* n <= 64; the handles stay owned by the caller */
/* A handle may appear only once in a batch: a duplicate is refused with DMV_ERR_INVALID, naming both positions. */
int dmv_ba_batch_destroy(dmv_ba_batch* batch);
/* dmv_ba_gn_step on every handle: x[i] may be NULL (x itself may be NULL), st[i] as for dmv_ba_gn_step; out (n entries) and sums3 (3 n doubles)
 * may be NULL.  Afterwards: dmv_ba_apply_res / dmv_ba_accumulate / ... per handle as usual.  Every member is checked before any is staged:
 * a refused call uploads nothing and leaves every handle as it was. */
int dmv_ba_batch_gn_step(dmv_ba_batch* batch, const double* const* x, const dmv_ba_state* const* st, dmv_ba_lin_result* out, double* sums3);
int dmv_ba_batch_set_timing(dmv_ba_batch* batch, int enable);
int dmv_ba_batch_last_kernel_ms(dmv_ba_batch* batch, float* ms);   /* CUDA-event time of the last batched launch (after set_timing(1)) */

/* instrumentation (cheap, always present): CUDA-event timing of the last linearize / gn_step on the handle's stream, milliseconds:
 * [0] = total device time of the call, [1] = ba_fused_kernel, [2] = 0, [3] = what follows the kernel (NCCL all-reduce / D2H copy) */
int dmv_ba_last_timing(dmv_ba* ba, float ms[4]);
int dmv_ba_kernel_launch_count(dmv_ba* ba, long long* n);
/* enable/disable the CUDA-event timing of dmv_ba_linearize / dmv_ba_gn_step (off by default) */
int dmv_ba_set_timing(dmv_ba* ba, int enable);
/* bytes copied host->device and device->host by one dmv_ba_gn_step / dmv_ba_linearize call */
int dmv_ba_io_bytes(dmv_ba* ba, long long* h2d, long long* d2h);
/* The measurement-only entry points (dmv_ba_bench_device, dmv_ba_bench_e2e, ...) live in dmvio_b200_bench.h / csrc/ba_bench.cu and
 * are compiled in only with BENCH=1. */

/* ------------------------------------------------------------------------------------------------
 * Coarse-tracker handle  ==  the GPU side of CoarseTracker (FullSystem/CoarseTracker.{h,cpp})
 * ------------------------------------------------------------------------------------------------ */
typedef struct dmv_ct dmv_ct;
typedef struct dmv_ct_config {
  int w, h;
  int levels;      /* pyrLevelsUsed */
  int max_points;  /* capacity of pc_* per level */
  int device;
} dmv_ct_config;

int dmv_ct_create(const dmv_ct_config* cfg, dmv_ct** out);
int dmv_ct_destroy(dmv_ct* ct);
/* CoarseTracker::makeK (CoarseTracker.cpp:L105-134): per-level intrinsics */
int dmv_ct_set_K(dmv_ct* ct, int level, float fx, float fy, float cx, float cy);
/* pc_u/pc_v/pc_idepth/pc_color of one level (result of makeCoarseDepthL0, CoarseTracker.cpp:L249-293) */
int dmv_ct_set_ref(dmv_ct* ct, int level, int n, const float* pc_u, const float* pc_v, const float* pc_idepth, const float* pc_color);
/* CoarseTracker::setCoarseTrackingRef -> makeCoarseDepthL0 (CoarseTracker.cpp:L138-295, L524-538) on the device: builds pc_* of EVERY level from the
 * keyframe's IN residuals that target it: per residual centerProjectedTo = (Ku, Kv, new_idepth) and its point's HdiF (CoarseTracker.cpp:L148-158).
 * The reference frame (lastRef->dIp) is the frame currently resident in the handle (upload it first with dmv_ct_upload_new_image /
 * dmv_ct_upload_new of every level); afterwards a new frame may be uploaded for tracking.  pc_n_out (levels entries, may be NULL) = pc_n[].
 * Bit-identical lists (values and order) to the CPU code. */
int dmv_ct_make_coarse_depth(dmv_ct* ct, int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, int32_t* pc_n_out);
/* CoarseTracker::setCoarseTrackingRef (CoarseTracker.cpp:L524-538) + makeCoarseDepthL0 (L138-295) fed directly from a BA handle on the same
 * device, nothing crossing PCIe: the reference keyframe is the newest frame of the BA window (frame nf-1 of dmv_ba_set_window).
 *   - points: a point contributes exactly when its residual into that frame is still present (not removed by dmv_ba_drop_residuals) and
 *     ended the committed linearisation IN — ph->lastResiduals[0] IN after the tail's linearizeAll(true) (FullSystemOptimize.cpp:L175-203);
 *     its committed centerProjectedTo and the HdiF of the last dmv_ba_accumulate (dmv_ba_get_solve_HdiF) are used;
 *   - order: colliding splats are folded in makeCoarseDepthL0's order (CoarseTracker.cpp:L144-146): the frameHessians x fh->pointHessians
 *     order of the last dmv_ba_set_points, after FullSystem::removeOutliers (FullSystemOptimize.cpp:L680-697), which makeKeyFrame runs just
 *     before (FullSystem.cpp:L1438): in each host frame a point left without residuals is replaced by the host's last point (swap-with-back).
 *     The call applies that reorder itself; the handle must not have been re-uploaded since the tail;
 *   - frame: the BA slot's level-0 plane becomes the handle's level 0 and the coarser levels are built as dmv_ct_upload_new_image builds them,
 *     so afterwards the keyframe is the handle's resident frame, as after dmv_ct_upload_new_image + dmv_ct_make_coarse_depth.
 * Ordered behind everything queued on the BA handle (no host synchronisation needed in between); returns after one synchronisation.
 * pc_n_out as dmv_ct_make_coarse_depth.  Bit-identical lists (values and order) to dmv_ct_make_coarse_depth fed with the same residuals.
 * Errors: DMV_ERR_INVALID for handles on different devices, different image sizes, or a projection outside the image (the lowest such point
 * is reported; every level's list is then emptied); the capacity error of dmv_ct_make_coarse_depth; DMV_ERR_STATE without a committed
 * linearisation, without a dmv_ba_accumulate since dmv_ba_set_points, or on a sharded handle (its points are one rank's share: build the
 * reference on the host from the gathered outputs there). */
int dmv_ct_set_ref_from_ba(dmv_ct* ct, dmv_ba* ba, int32_t* pc_n_out);
/* download pc_u / pc_v / pc_idepth / pc_color of one level (any pointer may be NULL; *n = pc_n[level]) */
int dmv_ct_get_ref(dmv_ct* ct, int level, int* n, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color);
/* newFrame->dIp[level] (w_l*h_l*3 floats AoS) */
int dmv_ct_upload_new(dmv_ct* ct, int level, const float* dIp_aos3);
/* builds the whole pyramid of the new frame on the device from the raw image (FrameHessian::makeImages) */
int dmv_ct_upload_new_image(dmv_ct* ct, const float* image_wh);
/* settings read by calcRes: setting_huberTH */
int dmv_ct_set_huber(dmv_ct* ct, float huberTH);

/* Raw-frame ingest == the per-frame part of Undistort::undistort<T> (util/Undistort.cpp:L385-482) with
 * PhotometricUndistorter::processFrame (L213-252) on the device.  The tables are built once per sequence on the host, as the
 * reference builds them (camera model, makeOptimalK_*, G, vignetteMapInv), and uploaded by dmv_ct_set_undistort.
 *   remapX / remapY: w*h each (w, h = the handle's level 0); x < 0 marks a pixel outside the raw image (output 0), every other
 *                    entry must satisfy 0 <= x < wOrg-1 and 0 <= y < hOrg-1.  Both NULL = passthrough (requires wOrg = w, hOrg = h).
 *   G / nG:          the response map as PhotometricUndistorter holds it (256 <= nG <= 65536), or NULL = no photometric calibration.
 *                    A raw upload that applies G (exposure > 0, photometric_mode != 0) needs nG >= 256 (8-bit) / 65536 (16-bit).
 *   vignetteInv:     wOrg*hOrg (vignetteMapInv), required with photometric_mode 2 and G; may be NULL otherwise.
 *   photometric_mode = setting_photometricCalibration (0, 1, 2).
 * The benchmark-only distortions (benchmark_varNoise, benchmark_varBlurNoise) are not supported. */
typedef struct dmv_undistort_config {
  int wOrg, hOrg;
  const float* remapX;
  const float* remapY;
  const float* G;
  int nG;
  const float* vignetteInv;
  int photometric_mode;
} dmv_undistort_config;
int dmv_ct_set_undistort(dmv_ct* ct, const dmv_undistort_config* cfg);
/* One raw frame (wOrg*hOrg pixels of bytes_per_px = 1 (uint8) or 2 (uint16)) -> the level-0 intensity plane, then the whole pyramid, like
 * dmv_ct_upload_new_image with the image Undistort::undistort<T>(raw, exposure, 0, factor) returns; bit-identical.  factor multiplies the raw
 * value when the photometric map is off (no G, exposure <= 0 or photometric_mode 0): 1 for 8-bit, 1/256 as the reference's 16-bit reader.
 * Asynchronous like dmv_ct_upload_new_image (the frame goes through the handle's pinned staging buffer). */
int dmv_ct_upload_raw_image(dmv_ct* ct, const void* raw, int bytes_per_px, float exposure, float factor);
/* read-back of the resident frame's dIp[level] (w_l*h_l*3 floats AoS: I, dx, dy), e.g. for pixel selection on keyframes */
int dmv_ct_download_frame(dmv_ct* ct, int level, float* dIp_aos3);

/* CoarseTracker::calcRes (L361-517) fused with calcGSSSE (L299-356) for one pose:
 *   RKi = R * Ki[lvl] (row-major 3x3 float), t (3), affLL = AffLight::fromToVecExposure(...) (2),
 *   a_gs = affLL[0] (first argument `a` of calcGSSSE), b0 = lastRef_aff_g2l.b, cutoffTH.
 * out: res6 = Vec6 of calcRes; if want_gs: H (8x8 row-major) and b (8) exactly as calcGSSSE returns them
 * (divided by the 4-padded warped count, SCALE_* applied); n_warped = buf_warped_n (padded). */
int dmv_ct_calc_res_gs(dmv_ct* ct, int level, const float RKi[9], const float t[3], const float affLL[2], float b0, float cutoffTH,
                       int want_gs, double res6[6], double H[64], double b[8], int* n_warped);
/* CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:L539-770, visual-only branch L639-683) as ONE persistent launch: the whole
 * Levenberg-Marquardt loop over the pyramid levels (calcRes + calcGSSSE per evaluation, 8x8 LDLT, SE3 update, accept/reject, cutoff
 * doubling, level repeat) runs on the device; the host gets the tracked pose back.  Same semantics as driving dmv_ct_calc_res_gs from the
 * host loop: R,t = lastToNew_out (refToNew, row-major), a,b = aff_g2l_out; on an aborted track (NaN residual or > 1.5*minResForAbort)
 * trackingGood = 0, status = 2 and R,t,a,b are returned unchanged, like the reference's early `return false`.
 * Runs on one thread-block cluster (16, 8 or 4 CTAs, probed once per handle), which tracks any number of reference points.  On a device
 * that cannot schedule such a cluster (or encode the TMA tensor maps of the level planes) it returns DMV_ERR_INVALID on every call;
 * drive dmv_ct_calc_res_gs from a host LM loop there.
 * Test hook: DMV_CT_CLUSTER=16|8|4 (read at the probe) allows only that cluster size; dmv_ct_track returns an error when it cannot be
 * scheduled. */
typedef struct dmv_ct_track_args {
  double R[9], t[3];          /* in: initial refToNew */
  double a, b;                /* in: initial aff_g2l of the new frame */
  double ref_a, ref_b;        /* lastRef_aff_g2l */
  float ref_exposure, new_exposure; /* lastRef->ab_exposure, newFrame->ab_exposure */
  float coarseCutoffTH;       /* setting_coarseCutoffTH = 20 */
  float affineOptModeA, affineOptModeB;
  int coarsestLvl;
  double minResForAbort[5];   /* NaN = never abort */
} dmv_ct_track_args;
typedef struct dmv_ct_track_result {
  double R[9], t[3], a, b;
  double lastResiduals[5];    /* CoarseTracker::lastResiduals */
  double flowIndicators[3];   /* CoarseTracker::lastFlowIndicators */
  int trackingGood, iterations, evaluations, status;
} dmv_ct_track_result;
int dmv_ct_track(dmv_ct* ct, const dmv_ct_track_args* in, dmv_ct_track_result* out);
/* dmv_ct_track for n independent handles (several cameras or robots served by one host thread) in ONE launch: one thread-block cluster per
 * handle, so up to n frames are tracked side by side instead of one after the other on 16 SMs each.  Stateless: the handles' descriptors
 * travel as kernel parameters; pass whichever handles have a frame ready, in any order.
 * out[i] is bit-identical to what dmv_ct_track(handles[i], &in[i], &out[i]) returns (aborts included), and afterwards
 * dmv_ct_last_point_evaluations and dmv_ct_kernel_launch_count (+1) of every handle read as after that call.  The launch is ordered behind
 * the work queued on every handle's stream (asynchronous uploads included); the call returns after one synchronisation, with every
 * handle's staging buffer free.  dmv_ct_set_timing / dmv_ct_last_timing are not involved.
 * Errors, all before anything is launched or any out[i] is written: DMV_ERR_INVALID for n outside 1..DMV_CT_TRACK_MANY_MAX, a NULL pointer,
 * a handle passed twice, handles on different devices, or handles whose probed cluster sizes differ (a handle probes on its first track;
 * the message names two such handles); and dmv_ct_track's own errors for any member, with the member's index in the message. */
#define DMV_CT_TRACK_MANY_MAX 16
int dmv_ct_track_many(dmv_ct* const* handles, int n, const dmv_ct_track_args* in, dmv_ct_track_result* out);
/* The motion-hypothesis loop of FullSystem::trackNewCoarse (FullSystem.cpp:L412-506, visual-only: setting_useIMU false) in ONE launch: the
 * tries lastF_2_fh_tries (built by the caller, L364-402) tracked with trackNewestCoarse one after the other, each with the best residuals
 * so far (achievedRes) as its minResForAbort, until the first try whose achievedRes[0] < lastCoarseRMSE0 * reTrackThreshold.
 * Every field of out is bit-identical to that loop run with one dmv_ct_track per try on this handle: the winner test
 * (L467), the take-over of achievedRes with its NaN rules (L476-483), the break (L486), the fallback when no try is good (L491-497: try 0's
 * pose, (a, b) and zero flow) and CoarseTracker's lastResiduals / lastFlowIndicators after the last try the loop ran (lastResiduals is
 * reset to NaN at the start of every try, CoarseTracker.cpp:L551).
 * The tries run one after the other on one thread-block cluster of the handle's probed size, with the loop's bookkeeping on the device
 * between them; tries_started equals tries, and dmv_ct_last_point_evaluations afterwards reports the sum over the tries the loop ran.
 * Ordered on the handle's stream behind queued uploads; one synchronisation; dmv_ct_kernel_launch_count + 1.  The handle's frame,
 * reference and probed cluster size are unchanged, and a later dmv_ct_track behaves as before.  One pinned result (264 bytes) is allocated
 * on first use.
 * Errors, all before anything is launched and with out untouched: DMV_ERR_INVALID for n outside 1..DMV_CT_MAX_TRIES, a NULL pointer, and
 * dmv_ct_track's own errors (coarsestLvl out of range, missing intrinsics, a cluster size the device cannot schedule). */
#define DMV_CT_MAX_TRIES 32
typedef struct dmv_ct_tries_args {
  int n;                         /* 1..DMV_CT_MAX_TRIES, in lastF_2_fh_tries order */
  const double* R;               /* n*9 row-major refToNew per try */
  const double* t;               /* n*3 */
  double a, b;                   /* aff_last_2_l: initial aff_g2l of every try */
  double ref_a, ref_b;           /* lastRef_aff_g2l */
  float ref_exposure, new_exposure, coarseCutoffTH, affineOptModeA, affineOptModeB;   /* as dmv_ct_track_args */
  int coarsestLvl;               /* pyrLevelsUsed-1 in the reference */
  double lastCoarseRMSE0;        /* FullSystem::lastCoarseRMSE[0] (100 at construction) */
  float reTrackThreshold;        /* setting_reTrackThreshold = 1.5 */
} dmv_ct_tries_args;
typedef struct dmv_ct_tries_result {
  double R[9], t[3], a, b;       /* lastF_2_fh, aff_g2l: the winner's, else try 0's input pose and (a, b) */
  double achievedRes[5];         /* becomes lastCoarseRMSE */
  double flowVecs[3];            /* the winner's lastFlowIndicators, else 0 0 0 */
  double lastResiduals[5], flowIndicators[3];  /* CoarseTracker state after the last try the loop ran */
  int trackingGood;              /* trackingGoodRet */
  int haveOneGood, winner;       /* winner = index of the try taken, -1 if none */
  int tries;                     /* tryIterations: tries the sequential loop runs */
  int tries_started;             /* tries the device began (= tries: they run in order) */
} dmv_ct_tries_result;
int dmv_ct_track_tries(dmv_ct* ct, const dmv_ct_tries_args* in, dmv_ct_tries_result* out);
/* dmv_ct_track_tries for n independent handles (several visual-only camera streams served by one host thread) in ONE launch: one
 * thread-block cluster per handle runs that handle's try loop, and the clusters retire independently, so a frame that needs many tries
 * delays only its own member.  in[i] may differ from member to member in every field (n, coarsestLvl, lastCoarseRMSE0, exposures, affine
 * state), and the handles in image size and level count, as long as their probed cluster sizes match.
 * out[i] is bit-identical to what dmv_ct_track_tries(handles[i], &in[i], &out[i]) returns, and afterwards dmv_ct_last_point_evaluations
 * and dmv_ct_kernel_launch_count (+1) of every handle read as after that call.  Each handle's frame, reference and probed cluster size are
 * unchanged.  The launch goes on handles[0]'s stream, ordered behind the work queued on every handle's stream (asynchronous uploads
 * included); the call returns after one synchronisation, with every handle's staging buffer free.  With n > 1 each handle holds its try
 * table in a pinned block of 3 KB, allocated on first use beside dmv_ct_track_tries's result.
 * Errors, all before anything is launched or any out[i] is written, and with every launch count unchanged: those of dmv_ct_track_many
 * (n outside 1..DMV_CT_TRACK_MANY_MAX, a NULL pointer, a handle passed twice, handles on different devices or with different cluster sizes)
 * and dmv_ct_track_tries's own errors for any member, with the member's index in the message ("handles[3]: ..."). */
int dmv_ct_track_tries_many(dmv_ct* const* handles, int n, const dmv_ct_tries_args* in, dmv_ct_tries_result* out);

/* ------------------------------------------------------------------------------------------------
 * Immature-point tracing  ==  ImmaturePoint::traceOn (FullSystem/ImmaturePoint.cpp:L77-437) for all immature points of ONE host
 * frame against the newest frame, i.e. one iteration of the host loop of FullSystem::traceNewCoarse (FullSystem.cpp:L554-575).
 * Runs on the coarse-tracker handle: the frame traced against is the one last given to dmv_ct_upload_new_image / dmv_ct_upload_new
 * (level 0), which is resident there anyway.  Results are BIT-IDENTICAL to the reference's CPU code (the kernel is compiled without
 * FMA contraction and keeps the reference's operation order).
 * ------------------------------------------------------------------------------------------------ */
typedef struct dmv_ip_settings {   /* util/settings.cpp:L79, L178-187 */
  float maxPixSearch;              /* setting_maxPixSearch = 0.027 */
  float trace_stepsize;            /* 1.0 */
  float trace_GNThreshold;         /* 0.1 */
  float trace_extraSlackOnTH;      /* 1.2 */
  float trace_slackInterval;       /* 1.5 */
  float trace_minImprovementFactor;/* 2 */
  float huberTH;                   /* setting_huberTH = 9 */
  int trace_GNIterations;          /* 3 */
  int minTraceTestRadius;          /* 2 */
} dmv_ip_settings;
void dmv_ip_default_settings(dmv_ip_settings* s);
/* ImmaturePoint fields (ImmaturePoint.h:L56-90), structure of arrays over the n points of one host frame.
 * in: u, v, color[8], weights[8], gradH (Mat22f row-major), energyTH.   in/out: idepth_min, idepth_max, quality,
 * lastTraceStatus (ImmaturePointStatus: 0 GOOD, 1 OOB, 2 OUTLIER, 3 SKIPPED, 4 BADCONDITION, 5 UNINITIALIZED), lastTraceUV, lastTracePixelInterval. */
typedef struct dmv_ip_points {
  int n;
  const float *u, *v, *color8, *weights8, *gradH4, *energyTH;
  float *idepth_min, *idepth_max, *quality;
  int32_t* lastTraceStatus;
  float *lastTraceUV2, *lastTracePixelInterval;
} dmv_ip_points;
/* ImmaturePoint::ImmaturePoint (ImmaturePoint.cpp:L34-63) for n integer pixels (u, v) of the frame resident in the handle (the frame that
 * just became a keyframe, FullSystem::makeNewTraces, FullSystem.cpp:L1284-1330): pattern colours, weights (setting_outlierTHSumComponent = 50*50),
 * gradH (row-major 2x2), energyTH (= 8 * setting_outlierTH * setting_overallEnergyTHWeight^2 = 1152); ok[i] = 0 where a colour is not finite
 * (energyTH = NaN, the caller drops the point like the reference).  Bit-identical to the CPU code. */
int dmv_ct_init_points(dmv_ct* ct, int n, const int32_t* u, const int32_t* v, float* color8, float* weights8, float* gradH4, float* energyTH, int32_t* ok);
/* hostToFrame_KRKi (row-major 3x3), hostToFrame_Kt, hostToFrame_affine exactly as traceNewCoarse computes them (FullSystem.cpp:L557-561).
 * settings may be NULL (defaults). */
int dmv_ct_trace_points(dmv_ct* ct, const dmv_ip_points* pts, const float KRKi[9], const float Kt[3], const float aff[2], const dmv_ip_settings* settings);
/* The same for the immature points of SEVERAL host keyframes at once (the whole loop of FullSystem::traceNewCoarse, FullSystem.cpp:L554-575):
 * sets[k] = the points hosted by keyframe k, tables14 = per host [KRKi 9 | Kt 3 | aff 2]; one upload, one launch, one download. */
int dmv_ct_trace_points_multi(dmv_ct* ct, int nsets, const dmv_ip_points* sets, const float* tables14, const dmv_ip_settings* settings);
/* dmv_ct_trace_points_multi for n independent handles (several cameras or robots served by one host thread, each after its tracked frame)
 * in ONE launch.  jobs[i] holds exactly the arguments dmv_ct_trace_points_multi takes for handles[i].
 * Result: for every i, jobs[i]'s in/out arrays end bit-identical to what dmv_ct_trace_points_multi(handles[i], jobs[i].nsets, jobs[i].sets,
 * jobs[i].tables14, settings) leaves; each member traces against its own resident level-0 frame, at its own image size.
 * Launch count: each member's dmv_ct_kernel_launch_count reads as after that call (+1 if the member has at least one point, +0 otherwise);
 * a call in which no member has a point launches nothing.
 * Settings: one for the call, as DSO's settings are process-global; NULL means defaults.
 * Ordering: the launch is ordered behind the work queued on every member's stream (asynchronous dmv_ct_upload_new_image /
 * dmv_ct_upload_raw_image included); the call returns after one synchronisation, with every member's staging buffer free.
 * Errors, all before any allocation, copy or launch and before any output is written: DMV_ERR_INVALID for n outside
 * 1..DMV_CT_TRACE_MANY_MAX, a NULL handles / jobs, a NULL member, a handle passed twice (the message names both positions) or handles on
 * different devices; and, for each member, the errors dmv_ct_trace_points_multi reports for its arguments, prefixed "handles[i]: ".  A
 * member is accepted exactly when dmv_ct_trace_points_multi would accept it. */
#define DMV_CT_TRACE_MANY_MAX 16
typedef struct dmv_ct_trace_job {
  int nsets;                   /* host keyframes of this handle's window, as dmv_ct_trace_points_multi */
  const dmv_ip_points* sets;   /* in/out exactly as dmv_ct_trace_points_multi */
  const float* tables14;       /* nsets * 14: KRKi 9 | Kt 3 | aff 2 per host */
} dmv_ct_trace_job;
int dmv_ct_trace_many(dmv_ct* const* handles, int n, const dmv_ct_trace_job* jobs, const dmv_ip_settings* settings);

/* Immature-point store: a window's immature points kept on one device between frames, so that traceNewCoarse after every tracked frame
 * uploads only the 14-float tables of each host keyframe and downloads nothing.  Slot k holds the points hosted by one keyframe
 * (FrameHessian::immaturePoints), in that list's order.  A store belongs to no tracker handle: it can be traced against either of
 * FullSystem's two coarse trackers, which swap roles at every keyframe.
 * Results: any sequence of dmv_ct_trace_store calls between a put and a get leaves the slot's in/out fields bit-identical to the same
 * sequence of dmv_ct_trace_points_multi calls on host arrays with sets[k] = slot k, the same tables and the same frames.
 * Every call checks all its arguments before any allocation, copy or launch (a refused call leaves the store unchanged) and returns after
 * one synchronisation.  The caller serialises the calls on one store (the reference holds mapMutex over traceNewCoarse and activatePointsMT).
 * Device memory: 31 words per point in two buffers, grown on demand with their contents kept. */
typedef struct dmv_ip_store dmv_ip_store;
#define DMV_IP_STORE_SLOTS 64        /* = the per-call limit of host frames of dmv_ct_trace_points_multi */
int dmv_ip_store_create(int device, dmv_ip_store** out);
int dmv_ip_store_destroy(dmv_ip_store* s);
/* replaces the slot's points by pts (every field, read-only and in/out); pts->n == 0 empties the slot */
int dmv_ip_store_put(dmv_ip_store* s, int slot, const dmv_ip_points* pts);
/* downloads the 7 in/out words of the slot's points (idepth_min, idepth_max, quality, lastTraceStatus, lastTraceUV2, lastTracePixelInterval);
 * the read-only pointers of pts are not used.  pts->n must equal the slot's count (the error message gives it). */
int dmv_ip_store_get(dmv_ip_store* s, int slot, dmv_ip_points* pts);
/* removes the slot's points idx[0..n) (indices into the slot's current order, distinct) with activatePointsMT's swap-with-back loop
 * (FullSystem.cpp:L761-769): the slot's order afterwards is the host's immaturePoints order after that loop.  order_out (optional, one
 * entry per survivor) = each survivor's index before the call, so the caller can reorder its own copies of the read-only fields. */
int dmv_ip_store_remove(dmv_ip_store* s, int slot, int n, const int32_t* idx, int32_t* order_out);
/* traceNewCoarse over the store: the points of slot k traced with tables14[14k .. 14k + 14) (KRKi 9 | Kt 3 | aff 2, as
 * dmv_ct_trace_points_multi) against ct's resident level-0 frame.  Slots at or above nslots must be empty; tables14 may be NULL when no
 * slot below nslots holds a point.  One launch on ct's stream (launch count +1) when a point is present, none otherwise; ct's own
 * staging area (dmv_ct_trace_points_multi's) is not used.  Errors: DMV_ERR_INVALID for a NULL ct / s, nslots outside
 * 0..DMV_IP_STORE_SLOTS, a point in a slot at or above nslots, a NULL tables14 with points present, or a store on another device than ct. */
int dmv_ct_trace_store(dmv_ct* ct, dmv_ip_store* s, int nslots, const float* tables14, const dmv_ip_settings* settings);
/* dmv_ct_trace_store for n handles in ONE launch: member i traces jobs[i].store against handles[i]'s frame, bit-identical to
 * dmv_ct_trace_store(handles[i], jobs[i].store, jobs[i].nslots, jobs[i].tables14, settings).  Membership, launch counts and ordering as
 * dmv_ct_trace_many: the launch goes on handles[0]'s stream behind the work queued on every member's stream.  Errors, all before anything
 * is allocated, copied or launched: those of dmv_ct_trace_many's member list, a NULL handles / jobs, a store passed twice, and each member's
 * dmv_ct_trace_store errors prefixed "handles[i]: ". */
typedef struct dmv_ct_trace_store_job {
  dmv_ip_store* store;
  int nslots;
  const float* tables14;       /* nslots * 14 */
} dmv_ct_trace_store_job;
int dmv_ct_trace_store_many(dmv_ct* const* handles, int n, const dmv_ct_trace_store_job* jobs, const dmv_ip_settings* settings);

/* FullSystem::activatePointsMT (FullSystem.cpp:L642-770) from makeDistanceMap through the removal loop, with the window's immature points
 * read from a store: frame f's host->immaturePoints are slot slot[f] (-1: none; slots need not follow frame order).  Bit-identical to
 *   1. dmv_ip_store_get of every slot named by a frame, 2. dmv_ba_select_activation on those points (imm_offset from the slots' counts),
 *   3. dmv_ba_activate_points on its toOptimize, 4. activatePointsMT's choice of the points to drop, 5. dmv_ip_store_remove of every slot:
 * every output, the store's contents and counts, and every later trace of the store.  Removed: action DMV_ACT_DELETE, and toOptimize entries
 * with status 1 or -1, or status 0 and lastTraceStatus IPS_OOB (1); each slot keeps L761-769's order.  Slots no frame names and the newest
 * frame's slot are not touched.  The other arguments are those of dmv_ba_select_activation and dmv_ba_activate_points; my_type[f] is frame
 * f's ImmaturePoint::my_type in its slot's order (the only field the selection reads that the store does not hold).  Reads no BA state but
 * what dmv_ba_activate_points reads (images, calibration, PRE_aff_mode); its launch count moves as dmv_ba_activate_points' does (+1 when
 * toOptimize is not empty).  Three synchronisations.
 * Errors, all before any allocation, copy or launch, with the store unchanged: DMV_ERR_STATE as dmv_ba_activate_points; DMV_ERR_INVALID for a
 * NULL ba / s / a, nf other than the window's, a store on another device, a slot outside -1..DMV_IP_STORE_SLOTS-1 or named twice, a NULL
 * my_type[f] for a frame with points, NULL RT / opt_frame / opt_index / status / idepth / res_state with cap > 0, and every argument
 * dmv_ba_select_activation refuses.  More than cap entries in toOptimize: DMV_ERR_INVALID after the selection with *n_opt = the count
 * needed (action, map and stats written) and nothing removed. */
typedef struct dmv_ba_activate_store_args {
  int nf, newest;                      /* nf = the window's frames */
  const float* tables12;               /* as dmv_ba_select_args */
  const uint8_t* flagged;
  int n_active;
  const float *act_u, *act_v, *act_idepth_scaled;
  const int32_t* act_host;
  const int32_t* slot;                 /* nf */
  const float* const* my_type;         /* nf pointers, count of slot[f] floats each (NULL allowed for a frame without points) */
  float currentMinActDist, minTraceQuality;
  const float* RT;                     /* as dmv_ba_activate_args */
  int minObs;
  int cap;                             /* capacity of opt_frame, opt_index, status, idepth and res_state (nf per entry) */
  int* n_opt;                          /* out: toOptimize's size (on overflow the count needed) */
  int32_t *opt_frame, *opt_index;      /* out: toOptimize as (frame, index in its slot before the call) */
  int32_t* status;                     /* out, per toOptimize entry: as dmv_ba_activate_args */
  float* idepth;
  int32_t* res_state;
  int32_t* order_out;                  /* optional out: each survivor's index before the call, one segment per frame in frame order */
  int32_t* n_kept;                     /* optional out, nf: points left in frame f's slot (the segment lengths of order_out) */
  int32_t* action;                     /* optional out: as dmv_ba_select_args, the frames' points concatenated in frame order */
  float* map;                          /* optional out: as dmv_ba_select_args */
  int* stats;                          /* optional out [3]: as dmv_ba_select_args */
} dmv_ba_activate_store_args;
int dmv_ba_activate_store(dmv_ba* ba, dmv_ip_store* s, const dmv_ba_activate_store_args* a);

/* One change of the window's membership (FullSystem::makeKeyFrame's makeIDX points: a frame joins, activated points are inserted, points
 * and frames leave) made on the window already on the device.  Bit-identical to downloading the state (dmv_ba_get_idepth,
 * dmv_ba_get_residual_outputs) and re-uploading the whole window with dmv_ba_set_window + dmv_ba_set_points + dmv_ba_set_residuals from
 * lists built by these rules:
 *   - carried point (point_src[j] = i >= 0, point i of the current list): host frame remapped through frame_src; u, v, color8, weights8,
 *     priorF, and idepth / idepth_zero as dmv_ba_get_idepth reports them, kept.
 *   - activated point (point_src[j] = -1 - k): entry k of the last dmv_ba_activate_points / dmv_ba_activate_store on this window, whose
 *     status must be 1.  host, u, v, color8, weights8 from that call; idepth = idepth_zero = its idepth, priorF = 0; one IN / 0 residual per
 *     frame with res_state 0, remapped through frame_src (optimizeImmaturePoint's setIdepthZero / setIdepth, EFPoint::takeData without prior).
 *   - carried residual: (p, t) is kept when p is carried and t stays; its state and energy are those the next linearisation would read: the
 *     committed linearisation's state_NewState / state_NewEnergy if there is one, else the input state.  A tentative linearisation is
 *     discarded (as by dmv_ba_set_points).  Residuals into a frame that leaves are dropped.
 *   - new_res_target >= 0: every carried point gets an IN / 0 residual into that (new) frame index (makeKeyFrame's residuals of the old
 *     points into the new keyframe).
 *   - residual order (dmv_ba_get_residual_outputs): the carried residuals in their current order, then the new_res_target residuals in new
 *     point order, then the activated points' residuals in new point order, target ascending.
 * Afterwards the handle is as the three set calls leave it: no linearisation, adjoints and state must be set again, dmv_ba_get_solve_HdiF
 * refuses, and the chunk shape, host ranges and phase-D table are the new window's; no activation is available to a later edit.  One launch
 * (the gather; the handle's launch count moves by 1), about 4 + 4 bytes per point up and, when a committed linearisation exists, 5 bytes per
 * carried residual down; one synchronisation.
 * Errors, all before any allocation, copy or launch, with the handle unchanged: DMV_ERR_INVALID for NULL ba / a / frame_src / point_src,
 * nf or a slot outside dmv_ba_set_window's range, frame_src entries outside -1..nf_current-1 or repeated, npts outside 1..max_points,
 * point_src entries out of range or repeated, an activation entry without an activation on this window, beyond its size or with a status
 * other than 1, a point whose host frame leaves, points not ordered by host frame, a new_res_target outside -1..nf-1 or equal to a carried
 * point's host or to a target it already has a residual into, and too many chunks; DMV_ERR_STATE for a sharded handle or a window without
 * points and residuals. */
typedef struct dmv_ba_edit_args {
  int nf;                    /* frames of the new window, as dmv_ba_set_window */
  const int* slots;          /* nf image slots, as dmv_ba_set_window (NULL: 0..nf-1) */
  const int32_t* frame_src;  /* nf: the frame's index in the current window, or -1 for a frame that joins */
  int npts;                  /* points of the new window (ordered by host frame, as dmv_ba_set_points requires) */
  const int32_t* point_src;  /* npts: index in the current point list (>= 0), or -1 - k for entry k of the last activation */
  int new_res_target;        /* new frame index: every carried point gets an IN / 0 residual into it, or -1 */
} dmv_ba_edit_args;
int dmv_ba_edit_window(dmv_ba* ba, const dmv_ba_edit_args* a);

/* ------------------------------------------------------------------------------------------------
 * New immature points of a keyframe  ==  FullSystem::makeNewTraces (FullSystem.cpp:L1640-1667): PixelSelector::makeMaps
 * (FullSystem/PixelSelector2.cpp:L158-307) on the handle's RESIDENT frame (the one last given to dmv_ct_upload_new_image /
 * dmv_ct_upload_raw_image / dmv_ct_upload_new, or made resident by dmv_ct_set_ref_from_ba), then the raster loop over
 * [3, w-4) x [3, h-4) with the ImmaturePoint constructor of dmv_ct_init_points, keeping the points whose energyTH is finite.
 * Bit-identical to the reference's CPU code: selection map, point order, types and constructor fields.
 * ------------------------------------------------------------------------------------------------ */
typedef struct dmv_ps_settings {      /* util/settings.cpp:L144, L167-170 */
  float minGradHistCut;               /* 0.5 (must be < 0.99: the reference reads unset histogram bins above) */
  float minGradHistAdd;               /* 7 */
  float gradDownweightPerLevel;       /* 0.75 */
  int selectDirectionDistribution;    /* 1 */
  int gammaWeightsPixelSelect;        /* 1: absSquaredGrad *= getBGradOnly(I)^2 (HessianBlocks.cpp:L184-188) */
} dmv_ps_settings;
void dmv_ps_default_settings(dmv_ps_settings* s);
typedef struct dmv_new_traces_args {
  float density;                /* makeMaps' numWant: setting_desiredImmatureDensity = 1500 (finite, > 0) */
  int recursionsLeft;           /* 1 (0..8) */
  float thFactor;               /* 1 (CoarseInitializer::setFirst passes 2; finite, > 0) */
  const float* B;               /* CalibHessian::B[256] as FullSystem::setGammaFunction leaves it; NULL = identity */
  const dmv_ps_settings* settings;  /* NULL = defaults */
  int* potential;               /* in/out: PixelSelector::currentPotential (3 at construction; >= 1).  The caller's state: FullSystem owns
                                   one PixelSelector while its two coarse trackers swap roles */
  int cap;                      /* capacity of every per-point output */
  int* n;                       /* out: points created; on overflow the count needed (and DMV_ERR_INVALID: *potential and *numPointsTotal
                                   are then left unchanged, so a retry with a larger cap gives the same result) */
  int* numPointsTotal;          /* out: makeMaps' return value (numHaveSub) */
  int32_t *u, *v;               /* out, makeNewTraces' push_back order */
  float* type;                  /* out: the selectionMap value, 1 / 2 / 4 */
  float *color8, *weights8, *gradH4, *energyTH;   /* out: as dmv_ct_init_points */
  float* map;                   /* optional (w*h): selectionMap as makeMaps leaves it */
} dmv_new_traces_args;
/* PixelSelector's randomPattern (srand(3141592), rand() & 0xFF over w*h entries, L43-47) is generated once per handle, on first use, by a
 * restatement of glibc's rand(); the caller's rand() state is not touched.  The scratch (about 170 bytes of device memory per level-0 pixel, and 96 bytes of
 * pinned host memory per point of min(cap, w*h)) is allocated on first use, so dmv_ct_create is unchanged.  Ordered on the handle's stream; returns after one synchronisation (makeMaps' recursion is decided on the device).
 * Errors: DMV_ERR_INVALID for levels < 3, w or h not a multiple of 16, bad arguments (including *potential < 1), or more than cap points
 * (*n = the count needed); DMV_ERR_CUDA. */
int dmv_ct_make_new_traces(dmv_ct* ct, const dmv_new_traces_args* a);
/* dmv_ct_make_new_traces with the new points put straight into slot `slot` of an immature-point store, without their round trip through
 * host memory.  Bit-identical to the pair
 *   1. dmv_ct_make_new_traces(ct, a),
 *   2. dmv_ip_store_put(s, slot, pts) with pts = those points, u and v converted to float, and the ImmaturePoint constructor's in/out values:
 *      idepth_min 0, idepth_max NaN (0x7FC00000), quality 10000, lastTraceStatus 5 (IPS_UNINITIALIZED), lastTraceUV2 (0, 0),
 *      lastTracePixelInterval 0,
 * on every observable: the slot's contents and count (the slot is replaced, as by put; no point empties it), the other slots, every later
 * trace or activation of the store, *potential, *numPointsTotal, *n, map and the requested per-point outputs.
 * a: as dmv_ct_make_new_traces, but each per-point output (u, v, type, color8, weights8, gradH4, energyTH) may be NULL on its own, and cap is
 * the capacity of those that are not.  They are read back from the slot's rows after the edit (type, which the store does not hold, from
 * the staged copy beside them).  A caller that needs only ImmaturePoint::my_type for dmv_ba_activate_store asks for type alone: 4 bytes per
 * point come down, and the row map of the store's edit (4 bytes per point in the store) goes up.
 * Overflow: more points than cap with any per-point output requested gives DMV_ERR_INVALID with *n = the count needed, the store,
 * *potential and *numPointsTotal unchanged (a retry gives the same result); with no per-point output there is no cap.
 * Launch count: ct's moves as dmv_ct_make_new_traces' does on the same frame (the copy into the store takes the place of the copy into
 * host memory; the store's gather is not counted, as for put).  On overflow the copy is not launched: one launch fewer.
 * Two synchronisations: one after the selection (it reads the point count), one after the store's edit.
 * Errors, all before any allocation, copy or launch (the store, *potential and the launch counts unchanged): those of
 * dmv_ct_make_new_traces, with the same messages, except for NULL per-point outputs; DMV_ERR_INVALID for a NULL s, slot outside
 * 0..DMV_IP_STORE_SLOTS-1, or a store on another device than ct. */
int dmv_ct_make_new_traces_store(dmv_ct* ct, dmv_ip_store* s, int slot, const dmv_new_traces_args* a);

/* enable/disable the CUDA-event timing of dmv_ct_calc_res_gs (off by default); dmv_ct_last_timing()[0] = kernel milliseconds */
int dmv_ct_set_timing(dmv_ct* ct, int enable);
int dmv_ct_last_timing(dmv_ct* ct, float ms[4]);
int dmv_ct_kernel_launch_count(dmv_ct* ct, long long* n);
int dmv_ct_last_point_evaluations(dmv_ct* ct, double* n);   /* sum over the last dmv_ct_track's evaluations of the level's reference-point count
                                                               (after dmv_ct_track_tries: over its tries) */

/* ------------------------------------------------------------------------------------------------
 * Coarse-initialiser handle  ==  the GPU side of CoarseInitializer::calcResAndGS (FullSystem/CoarseInitializer.{h,cpp})
 * The rest of CoarseInitializer::trackFrame (doStep, applyStep, optReg, propagateUp/Down, the 8x8 solve; L85-281, L650-965) is scalar
 * per-point host code that runs once per sequence and stays with the caller: it owns the Pnt arrays and passes their live fields per call.
 * ------------------------------------------------------------------------------------------------ */
typedef struct dmv_ci dmv_ci;
typedef struct dmv_ci_config {
  int w, h;
  int levels;      /* pyrLevelsUsed */
  int max_points;  /* capacity of points[lvl] (numPoints[0] is the largest) */
  int device;
} dmv_ci_config;
int dmv_ci_create(const dmv_ci_config* cfg, dmv_ci** out);
int dmv_ci_destroy(dmv_ci* ci);
/* CoarseInitializer::makeK (CoarseInitializer.cpp:L967-999) */
int dmv_ci_set_K(dmv_ci* ci, int level, float fx, float fy, float cx, float cy);
/* firstFrame->dIp[level] / newFrame->dIp[level] (w_l*h_l*3 floats AoS) */
int dmv_ci_upload_first(dmv_ci* ci, int level, const float* dIp_aos3);
int dmv_ci_upload_new(dmv_ci* ci, int level, const float* dIp_aos3);
/* the constant fields of points[level] (Pnt::u, v, outlierTH; CoarseInitializer.h:L44-82), set by setFirst (L804-889) */
int dmv_ci_set_points(dmv_ci* ci, int level, int n, const float* u, const float* v, const float* outlierTH);

typedef struct dmv_ci_eval_args {
  int level;
  float RKi[9];          /* (refToNew.rotationMatrix() * Ki[lvl]).cast<float>(), row-major (L341) */
  double t_d[3];         /* refToNew.translation() */
  double t_log[3];       /* refToNew.log().head<3>() (L601) */
  float r2new_aff[2];    /* exp(refToNew_aff.a), refToNew_aff.b (L343) */
  float huberTH;         /* setting_huberTH */
  float alphaK, alphaW, couplingWeight;             /* CoarseInitializer members (CoarseInitializer.h:L107-111) */
  double weightZeroPriorX, weightZeroPriorY;        /* setting_weightZeroPriorDSOInitX / Y (L606-611) */
  /* live per-point fields of points[level], n entries (n as given to dmv_ci_set_points) */
  const float* idepth_new;
  const uint8_t* isGood;
  const float* energy2;   /* Pnt::energy, 2 per point */
  const float* iR;
  /* per-point results (any may be NULL): Pnt::isGood_new, energy_new (2 per point), maxstep, lastHessian_new and the JbBuffer_new rows
   * (10 per point) as L562-586 leave them.  maxstep / lastHessian_new / JbBuffer_new are meaningful for isGood_new points only. */
  uint8_t* isGood_new;
  float* energy_new2;
  float* maxstep;
  float* lastHessian_new;
  float* JbBuffer_new10;
} dmv_ci_eval_args;
typedef struct dmv_ci_eval_result {
  float H[64], b[8], Hsc[64], bsc[8];   /* H_out, b_out, H_out_sc, b_out_sc (row-major) */
  float res3[3];                        /* Vec3f(E.A, alphaEnergy, E.num) */
  float alphaOpt;
  int n_good_new;
} dmv_ci_eval_result;
/* CoarseInitializer::calcResAndGS (CoarseInitializer.cpp:L333-625) as ONE launch */
int dmv_ci_calc_res_and_gs(dmv_ci* ci, const dmv_ci_eval_args* args, dmv_ci_eval_result* out);
int dmv_ci_kernel_launch_count(dmv_ci* ci, long long* n);

#ifdef __cplusplus
}
#endif
#endif /* DMVIO_B200_H */
