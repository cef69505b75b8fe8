/* C glue over the C++ host adapters (WindowBA, CoarseTracker) so that the Python tests and bench can drive them through
 * ctypes.  Not part of the drop-in boundary (that is include/dmvio_b200.h); a C++ host links the classes directly. */
#pragma once
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
void* dmvh_window_create(int w, int h, int max_frames, int max_points, int device, const double calib_value_scaled[4]);
void dmvh_window_destroy(void* win);
const char* dmvh_window_error(void* win);
/* is_image: 1 = raw w*h float image (level-0 [I,dx,dy] built on the device), 0 = w*h*3 dI AoS */
int dmvh_window_add_frame(void* win, const float* data, int is_image, const double R[9], const double t[3], const double state[10],
                          const double state_zero[10], float ab_exposure, int frameID);
void dmvh_window_drop_frame(void* win, int idx); /* the frame leaves the window; its image slot is reused by the next add_frame */
int dmvh_window_set_points(void* win, int n, const int32_t* host, const float* u, const float* v, const float* idepth, const float* idepth_zero,
                           const float* color8, const float* weights8, const uint8_t* hasDepthPrior);
/* same, with WindowBA::insertPoints' carry_from (index of each point in the previous list, -1 = newly activated) */
int dmvh_window_set_points_carry(void* win, int n, const int32_t* host, const float* u, const float* v, const float* idepth, const float* idepth_zero,
                                 const float* color8, const float* weights8, const uint8_t* hasDepthPrior, const int32_t* carry_from);
int dmvh_window_set_residuals(void* win, int n, const int32_t* point, const int32_t* target);
/* installs WindowBA::computeBAUpdate (the slot of BAGTSAMIntegration::computeBAUpdate): cb(H N*N, b N, lambda, nFrames, HNoLambda N*N, x_out N, user); NULL removes it */
typedef void (*dmvh_ba_update_cb)(const double* H, const double* b, double lambda, int nFrames, const double* HNoLambda, double* x_out, void* user);
void dmvh_window_set_ba_update_hook(void* win, dmvh_ba_update_cb cb, void* user);
/* multi-GPU: WindowBA::setSharding + the application's host allgather (send `bytes`, receive nranks*bytes in rank order); call before
 * dmvh_window_prepare.  dmvh_window_p2p_setup / dmvh_window_comm_init choose the device-side exchange (NVLink peer memory / NCCL). */
typedef void (*dmvh_allgather_cb)(const void* send, void* recv_all, size_t bytes, void* user);
int dmvh_window_set_sharding(void* win, int rank, int nranks, dmvh_allgather_cb cb, void* user);
int dmvh_window_p2p_setup(void* win);
int dmvh_window_comm_init(void* win, const void* nccl_unique_id128);
int dmvh_window_get_idepths(void* win, float* idepth);
/* WindowBA::profile_us: microseconds spent in [solve, state step + tables, linearize, prior energies] and the iteration count */
void dmvh_window_profile(void* win, double out5[5], int reset);
/* WindowBA::s.<name> = value for the settings the optimisation loop reads (minOptIterations, thOptIterations, margWeightFac, ...); 0 ok, -1 unknown */
int dmvh_window_set_setting(void* win, const char* name, double value);
int dmvh_window_prepare(void* win); /* makeIDX + setAdjointsF + setPrecalcValues */
double dmvh_window_linearize(void* win, int fix);
void dmvh_window_apply(void* win);
int dmvh_window_solve(void* win, int iteration, double lambda, double* x_out);
int dmvh_window_optimize(void* win, int its, double* energyLog, int cap); /* the LM loop only (WindowBA::optimize(its, log, finish = false)) */
/* tail of FullSystem::optimize (WindowBA::finishOptimize): returns the energy; removed (cap entries) gets the indices of the deleted residuals */
double dmvh_window_finish_optimize(void* win, int32_t* removed, int cap, int* nremoved, int* nres_left);
void dmvh_window_get_point_stats(void* win, float* maxRelBaseline, int32_t* numGoodResiduals);
void dmvh_window_set_last_residuals(void* win, const int32_t* target_frameID2, const int32_t* state2); /* per point: lastResiduals[0..1] */
/* WindowBA::flagPointsForRemoval; returns counts through nmarg / ndrop (arrays sized npts) */
void dmvh_window_flag_points(void* win, int nflagged, const int32_t* flagged_frames, int32_t* marg, int* nmarg, int32_t* drop, int* ndrop);
void dmvh_window_get_tables(void* win, float* precalc, double* adHost, double* adTarget);
void dmvh_window_get_system(void* win, double* HA, double* bA, double* Hsc, double* bsc, double* lastHS, double* lastbS);
void dmvh_window_get_states(void* win, double* states10, float* idepth, float* frameEnergyTH);
double dmvh_window_energy_L(void* win);
double dmvh_window_energy_M(void* win); /* EnergyFunctional::calcMEnergyF: the marginalisation prior's energy at the current state */
/* WindowBA::marginalizeFrame: 0 ok, -1 error (dmvh_window_error) */
int dmvh_window_marginalize_frame(void* win, int idx, double* HM, double* bM, int* nf_left, int* nres_left);
/* host/nullspace.h on plain arrays (no handle, no GPU): evalPT = nf x (R row-major 9 | t 3); ns_out 7 x (8 nf + 4), may be NULL;
 * x (8 nf + 4, may be NULL) is orthogonalised in place (EnergyFunctional::orthogonalize) */
void dmvh_nullspaces_orthogonalize(int nf, const double* evalPT12, double* ns_out, double* x, double solverModeDelta);
/* host/marg_frame.h on plain arrays (no handle, no GPU): HM (odim*odim) / bM (odim) are overwritten with the ndim = odim - 8 system */
void dmvh_marginalize_frame_hm(double* HM, double* bM, int nFrames, int idx, const double prior8[8], const double delta_prior8[8]);
/* WindowBA::marginalizePointsF: marginalises `marg` (dropping the badly constrained ones) and drops `drop`; erases them, re-uploads the window.
 * Returns the resInM increment (-1 on error); HM/bM (N*N, N) and the surviving point count are written if non-NULL. */
int dmvh_window_marginalize_points(void* win, int nmarg, const int32_t* marg, int ndrop, const int32_t* drop, double* HM, double* bM, int* npts_left,
                                   int* nres_left);

void* dmvh_ct_create(int w, int h, int levels, int max_points, int device, const double calib_value_scaled[4]);
void dmvh_ct_destroy(void* ct);
int dmvh_ct_set_ref(void* ct, int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, const float* ref_dIp_concat,
                    double ref_a, double ref_b, float ref_exposure);
int dmvh_ct_pc_n(void* ct, int lvl);
int dmvh_ct_set_new_image(void* ct, const float* image, float exposure);
int dmvh_ct_set_ref_device(void* ct, int n, const float* Ku, const float* Kv, const float* new_idepth, const float* HdiF, const float* ref_image_wh,
                           double ref_a, double ref_b, float ref_exposure); /* makeCoarseDepthL0 on the device */
void dmvh_ct_set_device_lm(void* ct, int on);
double dmvh_ct_point_evaluations(void* ct); /* CoarseTracker::pointEvaluations of the last track (measurement) */ /* 1 (default): LM loop on the device (dmv_ct_track); 0: host loop */
int dmvh_ct_track(void* ct, double R[9], double t[3], double* a, double* b, int coarsestLvl, const double minResForAbort[5],
                  double lastResiduals[5], double flow[3], int* iterations, long long* evaluations);
/* raw-frame ingest (host/coarse_tracker_ingest.cpp): CoarseTracker::setUndistort / uploadRawImage / downloadFrame */
int dmvh_ct_set_undistort(void* ct, int wOrg, int hOrg, const float* remapX, const float* remapY, const float* G, int nG, const float* vignetteInv,
                          int photometric_mode);
int dmvh_ct_upload_raw_image(void* ct, const void* raw, int bytes_per_px, float exposure, float factor, float ab_exposure);
int dmvh_ct_download_frame(void* ct, int level, float* dIp_aos3);
/* new immature points of the resident keyframe (host/coarse_tracker_select.cpp): CoarseTracker::makeNewTraces (dmv_ct_make_new_traces);
 * settings5 = {minGradHistCut, minGradHistAdd, gradDownweightPerLevel, selectDirectionDistribution, gammaWeightsPixelSelect} or NULL */
int dmvh_ct_make_new_traces(void* ct, int* potential, float density, int recursionsLeft, float thFactor, const float* B, const float* settings5, int cap,
                            int* n, int* numPointsTotal, int32_t* u, int32_t* v, float* type, float* color8, float* weights8, float* gradH4,
                            float* energyTH, float* map);
/* the keyframe hand-off from the window (host/coarse_tracker_window.cpp): CoarseTracker::setCoarseTrackingRefFromWindow (dmv_ct_set_ref_from_ba) */
int dmvh_ct_set_ref_from_window(void* ct, void* win, double ref_a, double ref_b, float ref_exposure);
const char* dmvh_ct_error(void* ct);   /* CoarseTracker::error() */
/* the window's dmv_ba handle (for the C ABI directly) */
void* dmvh_window_ba_handle(void* win);
/* makeCoarseDepthL0's inputs as the host path gathers them from the window, in its fold order (WindowBA::coarseTrackingRefInputs): writes at
 * most cap entries (point: index in the window's point list, may be NULL), returns the count (or -1, dmvh_window_error says why) */
int dmvh_window_coarse_ref_inputs(void* win, float* Ku, float* Kv, float* new_idepth, float* HdiF, int32_t* point, int cap);
/* per point: lastResiduals[0..1] target frameIDs and states (the inverse of dmvh_window_set_last_residuals) */
void dmvh_window_get_last_residuals(void* win, int32_t* target_frameID2, int32_t* state2);

/* CoarseInitializer adapter (host/coarse_initializer.h): trackFrame on the host, calcResAndGS on the device */
void* dmvh_ci_create(int w, int h, int levels, int max_points, int device, const double calib_value_scaled[4]);
void dmvh_ci_destroy(void* ci);
const char* dmvh_ci_error(void* ci);
int dmvh_ci_set_first(void* ci, const float* dIp_concat, float exposure, const int32_t* n_per_level, const float* u, const float* v, const float* type,
                      const int32_t* parent, const int32_t* neighbours10);
int dmvh_ci_track(void* ci, const float* dIp_concat, float exposure, double* R9, double* t3, double* ab2, int32_t* state3);
int dmvh_ci_npts(void* ci, int lvl);
void dmvh_ci_get_points(void* ci, int lvl, float* out12);
long long dmvh_ci_evaluations(void* ci);

#ifdef __cplusplus
}
#endif
