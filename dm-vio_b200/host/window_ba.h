// Host-side C++ mirror of the reference's BA surface (FullSystem::optimize + EnergyFunctional), driving the CUDA hot
// path through the C ABI (include/dmvio_b200.h).  Names, argument meaning and call order follow the reference so that a
// DM-VIO checkout can forward its own methods 1:1 (see INTEGRATION.md):
//     FullSystem::setPrecalcValues / linearizeAll / applyRes_Reductor / setNewFrameEnergyTH / backupState /
//     doStepFromBackup / loadSateBackup / optimize                 (src/dso/FullSystem/FullSystemOptimize.cpp, FullSystem.cpp:L1670-1680)
//     EnergyFunctional::setAdjointsF / setDeltaF / solveSystemF / resubstituteF_MT / calcLEnergyF_MT / calcMEnergyF
//                                                                  (src/dso/OptimizationBackend/EnergyFunctional.cpp)
// The pointer graph of the reference (FrameHessian* / PointHessian* / PointFrameResidual*) is flattened to index-based
// vectors; everything numerical on the per-point path happens on the GPU, the O(nf^2) tables and the dense solve stay here.
#pragma once
#include "../../include/dmvio_b200.h"
#include "se3.h"
#include <functional>
#include <string>
#include <vector>

namespace dmvio_b200 {

// FullSystem/HessianBlocks.h:L60-68
constexpr float SCALE_IDEPTH = 1.0f, SCALE_XI_ROT = 1.0f, SCALE_XI_TRANS = 1.0f, SCALE_F = 50.0f, SCALE_C = 50.0f, SCALE_A = 10.0f, SCALE_B = 1000.0f;
constexpr int CPARS = 4, patternNum = 8;

struct Settings {  // util/settings.cpp:L60-160
  float setting_huberTH = 9, setting_outlierTH = 12 * 12, setting_outlierTHSumComponent = 50 * 50, setting_overallEnergyTHWeight = 1;
  float setting_coarseCutoffTH = 20, setting_affineOptModeA = 1e12f, setting_affineOptModeB = 1e8f;
  float setting_idepthFixPrior = 50 * 50, setting_initialRotPrior = 1e11f, setting_initialTransPrior = 1e10f;
  float setting_initialAffAPrior = 1e14f, setting_initialAffBPrior = 1e14f, setting_initialCalibHessian = 5e9f;
  float setting_frameEnergyTHConstWeight = 0.5f, setting_frameEnergyTHN = 0.7f, setting_frameEnergyTHFacMedian = 1.5f;
  float setting_thOptIterations = 1.2f;
  int setting_minOptIterations = 1;
  bool setting_orthogonalizeXLater = true;   // setting_solverMode & SOLVER_ORTHOGONALIZE_X_LATER (settings.cpp:L81)
  double setting_solverModeDelta = 0.00001;  // settings.cpp:L82
  float setting_minIdepth = 0.02f;                                       // settings.cpp:L53
  int setting_minGoodActiveResForMarg = 3, setting_minGoodResForMarg = 4;  // settings.cpp:L127-128
  float setting_idepthFixPriorMargFac = 600 * 600, setting_margWeightFac = 0.5f * 0.5f, setting_minIdepthH_marg = 50;  // settings.cpp:L68, L118, L89
};

struct AffLight {  // util/NumType.h:L166-192
  double a = 0, b = 0;
  static void fromToVecExposure(float exposureF, float exposureT, AffLight g2F, AffLight g2T, double out[2]);
};

struct CalibHessian {  // FullSystem/HessianBlocks.h:L309-409
  double value[4], value_zero[4], value_scaled[4], value_backup[4], step[4], value_minus_value_zero[4];
  float value_scaledf[4], value_scaledi[4];
  void setValue(const double v[4]);
  void setValueScaled(const double vs[4]);
};

struct FrameHessian {  // FullSystem/HessianBlocks.h:L113-307 (+ EFFrame: prior, delta, delta_prior)
  SE3 worldToCam_evalPT, PRE_worldToCam, PRE_camToWorld;
  double state_zero[10], state_scaled[10], state[10], step[10], state_backup[10];
  float frameEnergyTH = 8 * 8 * patternNum, ab_exposure = 1;
  int frameID = 0, slot = 0;
  bool addCamPrior = false;
  double prior[8], delta_prior[8], delta[8];
  void setState(const double s[10]);
  AffLight aff_g2l() const { AffLight l; l.a = state_scaled[6]; l.b = state_scaled[7]; return l; }
  AffLight aff_g2l_0() const { AffLight l; l.a = state_zero[6] * SCALE_A; l.b = state_zero[7] * SCALE_B; return l; }
};

struct PointHessian {  // FullSystem/HessianBlocks.h:L413-508 (+ EFPoint)
  int host = 0;
  float u = 0, v = 0, idepth = 0, idepth_zero = 0, idepth_backup = 0, step = 0;
  float color[8], weights[8];
  bool hasDepthPrior = false;
  float priorF = 0;
  float maxRelBaseline = 0;          // updated by linearizeAll(true) (FullSystemOptimize.cpp:L66-79)
  int numGoodResiduals = 0;
  // PointHessian::lastResiduals (HessianBlocks.h:L447): the residuals to the two newest keyframes, identified by the target's frameID
  // (-1 = none) instead of a pointer, with their last committed state (0 IN, 1 OOB, 2 OUTLIER)
  int lastResiduals_target[2] = {-1, -1};
  int lastResiduals_state[2] = {0, 0};
};

struct PointFrameResidual {  // FullSystem/Residuals.h:L53-110
  int point = 0, target = 0;
  int state_state = 0, state_NewState = 2;
  float state_energy = 0, state_NewEnergy = 0, state_NewEnergyWithOutlier = -1;
  float centerProjectedTo[3] = {0, 0, 0};
};

class WindowBA {
 public:
  WindowBA(int w, int h, int max_frames, int max_points, int device = 0);
  ~WindowBA();
  WindowBA(const WindowBA&) = delete;
  WindowBA& operator=(const WindowBA&) = delete;
  bool ok() const { return ba_ != nullptr; }
  const std::string& error() const { return err_; }

  Settings s;
  CalibHessian Hcalib;
  std::vector<FrameHessian> frameHessians;
  std::vector<PointHessian> points;            // EnergyFunctional::allPoints order (by host frame)
  std::vector<PointFrameResidual> activeResiduals;
  std::vector<double> HM, bM;                  // marginalisation prior (EnergyFunctional::HM / bM), N*N / N
  std::vector<double> lastHS, lastbS, lastX;   // EnergyFunctional.h:L113-116
  // Downstream consumer of the reduced system (SURVEY §8b): the slot of dmvio::BAGTSAMIntegration::computeBAUpdate (BAGTSAMIntegration.h:L189-190,
  // called from EnergyFunctional.cpp:L958-968 when setting_useGTSAMIntegration): gets the lambda-damped Schur-reduced H (N*N row-major, DSO
  // ordering [C4 | per frame trans3 rot3 a b]), b, lambda and the undamped H; returns x (N).  Unset = the no-GTSAM branch (Jacobi-preconditioned
  // LDL^T, EnergyFunctional.cpp:L971-973).  IMU / GTSAM code stays on the host and plugs in here.
  std::function<std::vector<double>(const std::vector<double>& H, const std::vector<double>& b, double lambda, int nFrames, const std::vector<double>& HNoLambda)>
      computeBAUpdate;
  std::function<void(double energy)> acceptBAUpdate;   // BAGTSAMIntegration::acceptBAUpdate (FullSystemOptimize.cpp:L571)
  int resInA = 0;
  double lastEnergyTotal = 0;
  // wall-clock microseconds accumulated over the LM iterations of optimize(): [backup + solveSystemF, doStepFromBackup (states + precalc tables),
  // linearizeAll (upload of the tables, fused launch, sync), calcLEnergy + calcMEnergy, #iterations]; reset by the caller
  double profile_us[5] = {0, 0, 0, 0, 0};

  // ---- construction (EnergyFunctional::insertFrame / insertPoint / insertResidual + FrameHessian::makeImages on the device)
  int insertFrame(const float* image_wh, const SE3& worldToCam_evalPT, const double state[10], const double state_zero[10], float ab_exposure,
                  int frameID);
  int insertFrameDI(const float* dI_aos3, const SE3& worldToCam_evalPT, const double state[10], const double state_zero[10], float ab_exposure,
                    int frameID);
  void dropFrame(int idx);             // the frame leaves the window and the marginalisation prior is RESET (tests / streaming bench)
  // FullSystem::marginalizeFrame (FullSystem/FullSystemMarginalize.cpp:L156-219) + EnergyFunctional::marginalizeFrame (EnergyFunctional.cpp:L522-675):
  // the residuals that still target the frame are dropped, HM/bM are Schur-complemented with respect to the frame's 8 variables (host fp64,
  // host/marg_frame.h), the frame leaves the window (its image slot becomes free) and the smaller window is re-uploaded.  The frame must not
  // host points any more (flagPointsForRemoval + marginalizePointsF first).  Returns false on error.
  bool marginalizeFrame(int idx);
  // Replaces the point set (must be ordered by host frame).  carry_from (optional, n entries): index of the same point in the previous list, or
  // -1 for a newly activated point; carries numGoodResiduals / maxRelBaseline / lastResiduals over, everything else is reset (see INTEGRATION.md).
  void insertPoints(int n, const int* host, const float* u, const float* v, const float* idepth, const float* idepth_zero, const float* color8,
                    const float* weights8, const unsigned char* hasDepthPrior, const int* carry_from = nullptr);
  void insertResiduals(int n, const int* point, const int* target);
  bool makeIDX();  // uploads points/residuals (EnergyFunctional::makeIDX, EnergyFunctional.cpp:L998-1016)

  // ---- reference surface
  void setAdjointsF();                 // EnergyFunctional.cpp:L48-108
  void setPrecalcValues();             // FullSystem.cpp:L1670-1680 (+ setDeltaF)
  double linearizeAll(bool fixLinearization);  // FullSystemOptimize.cpp:L150-218 (energy = Vec3[0])
  void applyRes_Reductor();            // FullSystemOptimize.cpp:L90-94
  void setNewFrameEnergyTH();          // FullSystemOptimize.cpp:L96-149
  void solveSystemF(int iteration, double lambda);  // EnergyFunctional.cpp:L841-996, no-GTSAM branch
  double calcLEnergyF_MT();            // EnergyFunctional.cpp:L411-431 (priors; no linearised residuals in the active set)
  double calcMEnergyF();               // EnergyFunctional.cpp:L324-346
  void backupState();                  // FullSystemOptimize.cpp:L322-370
  bool doStepFromBackup();             // FullSystemOptimize.cpp:L224-317 (point part deferred to the next linearizeAll: fused on the GPU)
  void loadSateBackup();               // FullSystemOptimize.cpp:L371-388
  // FullSystemOptimize.cpp:L417-647 (no IMU); returns #iterations.  finish = true runs the reference's tail (L591-609): setEvalPT of the newest
  // frame, setAdjointsF, setPrecalcValues and linearizeAll(true); finish = false stops after the LM loop (tests / benches of the loop alone).
  int optimize(int mnumOptIts, std::vector<double>* energyLog = nullptr, bool finish = true);
  double finishOptimize();             // the tail alone; returns the energy of linearizeAll(true)
  std::vector<int> lastRemovedResiduals;   // indices (before the erase) of the residuals linearizeAll(true) deleted (L196-214)
  // FullSystem::flagPointsForRemoval (FullSystem.cpp:L785-879), decision part: which points leave the window when the frames in
  // `flaggedFrames` (window indices, FrameHessian::flaggedForMarginalization) are about to be marginalised.  toMarg: candidates for
  // marginalizePointsF (isOOB || host flagged, and isInlierNew); toDrop: PS_DROP.
  void flagPointsForRemoval(const std::vector<int>& flaggedFrames, std::vector<int>* toMarg, std::vector<int>* toDrop);

  // ---- keyframe marginalisation of points (FullSystem::makeKeyFrame: flagPointsForRemoval -> marginalizePointsF / dropPointsF)
  // toMarg: the caller's PS_MARGINALIZE candidates (PointHessian::isOOB && isInlierNew, or host frame flagged); for each the device runs
  // resetOOB / linearize / applyRes / fixLinearizationF (FullSystem.cpp:L826-838) and EnergyFunctional::marginalizePointsF
  // (EnergyFunctional.cpp:L678-742); candidates whose idepth_hessian (1 / HdiF of the last accumulation) is <= setting_minIdepthH_marg
  // are dropped instead (FullSystem.cpp:L840-850).  toDrop: PS_DROP points (EnergyFunctional::dropPointsF).  HM / bM are updated with
  // setting_margWeightFac, all listed points and their residuals are erased and the window is re-uploaded (makeIDX).  Returns the number
  // of residuals that entered the prior (resInM increment), -1 on error.
  int marginalizePointsF(const std::vector<int>& toMarg, const std::vector<int>& toDrop = std::vector<int>());
  std::vector<float> adHTdeltaF() const;   // EnergyFunctional::setDeltaF (EnergyFunctional.cpp:L175-187), [h + t*nf][8]
  int resInM = 0;

  // ---- multi-GPU (SURVEY.md §8e): one WindowBA per rank / GPU.  Every rank holds the WHOLE window on the host (frames, point and residual
  // lists, priors: small) and uploads only its share of the points (index % nranks == rank) with their residuals; the linearised system,
  // energies and counters are summed over the ranks inside the launch (peer memory or NCCL, dmv_ba_p2p_* / dmv_ba_comm_init), so every rank
  // takes the identical LM decisions and steps.  Per-point / per-residual results live on the owning rank's device; where the host logic needs
  // them for ALL points (setNewFrameEnergyTH's percentile, flagPointsForRemoval, residual removal, depth read-back) the adapter gathers them
  // with `allgather`, supplied by the application's host communicator (MPI_Allgather / torch.distributed / ...): send `bytes` bytes, receive
  // nranks * bytes in rank order.  Call setSharding before makeIDX; the exchange set-up calls forward to the C ABI.
  std::function<void(const void* send, void* recv_all, size_t bytes)> allgather;
  bool setSharding(int rank, int nranks);
  bool p2pExport(void* ipc_handle64);                      // dmv_ba_p2p_export
  bool p2pImport(const void* ipc_handles);                 // dmv_ba_p2p_import(nranks, rank, handles)
  bool commInit(const void* nccl_unique_id);               // dmv_ba_comm_init (NCCL fallback)
  bool p2pSetup();                                         // export -> allgather of the 64-byte handles -> import
  int rank() const { return rank_; }
  int nranks() const { return nranks_; }
  // the device handle, for consumers that read the window on the device (CoarseTracker::setCoarseTrackingRefFromWindow)
  dmv_ba* handle() const { return ba_; }

  // ---- results
  void syncResidualStates();           // pulls state_NewState / energies / centerProjectedTo of the last linearisation from the device
  void getIdepths(float* idepth);      // current device depths
  // makeCoarseDepthL0's inputs as the host path collects them (CoarseTracker.cpp:L144-158) for the newest frame: per point whose
  // lastResiduals[0] targets it and is IN, that residual's centerProjectedTo, the point's HdiF of the last solve (downloaded) and its index in
  // `points`.  The order is makeCoarseDepthL0's: `points` after FullSystem::removeOutliers' swap-with-back removal of the points without
  // residuals (csrc/remove_outliers.h), which makeKeyFrame runs right before setCoarseTrackingRef.  Writes at most cap entries (point may be
  // null) and returns their number, or -1 with error() set (more than cap entries; a failed download — sharded windows need the allgather).
  int coarseTrackingRefInputs(float* Ku, float* Kv, float* new_idepth, float* HdiF, int32_t* point, int cap);
  void getFrameStates(double* state10) const;
  double lastGpuMs() const;

  // tables (exposed for tests)
  std::vector<float> precalc;          // nf*nf*32, [h*nf+t]
  std::vector<double> adHost, adTarget;  // nf*nf*64, [h+t*nf]
  std::vector<double> last_HA, last_bA, last_Hsc, last_bsc;

 private:
  bool fail(const char* what);
  void framePrior(const FrameHessian& f, double p[10]) const;
  int nf() const { return (int)frameHessians.size(); }
  void fillState(dmv_ba_state* st, float* th) const;
  dmv_ba* ba_ = nullptr;
  int w_, h_, max_frames_, max_points_;
  std::string err_;
  bool have_pending_x_ = false;      // resubstitute + point step are fused into the next linearizeAll
  std::vector<double> pending_x_;
  double step_sums_[3] = {0, 0, 0};
  bool solved_since_makeIDX_ = false;  // dmv_ba_get_solve_HdiF is valid
  // sharding: global index of every local point / residual, per rank (the same lists on every rank)
  int rank_ = 0, nranks_ = 1;
  std::vector<std::vector<int>> pts_of_rank_, res_of_rank_;
  std::vector<int> local_of_point_, local_of_res_;   // global -> local index on the owning rank
  void rebuildResidualMaps();
  // device read-backs in GLOBAL indexing (gathered over the ranks when sharded); any pointer may be null
  bool fetchResidualOutputs(int32_t* newState, float* newEnergy, float* newEnergyWithOutlier, float* cpt3);
  bool fetchPointFloats(int what, float* out);   // 0: idepth, 1: HdiF of the last solve
  template <class T> bool gatherRows(const std::vector<std::vector<int>>& of_rank, const T* local, int width, T* global);
  float canbreak_frames_[4] = {0, 0, 0, 0};
  std::vector<double> gauge_key_;                 // evaluation points the cached gauge basis belongs to
  std::vector<std::vector<double>> gauge_U_;      // orthonormal basis of the 7 gauge directions (host/nullspace.h: gaugeBasis)
};

}  // namespace dmvio_b200
