// TEST INFRASTRUCTURE ONLY — CPU oracle (restatement) of DM-VIO's immature-point tracing (SURVEY.md §8f-2):
// ImmaturePoint::ImmaturePoint (FullSystem/ImmaturePoint.cpp:L34-63) and ImmaturePoint::traceOn (L77-437), as driven by
// FullSystem::traceNewCoarse (FullSystem/FullSystem.cpp:L541-584).  Pinned bit-exact against the reference's own ImmaturePoint.cpp
// compiled into oracle/_ref (tests/test_ref_pin.py).  Plain float arithmetic in the reference's operation order, no FMA contraction
// (the oracle is built without -march, like the reference).
#pragma once
#include <cstdint>

namespace orc {

struct TraceSettings {  // util/settings.cpp:L111,159,178-187, L79 (huberTH), L82 (outlierTHSumComponent)
  float maxPixSearch = 0.027f, trace_stepsize = 1.0f, trace_GNThreshold = 0.1f, trace_extraSlackOnTH = 1.2f, trace_slackInterval = 1.5f,
        trace_minImprovementFactor = 2.f, huberTH = 9.f, outlierTH = 12 * 12, overallEnergyTHWeight = 1.f, outlierTHSumComponent = 50 * 50;
  int trace_GNIterations = 3, minTraceTestRadius = 2;
};

enum { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };  // ImmaturePoint.h:L47-53

struct ImmaturePt {  // the fields of ImmaturePoint that the constructor writes and traceOn reads / updates (ImmaturePoint.h:L56-90)
  float u, v;
  float color[8], weights[8];
  float gradH[4];  // Mat22f row-major: g00 g01 g10 g11
  float energyTH;
  float idepth_min, idepth_max, quality;
  int lastTraceStatus;
  float lastTraceUV[2], lastTracePixelInterval;
};

// ImmaturePoint constructor: colours, weights, gradH, energyTH from the host's level-0 [I,dx,dy]; returns false if a colour is not finite
bool initImmature(ImmaturePt& p, const float* dI_host, int w, int u, int v, const TraceSettings& s);
// What one traceOn call went through (test coverage only; the arithmetic is the same with or without it).  diag[IPD_*]:
enum {
  IPD_NUM_STEPS = 0,   // numSteps of the discrete search after the clamp at 99 (0: no search)
  IPD_BEST_IDX,        // bestIdx of the search (-1: no search)
  IPD_N_TIED,          // steps whose energy equals the best energy exactly (the best step included)
  IPD_MAX_TIED_IDX,    // the largest such step index
  IPD_GN_ITS,          // Gauss-Newton iterations executed
  IPD_GN_BREAK,        // 1 if the GN loop left by its |stepBack| < trace_GNThreshold break, 0 if it ran out of iterations (or never ran)
  IPD_NONFINITE_SEARCH,// non-finite samples in the search (each added 1e5 to a step's energy)
  IPD_NONFINITE_GN,    // non-finite samples in the GN iterations (each added 1e5)
  IPD_EXIT,            // the return taken: IPX_*
  IPD_N
};
enum {
  IPX_STICKY_OOB = 0,  // entered OOB, returned at once
  IPX_UMIN_OOB,        // uMin outside the image
  IPX_UMAX_OOB,        // uMax outside the image
  IPX_DEPTH_RANGE,     // idepth_min >= 0 and ptpMin[2] outside (0.75, 1.5)
  IPX_SKIPPED,         // interval shorter than trace_slackInterval
  IPX_BADCONDITION,    // errorInPixel * trace_minImprovementFactor > dist
  IPX_NONFINITE_DIR,   // dx or dy not finite
  IPX_GN_OOB,          // a GN pattern sample outside [0, w-1) x [0, h-1)
  IPX_OUTLIER,         // energy test failed, previous status not OUTLIER -> OUTLIER
  IPX_OUTLIER_TWICE,   // energy test failed, previous status OUTLIER -> OOB
  IPX_BAD_INTERVAL,    // new depth interval not finite or idepth_max < 0 -> OUTLIER
  IPX_GOOD,
  IPX_N
};
// ImmaturePoint::traceOn; dI = frame->dI (w*h*3), KRKi row-major 3x3; returns lastTraceStatus.  diag: NULL or IPD_N ints.
int traceOn(ImmaturePt& p, const float* dI, int w, int h, const float KRKi[9], const float Kt[3], const float aff[2], const TraceSettings& s,
            int32_t* diag = nullptr);

}  // namespace orc

extern "C" {
// SoA views for ctypes: every array has n (or n*8, n*4, n*2) entries
int orc_ip_init(int n, const float* dI_host, int w, int h, const int32_t* u, const int32_t* v, float* color8, float* weights8, float* gradH4,
                float* energyTH, uint8_t* ok);
void orc_ip_trace(int n, const float* dI, int w, int h, const float* KRKi9, const float* Kt3, const float* aff2, const float* u, const float* v,
                  const float* color8, const float* weights8, const float* gradH4, const float* energyTH, float* idepth_min, float* idepth_max,
                  float* quality, int32_t* status, float* lastTraceUV2, float* lastTracePixelInterval);
// orc_ip_trace plus diag[n * IPD_N] (see IPD_* / IPX_*)
void orc_ip_trace_diag(int n, const float* dI, int w, int h, const float* KRKi9, const float* Kt3, const float* aff2, const float* u, const float* v,
                       const float* color8, const float* weights8, const float* gradH4, const float* energyTH, float* idepth_min, float* idepth_max,
                       float* quality, int32_t* status, float* lastTraceUV2, float* lastTracePixelInterval, int32_t* diag);
}

extern "C" {
// FullSystem::optimizeImmaturePoint for n immature points of a window: dI_all = nf planes (w*h*3 each); RT[h*nf+t][12] = PRE_RTll (row-major) | PRE_tTll;
// aff[h*nf+t][2] = PRE_aff_mode; calib6 = fxl fyl cxl cyl fxli fyli.  status: 1 activated, 0 skipped (not well constrained), -1 outlier;
// huberTH: setting_huberTH (9 in DSO's defaults); idepth: the optimised inverse depth; res_state[i*nf + f]: 0 IN, 1 OOB, 2 OUTLIER, 255 no residual
// (f == host or early exit).
void orc_ip_activate(int n, int nf, int w, int h, const float calib6[6], const float* dI_all, const float* RT, const float* aff, const int32_t* host,
                     const float* u, const float* v, const float* color8, const float* weights8, const float* energyTH, const float* idepth_min,
                     const float* idepth_max, int minObs, float huberTH, int32_t* status, float* idepth, int32_t* res_state);
}
