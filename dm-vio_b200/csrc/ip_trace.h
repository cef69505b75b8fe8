// ip_init_kernel (ip_trace.cu), which pixel selection (ps_select.cu) also runs on its candidates, and the launch of ip_trace_kernel
// (ip_trace.cu) that the traces on host arrays and on an immature-point store (ip_store.cu) share
#pragma once
#include "../../include/dmvio_b200.h"
#include <cuda_runtime.h>
namespace dmv {
struct IPInitArgs {
  int n, w;
  const int* n_dev;   // non-null: the point count is read there (written by an earlier kernel on the stream); n bounds it and sizes the grid
  float outlierTHSumComponent, outlierTH, overallEnergyTHWeight;
  const int *u, *v;
  float *color, *weights, *gradH, *energyTH;
  int* ok;
  const float4* img;
};
void launch_ip_init(const IPInitArgs& A, cudaStream_t s);

// The tracing layout of a point array (a handle's staging area d_ip, an immature-point store's buffer): cap points per array, the array of
// word w at ip + w * cap (uv and the 8 / 4 per-point vectors interleaved per point), then 14 floats per host frame (KRKi 9 | Kt 3 | aff 2).
// The host staging and ip_trace_kernel both read these offsets.  set is the host frame of each point (an int), status an int too.
namespace ipw {
constexpr int u = 0, v = 1, color = 2, weights = 10, gradH = 18, energyTH = 22;          // read only
constexpr int idepth_min = 23, idepth_max = 24, quality = 25, status = 26, uv = 27, interval = 29;   // in/out: the 7 words from idepth_min on
constexpr int set = 30, tables = 31;
constexpr int inout = 7;
}  // namespace ipw

// One member of a trace launch: a coarse-tracker handle's resident level-0 plane and a point array in the ipw layout
struct IPTraceMember {
  const float4* img;
  float* ip;          // d_ip or a store's buffer (ipw layout)
  int cap, w, h;
  int n;              // points
};
struct IPTraceArgs {
  int n;                                     // members
  int first[DMV_CT_TRACE_MANY_MAX + 1];      // member k's points are the warps first[k] .. first[k] + m[k].n - 1; first[k] % 4 == 0
  dmv_ip_settings s;
  IPTraceMember m[DMV_CT_TRACE_MANY_MAX];
};
static_assert(sizeof(IPTraceArgs) == 624, "ip_trace_kernel's parameter block");

// A for n members with the call's settings (NULL: defaults), every member empty
void ip_trace_args(IPTraceArgs& A, int n, const dmv_ip_settings* settings);
// member i of A: np points of the array ip (capacity cap) traced against handle c's resident level-0 frame.  Members are set in order.
void ip_trace_member(IPTraceArgs& A, int i, const dmv_ct* c, float* ip, int cap, int np);
// ip_trace_kernel over A's members on handles[0]'s stream, behind the work queued on every other member's stream; each member with a point
// counts one launch.  Does not synchronise.
int ip_trace_launch(dmv_ct* const* hs, const IPTraceArgs& A);
}  // namespace dmv
