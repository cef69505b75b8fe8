// device-side PixelSelector::makeMaps + FullSystem::makeNewTraces (ps_select.cu): arguments and scratch, shared with the C ABI in ct_kernels.cu
#pragma once
#include "../../include/dmvio_b200.h"
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>
namespace dmv {
// makeMaps' running state on the device: the recursion is decided there, so the host learns it only at the end
struct PSState {
  int pot;          // potential of the current select pass
  int recLeft;      // recursions left
  int done;         // makeMaps has returned: later passes are no-ops
  int n3, n4;       // level-1 / level-2 picks of the current pass (level 0: the n2 prefix)
  int numHaveSub;   // makeMaps' return value
  int ideal;        // idealPotential = the potential makeMaps leaves behind
  float quotia;
  int n_cand;       // nonzero map entries inside makeNewTraces' raster window
  int n_points;     // of those, points with a finite energyTH
  int n_mixed;      // mixed pot-blocks met, summed over the select passes (the serial chain's length)
  int pad;
};
// per-handle scratch, allocated on first use for the handle's level-0 size
struct PSScratch {
  int w = 0, h = 0;
  uint8_t* pat = nullptr;         // PixelSelector::randomPattern (w*h)
  uint8_t* nib = nullptr;         // its low nibbles, two per byte (w*h/2): the directions the serial chain reads
  float* ths = nullptr;           // thsSmoothed (nbW*nbH) and ths (nbW*nbH)
  float* B = nullptr;             // CalibHessian::B (256)
  uint32_t* mask = nullptr;       // per pot-block / 2pot-block / 4pot-block: directions with a candidate (w*h + w*h/4 + w*h/16)
  unsigned long long* best = nullptr;  // per pot-block / 2pot / 4pot: (value bits << 32) | ~position of the first maximum
  unsigned long long* scan_in = nullptr;  // (w*h+1): constant pick | mixed block << 32 per pot-block key
  unsigned long long* scan = nullptr;  // (w*h+1): its exclusive prefix of (constant picks | mixed blocks << 32) in nested order
  int2* mixed = nullptr;          // (w*h): per mixed block in order: (constant-pick prefix, direction mask)
  int* delta = nullptr;           // (w*h): mixed picks up to and including mixed block j
  int* n2b = nullptr;             // (w*h+1): level-0 picks before each pot-block in nested order
  float* map = nullptr;           // selectionMap (w*h)
  int* flag = nullptr;            // (w*h): scan input
  int* rank = nullptr;            // (w*h): scan output
  float* cand = nullptr;          // candidates of makeNewTraces' loop: u | v | type | color*8 | weights*8 | gradH*4 | energyTH | ok  (25 * w*h words)
  PSState* st = nullptr;
  void* temp = nullptr;           // CUB scan storage
  size_t temp_bytes = 0;
  float* h_out = nullptr;         // pinned, device-visible: PSState then per point u | v | type | color*8 | weights*8 | gradH*4 | energyTH
  int h_cap = 0;
  bool smem_chain = false;        // the chain stages the nibbles in shared memory (w*h/2 <= 200 KB); larger frames read them from global memory
};
struct PSArgs {
  int w, h;
  const float4* img[3];           // the resident frame's levels 0-2 (I, dx, dy, 0)
  dmv_ps_settings s;
  float density, thFactor;
  int recursionsLeft, potential;
  int out_cap;                    // points written to h_out (min(cap, w*h))
};
void ps_free(PSScratch& S);
// allocates S for a w x h frame and builds the random pattern; returns the first CUDA error
cudaError_t ps_alloc(PSScratch& S, int w, int h);
cudaError_t ps_ensure_out(PSScratch& S, int cap);
// every launch of the call: the points and the final PSState land in S.h_out, which the host reads after one stream synchronisation;
// the selection map stays in S.map.  *kernels = kernels launched (CUB's own launches not counted)
cudaError_t ps_launch(const PSArgs& A, PSScratch& S, cudaStream_t s, int* kernels);
// glibc's random(3) TYPE_3 generator restated (srand(seed); rand() & 0xFF per entry), without touching the process's rand() state
void ps_random_pattern(uint8_t* out, size_t n, unsigned seed);
}  // namespace dmv
