// PixelSelector::makeMaps (FullSystem/PixelSelector2.cpp:L94-307) and FullSystem::makeNewTraces (FullSystem.cpp:L1640-1667) on the coarse
// tracker's resident frame.  Bit-identical to the reference: compiled with -fmad=false like ip_trace.cu, and every conversion and comparison
// of the reference is kept (see below).
//
// absSquaredGrad (HessianBlocks.cpp:L169-189) is recomputed where it is read from the resident [I, dx, dy] planes of levels 0-2, with the
// getBGradOnly(I)^2 weight of setting_gammaWeightsPixelSelect; the rows the reference never writes (0 and h_l-1) read as 0.
// makeHists (L94-157): one CTA per 16x16 block (histogram in shared memory, computeHistQuantil), then the 3x3 smoothing, once per call.
//
// select (L311-454) is a serial loop; it reduces to the following.
//  - Scan order: 4pot-blocks in raster order, inside each its 2x2 2pot-blocks, inside each of those its 2x2 pot-blocks, pixels in raster
//    order inside a pot-block.  The pot-grid is uniform (origins at multiples of pot) with partial blocks at the right and bottom edges, so a
//    pot-block (px, py) has the nested key ((py/4)*nx4 + px/4)*16 + ((py/2)&1)*8 + ((px/2)&1)*4 + (py&1)*2 + (px&1); keys of blocks that do
//    not exist at an edge stay empty.  The key order is the scan order.
//  - Level 0 (map = 1): a pot-block picks the first pixel in scan order attaining the maximum of |g.dir2| among pixels with ag0 > TH0*thFactor;
//    strict > from 0, so a dot product of exactly 0 never picks.
//  - Level 1 (map = 2): a 2pot-block picks only if none of its pot-blocks picked (bestIdx3 == -2 after any level-0 candidate).  It picks the
//    first maximum of |g0.dir3| over its pixels in scan order with ag1 > TH1*thFactor.
//  - Level 2 (map = 4): a 4pot-block picks only if none of its pixels was a level-0 or level-1 candidate, then the first maximum of |g0.dir4|
//    with ag2 > TH2*thFactor.
//  - dir2/dir3/dir4 = directions[randomPattern[n2] & 0xF], n2 = the level-0 picks made before the block starts.  With no level-0 pick
//    inside a 2pot- (4pot-) block, n2 is constant over it, so its level-1 (level-2) decision uses one direction.
//  - The serial dependency: a pot-block's 16-bit mask has bit d set when it has a level-0 candidate under directions[d].  A mask is 0 or
//    0xFFFF unless every qualifying pixel has a dot product of exactly 0 with some direction ("mixed", e.g. dx == 0 on 8-bit images).
//    n2 at a block = the prefix sum of the constant blocks' picks + the picks of the mixed blocks before it; only the mixed blocks form a
//    serial chain, walked by one thread from shared memory (ps_chain_kernel).
// The per-level argmax is an atomicMax over (value bits << 32 | ~position in scan order): values are > 0, so their bits order like the
// floats, and the smallest position wins a tie, as the reference's strict >.
// makeMaps' recursion (L203-244) is decided on the device (ps_decide_kernel): recursionsLeft + 1 select passes are queued and the passes after
// the decision to return are no-ops, so the host waits once.  Sub-selection (L248-265): the k-th nonzero map entry in raster order is cleared
// when randomPattern[k] > (unsigned char)(255*quotia), a prefix count over the map.  makeNewTraces' loop: a raster compaction of the nonzero
// entries in [3, w-4) x [3, h-4), the existing ip_init_kernel, and a compaction of the finite energyTH into the caller's pinned output, or,
// for dmv_ct_make_new_traces_store, into an immature-point store's edit staging (ps_store_rows_kernel) in the layout dmv_ip_store_put uploads.
#include "ct_handle.h"
#include "ip_store.h"
#include "ip_trace.h"
#include <cub/device/device_scan.cuh>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

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
  DevBuf<uint8_t> pat;            // PixelSelector::randomPattern (w*h)
  uint8_t* nib = nullptr;         // its low nibbles, two per byte (w*h/2), at pat + w*h: the directions the serial chain reads
  DevBuf<float> ths;              // thsSmoothed (nbW*nbH) and ths (nbW*nbH)
  DevBuf<float> B;                // CalibHessian::B (256)
  DevBuf<uint32_t> mask;          // per pot-block / 2pot-block / 4pot-block: directions with a candidate (w*h + w*h/4 + w*h/16)
  DevBuf<unsigned long long> best;     // per pot-block / 2pot / 4pot: (value bits << 32) | ~position of the first maximum
  DevBuf<unsigned long long> scan_in;  // (w*h+1): constant pick | mixed block << 32 per pot-block key
  DevBuf<unsigned long long> scan;     // (w*h+1): its exclusive prefix of (constant picks | mixed blocks << 32) in nested order
  DevBuf<int2> mixed;             // (w*h): per mixed block in order: (constant-pick prefix, direction mask)
  DevBuf<int> delta;              // (w*h): mixed picks up to and including mixed block j
  DevBuf<int> n2b;                // (w*h+1): level-0 picks before each pot-block in nested order
  DevBuf<float> map;              // selectionMap (w*h)
  DevBuf<int> flag;               // (w*h): scan input
  DevBuf<int> rank;               // (w*h): scan output
  DevBuf<float> cand;             // candidates of makeNewTraces' loop: u | v | type | color*8 | weights*8 | gradH*4 | energyTH | ok  (25 * w*h words)
  DevBuf<PSState> st;
  DevBuf<uint8_t> temp;           // CUB scan storage
  size_t temp_bytes = 0;
  PinnedBuf<float> h_out;         // device-visible: PSState then per point u | v | type | color*8 | weights*8 | gradH*4 | energyTH
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


// PixelSelector2.cpp:L328-344 (double literals converted to float, as Vec2f's constructor does)
__constant__ float c_ps_dir[16][2] = {{0, 1.0000},      {0.3827, 0.9239},  {0.1951, 0.9808},  {0.9239, 0.3827},  {0.7071, 0.7071},  {0.3827, -0.9239},
                                      {0.8315, 0.5556}, {0.8315, -0.5556}, {0.5556, -0.8315}, {0.9808, 0.1951},  {0.9239, -0.3827}, {0.7071, -0.7071},
                                      {0.5556, 0.8315}, {0.9808, -0.1951}, {1.0000, 0.0000},  {0.1951, -0.9808}};

struct PSDev {  // what every kernel reads (by value)
  int w, h, w1, h1, w2, h2, nbW, nbH;
  const float4 *img0, *img1, *img2;
  dmv_ps_settings s;
  float density, thFactor, dw1, dw2;
  const uint8_t *pat, *nib;
  const float* B;
  float *ths, *thsSm;
  uint32_t *mask0, *mask1, *mask2;
  unsigned long long *best0, *best1, *best2;
  unsigned long long *scan_in, *scan;
  int2* mixed;
  int* delta;
  int* n2b;
  float* map;
  int *flag, *rank;
  float* cand;
  PSState* st;
  float* out;
  int out_cap, cand_cap;
};

// CalibHessian::getBGradOnly (HessianBlocks.h:L394-400); int c = color+0.5f converts as x86's cvttss2si does (INT_MIN out of range / NaN)
__device__ __forceinline__ float ps_gw(const float* B, float color) {
  const float cf = color + 0.5f;
  int c = (cf >= -2147483648.f && cf < 2147483648.f) ? (int)cf : INT_MIN;
  if (c < 5) c = 5;
  if (c > 250) c = 250;
  return B[c + 1] - B[c];
}
__device__ __forceinline__ float ps_asg(const PSDev& D, const float4* img, int wl, int hl, int idx) {
  if (idx < wl || idx >= wl * (hl - 1)) return 0.f;
  const float4 p = img[idx];
  float d = p.y * p.y + p.z * p.z;
  if (D.s.gammaWeightsPixelSelect == 1) {
    const float gw = ps_gw(D.B, p.x);
    d *= gw * gw;
  }
  return d;
}
__device__ __forceinline__ int ps_nx4(const PSDev& D, int pot) { return (D.w + 4 * pot - 1) / (4 * pot); }
__device__ __forceinline__ int ps_nkeys(const PSDev& D, int pot) { return ps_nx4(D, pot) * ((D.h + 4 * pot - 1) / (4 * pot)) * 16; }
__device__ __forceinline__ int ps_key(int px, int py, int nx4) {
  return ((py >> 2) * nx4 + (px >> 2)) * 16 + (((py >> 1) & 1) << 3) + (((px >> 1) & 1) << 2) + ((py & 1) << 1) + (px & 1);
}
__device__ __forceinline__ float ps_dot(float gx, float gy, int d) { return fabsf(gx * c_ps_dir[d][0] + gy * c_ps_dir[d][1]); }

// per pixel of select's scan: the border test, the thresholds and the three qualifying tests (L385-425)
struct PSPix {
  bool in, q0, q1, q2;
  float ag0, ag1, ag2, gx, gy;
};
__device__ __forceinline__ PSPix ps_pixel(const PSDev& D, int xf, int yf) {
  PSPix P;
  P.in = !(xf < 4 || xf >= D.w - 5 || yf < 4 || yf > D.h - 4);
  P.q0 = P.q1 = P.q2 = false;
  if (!P.in) return P;
  const int idx = xf + D.w * yf;
  const float pixelTH0 = D.thsSm[xf / 16 + (yf / 16) * D.nbW];
  const float pixelTH1 = pixelTH0 * D.dw1;
  const float pixelTH2 = pixelTH1 * D.dw2;
  P.ag0 = ps_asg(D, D.img0, D.w, D.h, idx);
  P.ag1 = ps_asg(D, D.img1, D.w1, D.h1, (int)(xf * 0.5f + 0.25f) + (int)(yf * 0.5f + 0.25f) * D.w1);
  P.ag2 = ps_asg(D, D.img2, D.w2, D.h2, (int)(xf * 0.25f + 0.125) + (int)(yf * 0.25f + 0.125) * D.w2);   // double, as the reference
  P.q0 = P.ag0 > pixelTH0 * D.thFactor;
  P.q1 = P.ag1 > pixelTH1 * D.thFactor;
  P.q2 = P.ag2 > pixelTH2 * D.thFactor;
  const float4 g = D.img0[idx];
  P.gx = g.y; P.gy = g.z;
  return P;
}
// the directions under which a qualifying pixel is a candidate (dirNorm > 0); setting_selectDirectionDistribution = 0: dirNorm = ag
__device__ __forceinline__ uint32_t ps_bits(const PSDev& D, const PSPix& P, float ag) {
  if (!D.s.selectDirectionDistribution) return ag > 0.f ? 0xFFFFu : 0u;
  uint32_t b = 0;
#pragma unroll
  for (int d = 0; d < 16; d++) b |= (ps_dot(P.gx, P.gy, d) > 0.f ? 1u : 0u) << d;
  return b;
}
__device__ __forceinline__ float ps_norm(const PSDev& D, const PSPix& P, float ag, int d) {
  return D.s.selectDirectionDistribution ? ps_dot(P.gx, P.gy, d) : ag;
}

// ---- makeHists (L94-157)
__global__ void __launch_bounds__(256) ps_hist_kernel(const PSDev D) {
  __shared__ int hist[91];
  const int t = threadIdx.x + 16 * threadIdx.y;
  if (t < 91) hist[t] = 0;
  __syncthreads();
  const int it = blockIdx.x * 16 + threadIdx.x, jt = blockIdx.y * 16 + threadIdx.y;
  if (!(it > D.w - 2 || jt > D.h - 2 || it < 1 || jt < 1)) {
    int g = sqrtf(ps_asg(D, D.img0, D.w, D.h, it + jt * D.w));
    if (g > 48) g = 48;
    atomicAdd(&hist[g + 1], 1);
    atomicAdd(&hist[0], 1);
  }
  __syncthreads();
  if (t == 0) {  // computeHistQuantil (L82-91)
    int th = hist[0] * D.s.minGradHistCut + 0.5f;
    int q = 90;
    for (int i = 0; i < 90; i++) {
      th -= hist[i + 1];
      if (th < 0) { q = i; break; }
    }
    D.ths[blockIdx.x + blockIdx.y * D.nbW] = q + D.s.minGradHistAdd;
  }
}
__global__ void ps_smooth_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nbW * D.nbH) return;
  const int x = i % D.nbW, y = i / D.nbW, w32 = D.nbW, h32 = D.nbH;
  const float* ths = D.ths;
  float sum = 0, num = 0;
  if (x > 0) {
    if (y > 0) { num++; sum += ths[x - 1 + (y - 1) * w32]; }
    if (y < h32 - 1) { num++; sum += ths[x - 1 + (y + 1) * w32]; }
    num++; sum += ths[x - 1 + (y)*w32];
  }
  if (x < w32 - 1) {
    if (y > 0) { num++; sum += ths[x + 1 + (y - 1) * w32]; }
    if (y < h32 - 1) { num++; sum += ths[x + 1 + (y + 1) * w32]; }
    num++; sum += ths[x + 1 + (y)*w32];
  }
  if (y > 0) { num++; sum += ths[x + (y - 1) * w32]; }
  if (y < h32 - 1) { num++; sum += ths[x + (y + 1) * w32]; }
  num++; sum += ths[x + y * w32];
  D.thsSm[x + y * w32] = (sum / num) * (sum / num);
}

// ---- one select pass (pot = st->pot); every kernel is a no-op once makeMaps has returned
__global__ void ps_clear_kernel(const PSDev D) {
  if (D.st->done) return;
  const int n = D.w * D.h;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    D.mask0[i] = 0; D.best0[i] = 0; D.map[i] = 0.f;
    if (i < n / 4) { D.mask1[i] = 0; D.best1[i] = 0; }
    if (i < n / 16) { D.mask2[i] = 0; D.best2[i] = 0; }
  }
}
__global__ void ps_mask_kernel(const PSDev D) {
  if (D.st->done) return;
  const int xf = blockIdx.x * blockDim.x + threadIdx.x, yf = blockIdx.y;
  if (xf >= D.w) return;
  const PSPix P = ps_pixel(D, xf, yf);
  if (!P.q0 && !P.q1 && !P.q2) return;
  const int pot = D.st->pot;
  const int K = ps_key(xf / pot, yf / pot, ps_nx4(D, pot));
  if (P.q0) { const uint32_t b = ps_bits(D, P, P.ag0); if (b) atomicOr(&D.mask0[K], b); }
  if (P.q1) { const uint32_t b = ps_bits(D, P, P.ag1); if (b) atomicOr(&D.mask1[K >> 2], b); }
  if (P.q2) { const uint32_t b = ps_bits(D, P, P.ag2); if (b) atomicOr(&D.mask2[K >> 4], b); }
}
// scan input: constant pick (mask 0xFFFF) in the low word, mixed block in the high word
__global__ void ps_classify_kernel(const PSDev D) {
  const int n = D.w * D.h;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  unsigned long long v = 0;
  if (!D.st->done && i < n) {
    const uint32_t m = D.mask0[i];
    v = (m == 0xFFFFu ? 1ull : 0ull) | ((m != 0 && m != 0xFFFFu) ? (1ull << 32) : 0ull);
  }
  D.scan_in[i] = v;
}
__global__ void ps_scatter_mixed_kernel(const PSDev D) {
  if (D.st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ps_nkeys(D, D.st->pot)) return;
  const uint32_t m = D.mask0[i];
  if (m != 0 && m != 0xFFFFu) {
    const unsigned long long s = D.scan[i];
    D.mixed[(int)(s >> 32)] = make_int2((int)(s & 0xFFFFFFFFu), (int)m);
  }
}
// the serial chain: mixed block j picks when its mask has the bit of randomPattern[n2] & 0xF, n2 = its constant prefix + the mixed picks before it.
// Thread 0 walks it; the block stages each chunk of mixed blocks in shared memory first, so only the nibble load is on the dependent path.
// n2 stays below the pass's level-0 pick count, so only that prefix of the nibbles is staged (use_smem: it fits for every frame size).
constexpr int PS_CHAIN_CHUNK = 1024;
__global__ void __launch_bounds__(1024) ps_chain_kernel(const PSDev D, int use_smem) {
  extern __shared__ uint8_t s_nib[];
  __shared__ int2 s_e[PS_CHAIN_CHUNK];
  __shared__ int s_d[PS_CHAIN_CHUNK];
  if (D.st->done) return;
  const int n = D.w * D.h;
  const unsigned long long tot = D.scan[n];
  const int M = (int)(tot >> 32);
  if (M == 0) return;
  const uint8_t* nib = D.nib;
  if (use_smem) {
    const int bytes = min(n / 2, ((int)(tot & 0xFFFFFFFFu) + M) / 2 + 1);
    for (int i = threadIdx.x; i < bytes; i += blockDim.x) s_nib[i] = nib[i];
    nib = s_nib;
  }
  if (threadIdx.x == 0) D.st->n_mixed += M;
  int delta = 0;
  for (int j0 = 0; j0 < M; j0 += PS_CHAIN_CHUNK) {
    const int m = min(PS_CHAIN_CHUNK, M - j0);
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) s_e[i] = D.mixed[j0 + i];
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int j = 0; j < m; j++) {
        const int2 e = s_e[j];
        const int n2 = e.x + delta;
        delta += (e.y >> ((nib[n2 >> 1] >> ((n2 & 1) << 2)) & 0xF)) & 1;
        s_d[j] = delta;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) D.delta[j0 + i] = s_d[i];
  }
}
__global__ void ps_resolve_kernel(const PSDev D) {
  if (D.st->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > ps_nkeys(D, D.st->pot)) return;
  const unsigned long long s = D.scan[i];
  const int m = (int)(s >> 32);
  D.n2b[i] = (int)(s & 0xFFFFFFFFu) + (m > 0 ? D.delta[m - 1] : 0);
}
__device__ __forceinline__ unsigned long long ps_pack(float v, unsigned pos) { return ((unsigned long long)__float_as_uint(v) << 32) | (0xFFFFFFFFu - pos); }
__global__ void ps_pick_kernel(const PSDev D) {
  if (D.st->done) return;
  const int xf = blockIdx.x * blockDim.x + threadIdx.x, yf = blockIdx.y;
  if (xf >= D.w) return;
  const PSPix P = ps_pixel(D, xf, yf);
  if (!P.q0 && !P.q1 && !P.q2) return;
  const int pot = D.st->pot;
  const int px = xf / pot, py = yf / pot;
  const int K = ps_key(px, py, ps_nx4(D, pot));
  const unsigned pos = (unsigned)K * pot * pot + (yf - py * pot) * pot + (xf - px * pot);
  const int* n2b = D.n2b;
  if (P.q0 && n2b[K + 1] != n2b[K]) {
    const float v = ps_norm(D, P, P.ag0, D.pat[n2b[K]] & 0xF);
    if (v > 0.f) atomicMax(&D.best0[K], ps_pack(v, pos));
  }
  const int J = K >> 2, I = K >> 4;
  if (P.q1 && n2b[4 * J + 4] == n2b[4 * J]) {
    const float v = ps_norm(D, P, P.ag1, D.pat[n2b[4 * J]] & 0xF);
    if (v > 0.f) atomicMax(&D.best1[J], ps_pack(v, pos));
  }
  if (P.q2 && n2b[16 * I + 16] == n2b[16 * I]) {
    const int d = D.pat[n2b[16 * I]] & 0xF;
    const uint32_t l1 = D.mask1[4 * I] | D.mask1[4 * I + 1] | D.mask1[4 * I + 2] | D.mask1[4 * I + 3];
    if (!((l1 >> d) & 1)) {
      const float v = ps_norm(D, P, P.ag2, d);
      if (v > 0.f) atomicMax(&D.best2[I], ps_pack(v, pos));
    }
  }
}
__device__ __forceinline__ int ps_unpos(const PSDev& D, unsigned long long b, int pot) {
  const unsigned pos = 0xFFFFFFFFu - (unsigned)(b & 0xFFFFFFFFu);
  const int K = pos / (pot * pot), r = pos % (pot * pot);
  const int nx4 = ps_nx4(D, pot), q = K >> 4, sub = K & 15;
  const int px = (q % nx4) * 4 + ((sub >> 2) & 1) * 2 + (sub & 1);
  const int py = (q / nx4) * 4 + ((sub >> 3) & 1) * 2 + ((sub >> 1) & 1);
  return (px * pot + r % pot) + (py * pot + r / pot) * D.w;
}
__global__ void ps_finish_kernel(const PSDev D) {
  if (D.st->done) return;
  const int K = blockIdx.x * blockDim.x + threadIdx.x;
  const int pot = D.st->pot;
  if (K >= ps_nkeys(D, pot)) return;
  if (D.best0[K]) D.map[ps_unpos(D, D.best0[K], pot)] = 1.f;
  if ((K & 3) == 0 && D.best1[K >> 2]) { D.map[ps_unpos(D, D.best1[K >> 2], pot)] = 2.f; atomicAdd(&D.st->n3, 1); }
  if ((K & 15) == 0 && D.best2[K >> 4]) { D.map[ps_unpos(D, D.best2[K >> 4], pot)] = 4.f; atomicAdd(&D.st->n4, 1); }
}
// makeMaps after select (L205-244): recurse (next pass) or return
__global__ void ps_decide_kernel(const PSDev D) {
  PSState* S = D.st;
  if (S->done) return;
  const int pot = S->pot;
  const int n2 = D.n2b[ps_nkeys(D, pot)];
  const float numHave = (float)(n2 + S->n3 + S->n4);
  const float numWant = D.density;
  const float quotia = numWant / numHave;
  const float K = numHave * (pot + 1) * (pot + 1);
  int ideal = sqrtf(K / numWant) - 1;
  if (ideal < 1) ideal = 1;
  S->n3 = 0; S->n4 = 0;
  if (S->recLeft > 0 && quotia > 1.25 && pot > 1) {
    if (ideal >= pot) ideal = pot - 1;
    S->pot = ideal; S->recLeft--;
  } else if (S->recLeft > 0 && quotia < 0.25) {
    if (ideal <= pot) ideal = pot + 1;
    S->pot = ideal; S->recLeft--;
  } else {
    S->done = 1; S->quotia = quotia; S->ideal = ideal; S->numHaveSub = (int)numHave;
  }
}

// ---- sub-selection (L247-265) and makeNewTraces' loop (FullSystem.cpp:L1652-1663)
__device__ __forceinline__ bool ps_thin(const PSState* S) { return (double)S->quotia < 0.95; }
__global__ void ps_flag_nonzero_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.w * D.h) return;
  D.flag[i] = (ps_thin(D.st) && D.map[i] != 0.f) ? 1 : 0;
}
__global__ void ps_thin_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.w * D.h || !D.flag[i]) return;
  const unsigned char charTH = (unsigned char)(int)(255 * D.st->quotia);
  if (D.pat[D.rank[i]] > charTH) {
    D.map[i] = 0.f;
    atomicSub(&D.st->numHaveSub, 1);
  }
}
__global__ void ps_flag_window_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.w * D.h) return;
  const int x = i % D.w, y = i / D.w;
  D.flag[i] = (x >= 3 && x < D.w - 4 && y >= 3 && y < D.h - 4 && D.map[i] != 0.f) ? 1 : 0;
}
__global__ void ps_scatter_cand_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = D.w * D.h;
  if (i >= n) return;
  const int r = D.rank[i];
  if (i == n - 1) D.st->n_cand = r + D.flag[i];
  if (!D.flag[i]) return;
  const size_t C = D.cand_cap;
  reinterpret_cast<int*>(D.cand)[r] = i % D.w;
  reinterpret_cast<int*>(D.cand + C)[r] = i / D.w;
  D.cand[2 * C + r] = D.map[i];
}
__global__ void ps_flag_ok_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.w * D.h) return;
  D.flag[i] = (i < D.st->n_cand && reinterpret_cast<const int*>(D.cand + (size_t)24 * D.cand_cap)[i]) ? 1 : 0;
}
// the points into the pinned output: u | v | type | color*8 | weights*8 | gradH*4 | energyTH (capacity out_cap), then the state
__global__ void ps_scatter_out_kernel(const PSDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = D.w * D.h;
  if (i >= n) return;
  const int r = D.rank[i];
  if (i == n - 1) D.st->n_points = r + D.flag[i];
  if (!D.flag[i] || r >= D.out_cap) return;
  const size_t C = D.cand_cap, O = D.out_cap;
  const float* c = D.cand;
  float* o = D.out + sizeof(PSState) / sizeof(float);
  o[r] = c[i]; o[O + r] = c[C + i]; o[2 * O + r] = c[2 * C + i];
#pragma unroll
  for (int k = 0; k < 8; k++) { o[(3 + k) * O + r] = c[3 * C + 8 * (size_t)i + k]; o[(11 + k) * O + r] = c[11 * C + 8 * (size_t)i + k]; }
#pragma unroll
  for (int k = 0; k < 4; k++) o[(19 + k) * O + r] = c[19 * C + 4 * (size_t)i + k];
  o[23 * O + r] = c[23 * C + i];
}
// the points into an immature-point store's edit staging (dmv_ct_make_new_traces_store): the rows dmv_ip_store_put uploads, in the ipw
// layout of capacity m (the point count), u and v as floats, the ImmaturePoint constructor's in/out values (ImmaturePoint.cpp:L39-41) and
// set = slot; type into its own m words
__global__ void ps_store_rows_kernel(const PSDev D, float* __restrict__ rows, float* __restrict__ type, int m, int slot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.w * D.h || !D.flag[i]) return;
  const int r = D.rank[i];
  if (r >= m) return;
  const size_t C = D.cand_cap, M = m;
  const float* c = D.cand;
  rows[ipw::u * M + r] = (float)reinterpret_cast<const int*>(c)[i];
  rows[ipw::v * M + r] = (float)reinterpret_cast<const int*>(c + C)[i];
  type[r] = c[2 * C + i];
#pragma unroll
  for (int k = 0; k < 8; k++) { rows[ipw::color * M + 8 * r + k] = c[3 * C + 8 * (size_t)i + k]; rows[ipw::weights * M + 8 * r + k] = c[11 * C + 8 * (size_t)i + k]; }
#pragma unroll
  for (int k = 0; k < 4; k++) rows[ipw::gradH * M + 4 * r + k] = c[19 * C + 4 * (size_t)i + k];
  rows[ipw::energyTH * M + r] = c[23 * C + i];
  rows[ipw::idepth_min * M + r] = 0.f;
  rows[ipw::idepth_max * M + r] = __int_as_float(0x7FC00000);   // NaN, as the host's quiet NaN
  rows[ipw::quality * M + r] = 10000.f;
  reinterpret_cast<int*>(rows + ipw::status * M)[r] = 5;        // IPS_UNINITIALIZED
  rows[ipw::uv * M + 2 * r] = 0.f;
  rows[ipw::uv * M + 2 * r + 1] = 0.f;
  rows[ipw::interval * M + r] = 0.f;
  reinterpret_cast<int*>(rows + ipw::set * M)[r] = slot;
}
__global__ void ps_init_state_kernel(PSState* S, int pot, int recLeft) {
  S->pot = pot; S->recLeft = recLeft; S->done = 0; S->n3 = 0; S->n4 = 0; S->numHaveSub = 0; S->ideal = pot; S->quotia = 0.f;
  S->n_cand = 0; S->n_points = 0; S->n_mixed = 0; S->pad = 0;
}

// ---- host side
// glibc's random(3) TYPE_3 generator restated (srand(seed); rand() & 0xFF per entry), without touching the process's rand() state
static void ps_random_pattern(uint8_t* out, size_t n, unsigned seed) {
  // glibc random_r.c, TYPE_3 (degree 31, separation 3): the state is seeded by the Park-Miller recurrence, 310 outputs are discarded, and
  // each rand() returns (r[i-31] + r[i-3]) >> 1 in 32-bit arithmetic
  std::vector<int32_t> r(344 + n);
  if (seed == 0) seed = 1;
  r[0] = (int32_t)seed;
  for (int i = 1; i < 31; i++) {
    const long long hi = r[i - 1] / 127773, lo = r[i - 1] % 127773;
    long long word = 16807 * lo - 2836 * hi;
    if (word < 0) word += 2147483647;
    r[i] = (int32_t)word;
  }
  for (int i = 31; i < 34; i++) r[i] = r[i - 31];
  for (size_t i = 34; i < 344 + n; i++) r[i] = (int32_t)((uint32_t)r[i - 31] + (uint32_t)r[i - 3]);
  for (size_t k = 0; k < n; k++) out[k] = (uint8_t)(((uint32_t)r[344 + k] >> 1) & 0xFF);
}

// dynamic shared memory of ps_chain_kernel: one value for the process (the attribute belongs to the kernel, not to a handle)
static const int PS_SMEM_MAX = 200 * 1024;

void CTPartDelete::operator()(PSScratch* p) const { delete p; }

// S (empty) for a w x h frame, with the random pattern built; S.w / S.h are set only once all of it is
static int ps_alloc(PSScratch& S, int w, int h) {
  const size_t n = (size_t)w * h;
  CK(S.pat.alloc(n + n / 2));
  S.nib = S.pat + n;
  CK(S.ths.alloc(2 * (n / 256)));
  CK(S.B.alloc(256));
  CK(S.mask.alloc(n + n / 4 + n / 16));
  CK(S.best.alloc(n + n / 4 + n / 16));
  CK(S.scan.alloc(n + 1));
  CK(S.scan_in.alloc(n + 1));
  CK(S.mixed.alloc(n));
  CK(S.delta.alloc(n));
  CK(S.n2b.alloc(n + 1));
  CK(S.map.alloc(n));
  CK(S.flag.alloc(n));
  CK(S.rank.alloc(n));
  CK(S.cand.alloc(25 * n));
  CK(S.st.alloc(1));
  size_t t1 = 0, t2 = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, t1, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n + 1));
  CK(cub::DeviceScan::ExclusiveSum(nullptr, t2, (const int*)nullptr, (int*)nullptr, (int)n));
  S.temp_bytes = std::max(t1, t2);
  CK(S.temp.alloc(S.temp_bytes));
  std::vector<uint8_t> pat(n + n / 2);
  ps_random_pattern(pat.data(), n, 3141592);   // PixelSelector::PixelSelector (L43-47)
  for (size_t i = 0; i < n / 2; i++) pat[n + i] = (uint8_t)((pat[2 * i] & 0xF) | ((pat[2 * i + 1] & 0xF) << 4));
  CK(cudaMemcpy(S.pat, pat.data(), n + n / 2, cudaMemcpyHostToDevice));
  S.smem_chain = n / 2 <= (size_t)PS_SMEM_MAX;
  if (S.smem_chain) CK(cudaFuncSetAttribute(ps_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PS_SMEM_MAX));
  S.w = w; S.h = h;
  return DMV_OK;
}

// what every kernel of the call reads
static PSDev ps_dev(const PSArgs& A, PSScratch& S) {
  const int w = A.w, h = A.h, n = w * h;
  PSDev D;
  D.w = w; D.h = h; D.w1 = w >> 1; D.h1 = h >> 1; D.w2 = w >> 2; D.h2 = h >> 2; D.nbW = w / 16; D.nbH = h / 16;
  D.img0 = A.img[0]; D.img1 = A.img[1]; D.img2 = A.img[2];
  D.s = A.s; D.density = A.density; D.thFactor = A.thFactor;
  D.dw1 = A.s.gradDownweightPerLevel; D.dw2 = D.dw1 * D.dw1;
  D.pat = S.pat; D.nib = S.nib; D.B = S.B;
  D.thsSm = S.ths; D.ths = S.ths + n / 256;
  D.mask0 = S.mask; D.mask1 = S.mask + n; D.mask2 = S.mask + n + n / 4;
  D.best0 = S.best; D.best1 = S.best + n; D.best2 = S.best + n + n / 4;
  D.scan_in = S.scan_in; D.scan = S.scan; D.mixed = S.mixed; D.delta = S.delta; D.n2b = S.n2b; D.map = S.map; D.flag = S.flag; D.rank = S.rank;
  D.cand = S.cand; D.cand_cap = n; D.st = S.st;
  D.out = S.h_out; D.out_cap = A.out_cap;
  return D;
}

// the selection up to its final compaction: makeMaps, the sub-selection, the raster loop with ip_init_kernel, and the scan of the points with
// a finite energyTH (flag, rank over the candidates).  *kernels = kernels launched (CUB's own launches not counted)
static cudaError_t ps_select_launch(const PSArgs& A, const PSDev& D, PSScratch& S, cudaStream_t s, int* kernels) {
  const int w = A.w, h = A.h, n = w * h;
  int k = 0;
  cudaError_t e;
  const dim3 rows((w + 127) / 128, h);
  const int pb = (n + 255) / 256, kb = (n + 1 + 255) / 256;
  ps_init_state_kernel<<<1, 1, 0, s>>>(S.st, A.potential, A.recursionsLeft); k++;
  ps_hist_kernel<<<dim3(D.nbW, D.nbH), dim3(16, 16), 0, s>>>(D); k++;
  ps_smooth_kernel<<<(D.nbW * D.nbH + 127) / 128, 128, 0, s>>>(D); k++;
  for (int pass = 0; pass <= A.recursionsLeft; pass++) {
    ps_clear_kernel<<<264, 512, 0, s>>>(D); k++;
    ps_mask_kernel<<<rows, 128, 0, s>>>(D); k++;
    ps_classify_kernel<<<kb, 256, 0, s>>>(D); k++;
    size_t tb = S.temp_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(S.temp, tb, S.scan_in.get(), S.scan.get(), n + 1, s)) != cudaSuccess) return e;
    ps_scatter_mixed_kernel<<<pb, 256, 0, s>>>(D); k++;
    ps_chain_kernel<<<1, 1024, S.smem_chain ? n / 2 : 0, s>>>(D, S.smem_chain ? 1 : 0); k++;
    ps_resolve_kernel<<<kb, 256, 0, s>>>(D); k++;
    ps_pick_kernel<<<rows, 128, 0, s>>>(D); k++;
    ps_finish_kernel<<<pb, 256, 0, s>>>(D); k++;
    ps_decide_kernel<<<1, 1, 0, s>>>(D); k++;
  }
  size_t tb = S.temp_bytes;
  ps_flag_nonzero_kernel<<<pb, 256, 0, s>>>(D); k++;
  if ((e = cub::DeviceScan::ExclusiveSum(S.temp, tb, S.flag.get(), S.rank.get(), n, s)) != cudaSuccess) return e;
  ps_thin_kernel<<<pb, 256, 0, s>>>(D); k++;
  ps_flag_window_kernel<<<pb, 256, 0, s>>>(D); k++;
  if ((e = cub::DeviceScan::ExclusiveSum(S.temp, tb, S.flag.get(), S.rank.get(), n, s)) != cudaSuccess) return e;
  ps_scatter_cand_kernel<<<pb, 256, 0, s>>>(D); k++;
  IPInitArgs I;
  const size_t C = n;
  I.n = n; I.w = w; I.n_dev = &S.st->n_cand;
  I.outlierTHSumComponent = 50.f * 50.f; I.outlierTH = 12.f * 12.f; I.overallEnergyTHWeight = 1.f;  // util/settings.cpp:L111-114, L159
  I.u = reinterpret_cast<const int*>(S.cand.get()); I.v = reinterpret_cast<const int*>(S.cand + C);
  I.color = S.cand + 3 * C; I.weights = S.cand + 11 * C; I.gradH = S.cand + 19 * C; I.energyTH = S.cand + 23 * C;
  I.ok = reinterpret_cast<int*>(S.cand + 24 * C);
  I.img = A.img[0];
  launch_ip_init(I, s); k++;
  ps_flag_ok_kernel<<<pb, 256, 0, s>>>(D); k++;
  if ((e = cub::DeviceScan::ExclusiveSum(S.temp, tb, S.flag.get(), S.rank.get(), n, s)) != cudaSuccess) return e;
  *kernels = k;
  return cudaGetLastError();
}

// every launch of dmv_ct_make_new_traces: the points and the final PSState land in S.h_out, which the host reads after one stream
// synchronisation; the selection map stays in S.map.  *kernels = kernels launched (CUB's own launches not counted)
static cudaError_t ps_launch(const PSArgs& A, PSScratch& S, cudaStream_t s, int* kernels) {
  const PSDev D = ps_dev(A, S);
  cudaError_t e;
  if ((e = ps_select_launch(A, D, S, s, kernels)) != cudaSuccess) return e;
  ps_scatter_out_kernel<<<(A.w * A.h + 255) / 256, 256, 0, s>>>(D); (*kernels)++;
  if ((e = cudaMemcpyAsync(S.h_out, S.st, sizeof(PSState), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
  return cudaGetLastError();
}

}  // namespace dmv

using namespace dmv;

void dmv_ps_default_settings(dmv_ps_settings* s) {
  if (!s) return;
  s->minGradHistCut = 0.5f; s->minGradHistAdd = 7.f; s->gradDownweightPerLevel = 0.75f;   // util/settings.cpp:L144, L167-170
  s->selectDirectionDistribution = 1; s->gammaWeightsPixelSelect = 1;
}

// the checks of dmv_ct_make_new_traces (outputs_optional: those of dmv_ct_make_new_traces_store, where every per-point output may be NULL);
// *st = the settings.  No CUDA call.
static int ps_check(const dmv_ct* c, const dmv_new_traces_args* a, bool outputs_optional, dmv_ps_settings* st) {
  if (c->cfg.levels < 3) return set_error(DMV_ERR_INVALID, "pixel selection reads levels 0-2: the handle has %d", c->cfg.levels);
  const int w = c->w[0], h = c->h[0];
  if (w % 16 || h % 16) return set_error(DMV_ERR_INVALID, "pixel selection needs w and h divisible by 16 (%d x %d)", w, h);
  const bool outputs = a->u && a->v && a->type && a->color8 && a->weights8 && a->gradH4 && a->energyTH;
  if (!a->potential || !a->n || !a->numPointsTotal || a->cap < 0 || (a->cap > 0 && !outputs_optional && !outputs))
    return set_error(DMV_ERR_INVALID, "null argument");
  if (*a->potential < 1) return set_error(DMV_ERR_INVALID, "potential %d < 1", *a->potential);
  if (!(a->density > 0.f) || !std::isfinite(a->density)) return set_error(DMV_ERR_INVALID, "density must be finite and > 0");
  if (!(a->thFactor > 0.f) || !std::isfinite(a->thFactor)) return set_error(DMV_ERR_INVALID, "thFactor must be finite and > 0");
  if (a->recursionsLeft < 0 || a->recursionsLeft > 8) return set_error(DMV_ERR_INVALID, "recursionsLeft must be in 0..8");
  if (a->settings) *st = *a->settings; else dmv_ps_default_settings(st);
  if (!(st->minGradHistCut < 0.99f) || !std::isfinite(st->minGradHistCut) || !std::isfinite(st->minGradHistAdd) || !std::isfinite(st->gradDownweightPerLevel))
    return set_error(DMV_ERR_INVALID, "bad dmv_ps_settings");
  return DMV_OK;
}

// the handle's scratch for its frame size with room for out_cap points in h_out, the staging free, and B on its way; *A = the launch's arguments
static int ps_prepare(dmv_ct* c, const dmv_new_traces_args* a, const dmv_ps_settings& st, int out_cap, PSArgs* A) {
  const int w = c->w[0], h = c->h[0];
  CK(cudaSetDevice(c->device));
  if (!c->ps) c->ps.reset(new PSScratch());
  PSScratch& P = *c->ps;
  if (P.w != w || P.h != h) {
    P = PSScratch();
    const int rc = ps_alloc(P, w, h);
    if (rc != DMV_OK) { P = PSScratch(); return rc; }
  }
  CK(P.h_out.reserve(sizeof(PSState) / sizeof(float) + 24 * (size_t)std::max(out_cap, 1)));
  CK(ct_wait_staging(c));
  float B[256];
  for (int i = 0; i < 256; i++) B[i] = a->B ? a->B[i] : (float)i;   // CalibHessian's constructor: B[i] = i
  CK(cudaMemcpyAsync(P.B, B, sizeof(B), cudaMemcpyHostToDevice, c->stream));
  A->w = w; A->h = h;
  for (int l = 0; l < 3; l++) A->img[l] = c->d_img[l];
  A->s = st; A->density = a->density; A->thFactor = a->thFactor; A->recursionsLeft = a->recursionsLeft; A->potential = *a->potential;
  A->out_cap = out_cap;
  return DMV_OK;
}

// FullSystem::makeNewTraces on the resident frame
int dmv_ct_make_new_traces(dmv_ct* c, const dmv_new_traces_args* a) {
  if (!c || !a) return set_error(DMV_ERR_INVALID, "null argument");
  dmv_ps_settings st;
  int rc = ps_check(c, a, false, &st);
  if (rc != DMV_OK) return rc;
  const int w = c->w[0], h = c->h[0];
  const int out_cap = std::min(a->cap, w * h);
  PSArgs A;
  rc = ps_prepare(c, a, st, out_cap, &A);
  if (rc != DMV_OK) return rc;
  PSScratch& P = *c->ps;
  int kernels = 0;
  CK(ps_launch(A, P, c->stream, &kernels));
  c->launches += kernels;
  if (a->map) CK(cudaMemcpyAsync(a->map, P.map, sizeof(float) * (size_t)w * h, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  PSState S;
  std::memcpy(&S, P.h_out, sizeof(S));
  *a->n = S.n_points;
  // on overflow the selector's state stays as it was, so a retry with a larger cap continues from the same potential
  if (S.n_points > a->cap) return set_error(DMV_ERR_INVALID, "%d new points exceed cap %d", S.n_points, a->cap);
  *a->potential = S.ideal;
  *a->numPointsTotal = S.numHaveSub;
  const size_t n = (size_t)S.n_points, O = out_cap;
  const float* o = P.h_out + sizeof(PSState) / sizeof(float);
  std::memcpy(a->u, o, 4 * n); std::memcpy(a->v, o + O, 4 * n); std::memcpy(a->type, o + 2 * O, 4 * n);
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 8; k++) { a->color8[8 * i + k] = o[(3 + k) * O + i]; a->weights8[8 * i + k] = o[(11 + k) * O + i]; }
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 4; k++) a->gradH4[4 * i + k] = o[(19 + k) * O + i];
  std::memcpy(a->energyTH, o + 23 * O, 4 * n);
  return DMV_OK;
}

// makeNewTraces straight into slot `slot` of an immature-point store: the selection as above, its point count read back (synchronisation 1),
// ps_store_rows_kernel in place of ps_scatter_out_kernel writing the slot's rows into the store's edit staging, then the store's edit with
// the requested outputs read from the slot's rows (synchronisation 2)
int dmv_ct_make_new_traces_store(dmv_ct* c, dmv_ip_store* s, int slot, const dmv_new_traces_args* a) {
  if (!c || !s || !a) return set_error(DMV_ERR_INVALID, "null argument");
  dmv_ps_settings st;
  int rc = ps_check(c, a, true, &st);
  if (rc != DMV_OK) return rc;
  if (slot < 0 || slot >= DMV_IP_STORE_SLOTS) return set_error(DMV_ERR_INVALID, "slot %d: expected 0 to %d", slot, DMV_IP_STORE_SLOTS - 1);
  if (s->device != c->device) return set_error(DMV_ERR_INVALID, "the store is on device %d, the handle on device %d", s->device, c->device);
  const bool outputs = a->u || a->v || a->type || a->color8 || a->weights8 || a->gradH4 || a->energyTH;
  const int w = c->w[0], h = c->h[0], npx = w * h;
  PSArgs A;
  rc = ps_prepare(c, a, st, 0, &A);
  if (rc != DMV_OK) return rc;
  PSScratch& P = *c->ps;
  const PSDev D = ps_dev(A, P);
  int kernels = 0;
  CK(ps_select_launch(A, D, P, c->stream, &kernels));
  // the point count = rank + flag of the last candidate index, read beside the state
  int* cnt = reinterpret_cast<int*>(P.h_out + sizeof(PSState) / sizeof(float));
  CK(cudaMemcpyAsync(P.h_out, P.st, sizeof(PSState), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(cnt, P.rank + (npx - 1), sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(cnt + 1, P.flag + (npx - 1), sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  if (a->map) CK(cudaMemcpyAsync(a->map, P.map, sizeof(float) * (size_t)npx, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  PSState S;
  std::memcpy(&S, P.h_out, sizeof(S));
  const int m = cnt[0] + cnt[1];
  *a->n = m;
  if (outputs && m > a->cap) {   // as dmv_ct_make_new_traces: the store and the selector's state stay as they were
    c->launches += kernels;
    return set_error(DMV_ERR_INVALID, "%d new points exceed cap %d", m, a->cap);
  }
  float *rows = nullptr, *type = nullptr;
  rc = ip_store_rows_stage(s, slot, m, &rows, &type);
  if (rc != DMV_OK) return rc;
  ps_store_rows_kernel<<<(npx + 255) / 256, 256, 0, s->stream>>>(D, rows, type, m, slot);
  CK(cudaGetLastError());
  c->launches += kernels + 1;
  rc = ip_store_rows_put(s, slot, m, a);
  if (rc != DMV_OK) return rc;
  *a->potential = S.ideal;
  *a->numPointsTotal = S.numHaveSub;
  return DMV_OK;
}
