// ba_fused_kernel — one launch = one Gauss-Newton linearisation of the whole window (DESIGN.md §4):
//   FullSystem::linearizeAll (FullSystemOptimize.cpp:L150-218) + EFResidual::takeDataF + AccumulatedTopHessianSSE::addPoint<0/2> +
//   AccumulatedSCHessianSSE::addPoint + both stitchDouble passes (AccumulatedTopHessian.cpp:L241-303, AccumulatedSCHessian.cpp:L78-157)
//   + the point half of resubstituteF_MT / doStepFromBackup of the PREVIOUS iteration (EnergyFunctional.cpp:L295-321).
//
// Design: ONE THREAD PER POINT-RESIDUAL.  A residual is a ~1000-instruction chain whose reductions over the 8 pattern pixels
// stay in registers (no shuffles, nothing per-residual is computed twice), and the 16 / 32 residuals of one (host, target) pair sit in
// adjacent lanes, so the pair's 13x13 block is reduced with a transposing butterfly (96 exchanges per pair instead of 96 x log2 P).
//
//   chunk    P consecutive points of one host frame h; CTA = P x (nf-1) threads, lane = point, (half-)warp = target frame
//   phase A  per thread: optional fused resubstitute + step, PointFrameResidual::linearize (Residuals.cpp:L78-274): FEJ centre
//            projection, 8 pattern pixels x 4 float4 taps, Huber, classification; per-residual outputs; JpJdF; the residual's 91
//            AccumulatorApprox entries (MatrixAccumulators.h:L754-915) summed over the pair's lanes -> shared memory
//   phase B  per point: Hdd / bd / Hcd, HdiF, bdSum (AccumulatedSCHessian.cpp:L36-58) and its Schur vector in ABSOLUTE frame
//            coordinates w_p = [Hcd | sum_t adHost JpJdF_t | adTarget JpJdF_t ... | bdSum]  -> global (transposed for phase E)
//   phase C  the chunk's pair blocks pushed through the adjoints IN THE CTA (fp64): contributions to H[h,h], H[h,t], H[t,t], H[.,C], b
//            are written to the chunk's partial blob with plain coalesced stores — no atomics, no accumulators to zero
//   -------- grid barrier (cooperative launch; every CTA is resident) --------
//   phase D  every final entry of H_top / b_top = fixed-order fp64 sum of the chunk partials that touch it: a warp per entry
//   phase E  Schur complement [H_sc | b_sc] = sum_p HdiF w_p w_p^T as 4x4 tiles, one CTA per tile over ALL points (replaces the nf^3
//            accD blocks and their stitch)
//   every result entry has exactly one producing warp, which also streams it into the caller's pinned host buffer and, on a sharded
//   window, exchanges it with the peer GPUs (LL packets over NVLink peer memory, bounded spin).
// Results are bit-reproducible run to run (no atomics anywhere on the data path).
#include "ba_common.cuh"
#include <cstdlib>
#include <mutex>
#include <type_traits>

namespace dmv {

// ---------------------------------------------------------------------------------------------------------------------------
// compile-time helpers
// ---------------------------------------------------------------------------------------------------------------------------
template <int K, int END, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (K < END) {
    f(std::integral_constant<int, K>{});
    static_for<K + 1, END>(f);
  }
}
__host__ __device__ constexpr int top_row(int k) {  // packed upper-triangular index (rows 0..9, columns r..12) -> row
  int r = 0;
  while (r < 9 && k >= top_off(r + 1)) r++;
  return r;
}
__host__ __device__ constexpr int top_col(int k) { return top_row(k) + k - top_off(top_row(k)); }

struct PixSums {  // the 2x2 / 2x1 sums of RawResidualJacobian (RawResidualJacobian.h:L49-59) + right-hand sides
  float JI00, JI10, JI11, JabJI00, JabJI01, JabJI10, JabJI11, Jab00, Jab01, Jab11, JIr0, JIr1, Jabr0, Jabr1, rr;
};

// entry K of the residual's contribution to the pair's symmetric 13x13 block [C4 | xi6 | a b | r]
template <int K>
__device__ __forceinline__ float top_entry(const float (&x)[10], const float (&y)[10], const float (&al)[10], const float (&be)[10], const PixSums& s) {
  if constexpr (K < TOP_TRI) {
    constexpr int r = top_row(K), c = top_col(K);
    if constexpr (c < 10) return al[r] * x[c] + be[r] * y[c];
    else if constexpr (c == 10) return x[r] * s.JabJI00 + y[r] * s.JabJI01;
    else if constexpr (c == 11) return x[r] * s.JabJI10 + y[r] * s.JabJI11;
    else return x[r] * s.JIr0 + y[r] * s.JIr1;
  } else if constexpr (K == TOP_TRI) return s.Jab00;
  else if constexpr (K == TOP_TRI + 1) return s.Jab01;
  else if constexpr (K == TOP_TRI + 2) return s.Jabr0;
  else if constexpr (K == TOP_TRI + 3) return s.Jab11;
  else if constexpr (K == TOP_TRI + 4) return s.Jabr1;
  else if constexpr (K == TOP_TRI + 5) return s.rr;
  else return 0.f;
}

// (r, c) of the symmetric 13x13 block from the packed float layout; NH partial blocks (one per warp of the pair) are added.  The
// (a, b, r) entries follow row 9 exactly as rows 10..12 of a full upper-triangular packing would, so one formula indexes every entry.
static_assert(top_off(10) == TOP_TRI && top_off(11) == TOP_TRI + 3 && top_off(12) == TOP_TRI + 5, "bottom block = rows 10..12 of the packing");
template <int NH>
__device__ __forceinline__ float pair_entry(const float (*S)[96], int r, int c) {
  const int a = min(r, c), idx = top_off(a) + max(r, c) - a;
  if constexpr (NH == 2) return S[0][idx] + S[1][idx];
  else return S[0][idx];
}

// geometric Jacobians of the centre pixel (Residuals.cpp:L113-156): x = d(Ku)/d[C4|xi6], y = d(Kv)/d[C4|xi6], dd = d(Ku,Kv)/d(idepth)
__device__ __forceinline__ void geo_jac(const float* pc, float Kl0, float Kl1, float cu, float cv, float drescale, float new_idepth, float fx,
                                        float fy, float fxi, float fyi, float (&x)[10], float (&y)[10], float& ddx, float& ddy) {
  const float dCx2 = drescale * (pc[18] * cu - pc[12]);
  const float dCx3 = fx * drescale * (pc[19] * cu - pc[13]) * fyi;
  const float dCy2 = fy * drescale * (pc[18] * cv - pc[15]) * fxi;
  const float dCy3 = drescale * (pc[19] * cv - pc[16]);
  x[0] = (Kl0 * dCx2 + cu) * 50.0f; x[1] = (Kl1 * dCx3) * 50.0f; x[2] = (dCx2 + 1.f) * 50.0f; x[3] = dCx3 * 50.0f;
  y[0] = (Kl0 * dCy2) * 50.0f; y[1] = (Kl1 * dCy3 + cv) * 50.0f; y[2] = dCy2 * 50.0f; y[3] = (dCy3 + 1.f) * 50.0f;
  x[4] = new_idepth * fx; x[5] = 0.f; x[6] = -new_idepth * cu * fx; x[7] = -cu * cv * fx; x[8] = (1.f + cu * cu) * fx; x[9] = -cv * fx;
  y[4] = 0.f; y[5] = new_idepth * fy; y[6] = -new_idepth * cv * fy; y[7] = -(1.f + cv * cv) * fy; y[8] = cu * cv * fy; y[9] = cu * fy;
  ddx = drescale * (pc[21] - pc[23] * cu) * fx;  // Jpdd (SCALE_IDEPTH = 1)
  ddy = drescale * (pc[22] - pc[23] * cv) * fy;
}

constexpr int OPS = 57;            // operand record of one residual for the lane-split entry computation (54 used; odd stride: conflict-free)
template <int P, int LPR>
struct FusedSmem {
  static constexpr int NH = (LPR == 4) ? 2 : 1;   // warps per (host, target) pair: each leaves its own partial pair block
  double AhD[MAXF][64];        // adHost(h, t) fp64, row-major, slot = target frame
  double dT[MAXF][8];          // diag adTarget(h, t)
  double G[MAXF][8][16];       // adHost * [P | Q | p]: row i = columns 0..7 P, 8..11 Q, 12 p (16-byte aligned rows)
  float adH[MAXF][64];         // fp32 copies used for the Schur vector (the reference's adHostF / adTargetF); LPR = 1 only
  float adT[MAXF][8];
  float pair[MAXF][NH][96];    // the chunk's pair blocks (91 used), slot = target frame
  float rec[MAXF][16][P];      // per target: adHost*JpJdF [8], Hdd, bd, Hcd[4], active, pad   (lane = point: conflict-free)
  float Wv[P][8 * MAXF + 8];   // Schur vectors
  float hdi[P];
  float prior[P];              // priorF of the chunk's points (staged with the adjoints: phase B has no load round trip of its own)
  float id[P], idz[P];
  float misc[16][8];           // per warp: energy, n_in, n_oob, n_outlier, step^2, |idepth_backup|, count
  double red[16][32];          // phase E: per-warp partials of up to two 4x4 tiles
};

// operand indices of entry k of the pair block: entry = ops[a] * ops[b] + ops[c] * ops[d]   (LPR = 4 path; same arithmetic as top_entry<K>)
// ops = x[0..9] | y[10..19] | al[20..29] | be[30..39] | JabJI00 JabJI01 JabJI10 JabJI11 JIr0 JIr1 [40..45] | Jab00 Jab01 Jabr0 Jab11 Jabr1 rr [46..51] | 0 [52] | 1 [53]
struct alignas(16) EntryTab { unsigned char v[96][4]; };
constexpr EntryTab make_entry_tab() {
  EntryTab t{};
  for (int k = 0; k < 96; k++) {
    if (k < TOP_TRI) {
      const int r = top_row(k), c = top_col(k);
      if (c < 10) { t.v[k][0] = 20 + r; t.v[k][1] = c; t.v[k][2] = 30 + r; t.v[k][3] = 10 + c; }
      else { t.v[k][0] = r; t.v[k][1] = 40 + 2 * (c - 10); t.v[k][2] = 10 + r; t.v[k][3] = 41 + 2 * (c - 10); }
    } else if (k < TOP_USED) { t.v[k][0] = 46 + (k - TOP_TRI); t.v[k][1] = 53; t.v[k][2] = 52; t.v[k][3] = 52; }
    else { t.v[k][0] = 52; t.v[k][1] = 52; t.v[k][2] = 52; t.v[k][3] = 52; }
  }
  return t;
}
static __device__ __constant__ EntryTab c_entry_tab = make_entry_tab();

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// all CTAs of the (cooperative) grid; monotonic arrival counter, target = arrivals expected so far.  Bounded: a lost CTA can delay the
// launch by ~0.1 s but never hang the GPU (the result then carries the error flag).  Visibility of the other CTAs' part / wg / hdig stores
// rests on the release add and the acquire poll of thread 0, extended to the whole CTA by the block barriers on both sides (release and
// acquire are cumulative over what the barrier ordered): no sequentially consistent fence is needed.
__device__ __forceinline__ bool grid_barrier(unsigned* bar, unsigned target) {
  __shared__ int ok_s;
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
    int ok = 1;
    const long long t0 = clock64();
    while ((int)(ld_acquire_u32(bar) - target) < 0) {
      if (clock64() - t0 > 200000000ll) { ok = 0; break; }
    }
    ok_s = ok;
  }
  __syncthreads();
  return ok_s != 0;
}

// phase clock of the measurement-only instantiation (CLK = true, dmv_ba_bench_phases): thread 0 of the CTA writes %globaltimer to slot k of
// its row of clk once `dep`, a value the timed phase produced, is available (the predicate on it orders the read after the producing
// load).  Compiles to nothing in the product kernels.
constexpr int NCLK = FUSED_NCLK;  // entry, chunk decoded, first loads, taps, end A, end C, barrier released, end D, end E
template <bool CLK>
__device__ __forceinline__ void clk_stamp(unsigned long long* clk, int k, unsigned dep = 0u) {
  if constexpr (CLK) {
    if (threadIdx.x == 0) {
      unsigned long long t = 0;
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0x7fbadbad;\n\t@p mov.u64 %0, %%globaltimer;\n\t}" : "+l"(t) : "r"(dep) : "memory");
      clk[(size_t)blockIdx.x * NCLK + k] = t;
    }
  }
}

// ---- exchange of result entries between ranks (sharded BA, SURVEY.md §8e): "LL" packets over NVLink peer memory.  Every result
// entry has one producing warp (the same on every rank): it pushes the entry as a 16-byte packet {lo, seq, hi, seq} into slot
// [parity][my rank][entry] of every peer's inbox (st.volatile.v4: each 8-byte half carries its own flag, no fence, no separate flag
// round trip), later polls its OWN inbox until the peers' packets of that entry carry this exchange's sequence number and adds them in
// RANK ORDER (bit-identical sums on every rank).  Double-buffered by parity; the poll is bounded (a dead peer yields an error flag).
__device__ __forceinline__ void xchg_push(const BAXchg& X, int idx, double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  const uint4 pk = make_uint4((unsigned)(u & 0xffffffffull), X.seq, (unsigned)(u >> 32), X.seq);
  const size_t off = (size_t)(((X.seq & 1u) * XCHG_MAXR + X.rank)) * X.pitch + idx;
#pragma unroll 1
  for (int k = 1; k < X.nranks; k++) {
    const int r = (X.rank + k) % X.nranks;  // start with the neighbour: spreads the NVSwitch ports
    uint4* dst = X.inbox[r] + off;
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(pk.x), "r"(pk.y), "r"(pk.z), "r"(pk.w) : "memory");
  }
}
// Both pull variants are WARP-COLLECTIVE with warp-uniform spin loops (votes decide when to leave): lanes of one warp never wait on
// different conditions, so the warp is converged at the __syncthreads() that follow (an aligned barrier executed by a diverged warp counts
// the warp twice: premature release or "warp illegal instruction").
constexpr long long XCHG_SPIN_LIMIT = 400000000ll;  // ~0.2 s of SM clocks: peer lost

// lane-per-entry: every lane with active == true owns entry idx and polls the nranks - 1 packets of it
__device__ __forceinline__ double xchg_pull_sum_lanes(const BAXchg& X, int idx, double mine, bool active, bool& ok) {
  const uint4* base = X.inbox[X.rank] + (size_t)((X.seq & 1u) * XCHG_MAXR) * X.pitch + idx;
  uint4 pk[XCHG_MAXR];
  unsigned pending = active ? (((1u << X.nranks) - 1u) & ~(1u << X.rank)) : 0u;
  const long long t0 = clock64();
  while (__any_sync(0xffffffffu, pending != 0u)) {
#pragma unroll
    for (int r = 0; r < XCHG_MAXR; r++)
      if ((pending >> r) & 1u) {
        const uint4* src = base + (size_t)r * X.pitch;
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(pk[r].x), "=r"(pk[r].y), "=r"(pk[r].z), "=r"(pk[r].w) : "l"(src) : "memory");
      }
#pragma unroll
    for (int r = 0; r < XCHG_MAXR; r++)
      if (((pending >> r) & 1u) && pk[r].y == X.seq && pk[r].w == X.seq) pending &= ~(1u << r);
    if (__any_sync(0xffffffffu, clock64() - t0 > XCHG_SPIN_LIMIT)) break;
  }
  if (pending) { ok = false; return mine; }
  double s = 0.0;
#pragma unroll
  for (int r = 0; r < XCHG_MAXR; r++) {
    if (r >= X.nranks) break;
    s += (r == X.rank) ? mine : __longlong_as_double((long long)(((unsigned long long)pk[r].z << 32) | pk[r].x));
  }
  return active ? s : mine;
}

// 16-lane group per entry (phase D): lane gl of the group polls the packet of rank gl, all ranks in flight at once; `mine` is the value of
// lane gl == 0.  Returns the rank-ordered sum in every lane of the group.
__device__ __forceinline__ double xchg_pull_sum_group(const BAXchg& X, int idx, double mine, bool active, bool& ok) {
  const int lane = threadIdx.x & 31, gl = lane & 15;
  const bool poll = active && gl < X.nranks && gl != X.rank;
  const uint4* src = X.inbox[X.rank] + (size_t)((X.seq & 1u) * XCHG_MAXR + (poll ? gl : 0)) * X.pitch + idx;
  uint4 pk = make_uint4(0u, 0u, 0u, 0u);
  bool pending = poll;
  const long long t0 = clock64();
  while (__any_sync(0xffffffffu, pending)) {
    if (pending) {
      asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(pk.x), "=r"(pk.y), "=r"(pk.z), "=r"(pk.w) : "l"(src) : "memory");
      pending = !(pk.y == X.seq && pk.w == X.seq);
    }
    if (__any_sync(0xffffffffu, clock64() - t0 > XCHG_SPIN_LIMIT)) break;
  }
  if (__any_sync(0xffffffffu, pending)) ok = false;
  const double own = __shfl_sync(0xffffffffu, mine, lane & 16);
  const double v = (gl == X.rank) ? own : (poll ? __longlong_as_double((long long)(((unsigned long long)pk.z << 32) | pk.x)) : 0.0);
  double s = 0.0;
  for (int r = 0; r < X.nranks; r++) s += __shfl_sync(0xffffffffu, v, (lane & 16) | r);  // rank order: bit-identical on every rank
  return s;
}

// MARG = true is the marginalisation launch (dmv_ba_marginalize_points): only the points flagged in W.marg_mask take part, their
// residuals are re-linearised from scratch (PointFrameResidual::resetOOB; FullSystem.cpp:L826-838), EFResidual::fixLinearizationF
// (EnergyFunctionalStructs.cpp:L88-114) turns resF into res_toZeroF, and the accumulation is AccumulatedTopHessian::addPoint<2> +
// AccumulatedSCHessian::addPoint(p, shiftPriorToZero = false) with priorF * idepthFixPriorMargFac (EnergyFunctional.cpp:L678-742).
// phases A-C for one chunk of one window (W / it may live in kernel-parameter space or in global memory)
template <int P, int LPR, bool MARG, bool CLK = false>
__device__ __forceinline__ void fused_chunk(const BAWinDev& W, const BAIter& it, FusedSmem<P, LPR>& S, const int chunk, unsigned long long* clk = nullptr) {
  constexpr int LOGP = (P == 32) ? 5 : 4;
  constexpr int NH = FusedSmem<P, LPR>::NH;
  const int nf = W.nf, N = W.N, mp = W.mp;
  const int tid = threadIdx.x, nthreads = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
  const BAAdj* __restrict__ A = W.adj;
  int h = 0;  // host frame of this chunk: branch-free so that the constant-bank loads are independent
#pragma unroll
  for (int k = 1; k < MAXF; k++) h += (chunk >= W.chunk_beg[k]) ? 1 : 0;
  h = min(h, nf - 1);
  const int ch_start = W.host_start[h] + (chunk - W.chunk_beg[h]) * P;
  const int ch_count = min(P, W.host_start[h + 1] - ch_start);
  clk_stamp<CLK>(clk, 1, (unsigned)ch_count);

  // ---- stage the host's adjoint blocks (fp64 for phase C, fp32 for the Schur vectors); waited for at the first block barrier,
  // except the fp32 block of a warp's own pair(s), which the warp fetches itself below
  for (int i = tid; i < nf * 32; i += nthreads) cp_async16(&S.AhD[i >> 5][(i & 31) * 2], &A->adHost[h * nf + (i >> 5)][(i & 31) * 2]);
  for (int i = tid; i < nf * 4; i += nthreads) cp_async16(&S.dT[i >> 2][(i & 3) * 2], &A->adTdiag[h * nf + (i >> 2)][(i & 3) * 2]);
  if (tid < ch_count) cp_async4(&S.prior[tid], W.priorF + ch_start + tid);
  asm volatile("cp.async.commit_group;" ::: "memory");

  float e_sum = 0.f, rs_step2 = 0.f, rs_nid = 0.f, rs_cnt = 0.f;
  int n_in = 0, n_oob = 0, n_outl = 0;
  if constexpr (LPR == 1) {
  // ---------------------------------------------------------------- phase A (LPR = 1): one thread = one point-residual
  const int r = tid >> LOGP, pl = tid & (P - 1);  // r-th target frame other than h
  const int t = r + (r >= h ? 1 : 0);
  const bool slot_ok = r < nf - 1;
  {  // every warp runs the phase (no thread-dependent branch around the shuffles: ptxas then emits plain SHFL, not WARPSYNC-wrapped ones)
    const int tc = slot_ok ? t : (h == 0 ? 1 : 0);  // lanes without a pair shadow a valid one (loads stay in bounds, nothing is written)
    if (slot_ok) {  // the pair's fp32 adjoints: fetched by the lanes that use them (no block barrier before phase A's tail)
      if (pl < 16) *reinterpret_cast<float4*>(&S.adH[t][pl * 4]) = __ldg(reinterpret_cast<const float4*>(&A->adHostF[h * nf + t][pl * 4]));
      if (pl < 2) *reinterpret_cast<float4*>(&S.adT[t][pl * 4]) = __ldg(reinterpret_cast<const float4*>(&A->adTdiagF[h * nf + t][pl * 4]));
    }
    const bool valid = slot_ok && pl < ch_count;
    const int p = ch_start + min(pl, ch_count - 1);
    const int slot = tc * mp + p;
    const float* pc = it.precalc[h * nf + tc];
    const float fx = it.calib[0], fy = it.calib[1], cx = it.calib[2], cy = it.calib[3];
    const float fxi = it.calib[4], fyi = it.calib[5];
    const float TH = fmaxf(it.TH[h], it.TH[tc]);
    const float wM3 = (float)(W.w - 3), hM3 = (float)(W.h - 3);
    const float4* __restrict__ img = W.img[tc];
    const int iw = W.w;
    const float huber = W.huberTH, oth = W.outlierTHSum;

    // ---- direct loads (all independent: one memory round trip)
    int st = valid ? (int)__ldg(W.st_in + slot) : RES_NONE;
    float en_old = __ldg(W.en_in + slot);
    bool masked = true;
    if constexpr (MARG) {  // resetOOB: every existing residual of a flagged point starts as IN with zero energy; other points sit out
      masked = valid && __ldg(W.marg_mask + p) != 0;
      st = (masked && st != RES_NONE) ? RES_IN : RES_NONE;
      en_old = 0.f;
    }
    const float2 uv = __ldg(W.uv + p);
    float col[8], wgt[8];
    {
      const float4 c0 = __ldg(reinterpret_cast<const float4*>(W.color + (size_t)p * 8)), c1 = __ldg(reinterpret_cast<const float4*>(W.color + (size_t)p * 8) + 1);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(W.weights + (size_t)p * 8)), w1 = __ldg(reinterpret_cast<const float4*>(W.weights + (size_t)p * 8) + 1);
      col[0] = c0.x; col[1] = c0.y; col[2] = c0.z; col[3] = c0.w; col[4] = c1.x; col[5] = c1.y; col[6] = c1.z; col[7] = c1.w;
      wgt[0] = w0.x; wgt[1] = w0.y; wgt[2] = w0.z; wgt[3] = w0.w; wgt[4] = w1.x; wgt[5] = w1.y; wgt[6] = w1.z; wgt[7] = w1.w;
    }
    float idepth, idz;
    if (it.have_x) {
      // fused EnergyFunctional::resubstituteFPt (EnergyFunctional.cpp:L295-321) + point step (FullSystemOptimize.cpp:L264-272): every
      // thread of the point recomputes the same step from the committed linearisation (loads hit L1/L2), the first target's publishes
      const float4 po0 = __ldg(reinterpret_cast<const float4*>(W.c_pout + (size_t)p * 8));
      const float4 po1 = __ldg(reinterpret_cast<const float4*>(W.c_pout + (size_t)p * 8) + 1);
      const float idb = __ldg(W.idepth_backup + p);
      float b = po1.w - (it.xc[0] * po0.z + it.xc[1] * po0.w + it.xc[2] * po1.x + it.xc[3] * po1.y);
      int ngood = 0;
#pragma unroll
      for (int t4 = 0; t4 < MAXF; t4 += 4) {  // the loads of 4 targets are issued before any is used (2 memory round trips, not one per target)
        int stc[4];
        float4 a0[4], a1[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int cs = min(t4 + u, nf - 1) * mp + p;
          stc[u] = __ldg(W.c_st + cs);
          a0[u] = __ldg(reinterpret_cast<const float4*>(W.c_jpjd + (size_t)cs * 8));
          a1[u] = __ldg(reinterpret_cast<const float4*>(W.c_jpjd + (size_t)cs * 8) + 1);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int tt = t4 + u;
          const bool good = tt < nf && tt != h && stc[u] == RES_IN;
          const float* xa = it.xAd[h * nf + min(tt, nf - 1)];
          const float dot = xa[0] * a0[u].x + xa[1] * a0[u].y + xa[2] * a0[u].z + xa[3] * a0[u].w + xa[4] * a1[u].x + xa[5] * a1[u].y + xa[6] * a1[u].z + xa[7] * a1[u].w;
          b -= good ? dot : 0.f;
          ngood += good;
        }
      }
      const float step = ngood > 0 ? -b * po1.z : 0.f;
      idepth = idb + step;
      idz = idepth;  // DM-VIO: idepth_zero follows (setIdepthZero in doStepFromBackup); the host aliases the pointers
      if (r == 0 && valid) {
        W.step[p] = step;
        W.idepth_out[p] = idepth;
        rs_step2 = step * step; rs_nid = fabsf(idb); rs_cnt = 1.f;
      }
    } else {
      idepth = __ldg(W.idepth + p);
      idz = __ldg(W.idepth_zero + p);
    }
    if (r == 0 && valid) { S.id[pl] = idepth; S.idz[pl] = idz; }
    clk_stamp<CLK>(clk, 2, __float_as_uint(idepth) ^ __float_as_uint(uv.x) ^ (unsigned)st);
    bool live = (st != RES_NONE) && (st != RES_OOB);

    // ---- centre pixel at the FEJ point (ResidualProjections.h:L62-87, Residuals.cpp:L108-157)
    const float Kl0 = (uv.x - cx) * fxi, Kl1 = (uv.y - cy) * fyi;
    const float q2 = pc[18] * Kl0 + pc[19] * Kl1 + pc[20] + pc[23] * idz;
    const float drescale = 1.0f / q2;
    const float new_idepth = idz * drescale;
    const float cu = (pc[12] * Kl0 + pc[13] * Kl1 + pc[14] + pc[21] * idz) * drescale;
    const float cv = (pc[15] * Kl0 + pc[16] * Kl1 + pc[17] + pc[22] * idz) * drescale;
    const float cKu = cu * fx + cx, cKv = cv * fy + cy;
    live = live && (drescale > 0.f) && cKu > 1.1f && cKv > 1.1f && cKu < wM3 && cKv < hM3;

    // ---- the 8 pattern pixels at the current state (ResidualProjections.h:L47-57): all must project inside the image
    float Ku[8], Kv[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float pu = uv.x + (float)c_pattern[j][0], pv = uv.y + (float)c_pattern[j][1];
      const float r2 = pc[6] * pu + pc[7] * pv + pc[8] + pc[11] * idepth;
      Ku[j] = (pc[0] * pu + pc[1] * pv + pc[2] + pc[9] * idepth) / r2;
      Kv[j] = (pc[3] * pu + pc[4] * pv + pc[5] + pc[10] * idepth) / r2;
      live = live && Ku[j] > 1.1f && Kv[j] > 1.1f && Ku[j] < wM3 && Kv[j] < hM3;
    }
    float x[10], y[10], ddx = 0.f, ddy = 0.f, jpx = 0.f, jpy = 0.f, dp6 = 0.f, dp7 = 0.f;
    if constexpr (MARG) {  // fixLinearizationF needs the geometric Jacobians per pixel: res_toZeroF = resF - J * delta
      if (live) {
        geo_jac(pc, Kl0, Kl1, cu, cv, drescale, new_idepth, fx, fy, fxi, fyi, x, y, ddx, ddy);
        const float* dp = W.marg->adHTdelta[h * nf + tc];
        const float* cD = W.marg->cDelta;
        const float dlt = idepth - idz;  // EFPoint::deltaF
        jpx = (x[4] * dp[0] + x[5] * dp[1] + x[6] * dp[2] + x[7] * dp[3] + x[8] * dp[4] + x[9] * dp[5]) +
              (x[0] * cD[0] + x[1] * cD[1] + x[2] * cD[2] + x[3] * cD[3]) + ddx * dlt;
        jpy = (y[4] * dp[0] + y[5] * dp[1] + y[6] * dp[2] + y[7] * dp[3] + y[8] * dp[4] + y[9] * dp[5]) +
              (y[0] * cD[0] + y[1] * cD[1] + y[2] * cD[2] + y[3] * cD[3]) + ddy * dlt;
        dp6 = dp[6]; dp7 = dp[7];
      }
    }

    // ---- getInterpolatedElement33 (util/globalFuncs.h:L103-118), photometric residual, gradient weight, Huber (Residuals.cpp:L194-258)
    PixSums s = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float energy = 0.f, wJI2 = 0.f, rtz[8];
    if (live) {
      const bool zA = W.zeroA != 0, zB = W.zeroB != 0;
#pragma unroll
      for (int half = 0; half < 2; half++) {  // 16 float4 taps in flight per thread, twice
      float4 tap[4][4];
#pragma unroll
      for (int jj = 0; jj < 4; jj++) {
        const int j = half * 4 + jj;
        const int ix = (int)Ku[j], iy = (int)Kv[j];
        const float4* bp = img + (size_t)iy * iw + ix;
        tap[jj][0] = __ldg(bp); tap[jj][1] = __ldg(bp + 1); tap[jj][2] = __ldg(bp + iw); tap[jj][3] = __ldg(bp + iw + 1);
      }
#pragma unroll
      for (int jj = 0; jj < 4; jj++) {
        const int j = half * 4 + jj;
        const int ix = (int)Ku[j], iy = (int)Kv[j];
        const float dx = Ku[j] - ix, dy = Kv[j] - iy, dxdy = dx * dy;
        const float w11 = dxdy, w10 = dy - dxdy, w01 = dx - dxdy, w00 = 1 - dx - dy + dxdy;
        const float h0 = w11 * tap[jj][3].x + w10 * tap[jj][2].x + w01 * tap[jj][1].x + w00 * tap[jj][0].x;
        const float h1 = w11 * tap[jj][3].y + w10 * tap[jj][2].y + w01 * tap[jj][1].y + w00 * tap[jj][0].y;
        const float h2 = w11 * tap[jj][3].z + w10 * tap[jj][2].z + w01 * tap[jj][1].z + w00 * tap[jj][0].z;
        live = live && isfinite(h0);
        const float residual = h0 - (pc[24] * col[j] + pc[25]);
        const float drdA = col[j] - pc[26];
        float w = sqrtf(oth / (oth + (h1 * h1 + h2 * h2)));
        w = 0.5f * (w + wgt[j]);
        const float ar = fabsf(residual);
        float hw = ar < huber ? 1.f : huber / ar;
        energy += w * w * hw * residual * residual * (2.f - hw);
        if (hw < 1.f) hw = sqrtf(hw);
        hw = hw * w;
        const float gx = h1 * hw, gy = h2 * hw;
        const float resF = residual * hw;
        const float ja = drdA * hw, jb = hw;
        const float jaF = zA ? 0.f : ja, jbF = zB ? 0.f : jb;
        float ra = resF;  // what the right-hand sides are built from: resF, or res_toZeroF when marginalising
        if constexpr (MARG) { ra = (((resF - gx * jpx) - gy * jpy) - jaF * dp6) - jbF * dp7; rtz[j] = ra; }
        s.JI00 += gx * gx; s.JI11 += gy * gy; s.JI10 += gx * gy;
        s.JabJI00 += ja * gx; s.JabJI01 += ja * gy; s.JabJI10 += jb * gx; s.JabJI11 += jb * gy;
        s.Jab00 += ja * ja; s.Jab01 += ja * jb; s.Jab11 += jb * jb;
        s.JIr0 += ra * gx; s.JIr1 += ra * gy; s.Jabr0 += ra * jaF; s.Jabr1 += ra * jbF; s.rr += ra * ra;
        // the reference sums hw*hw*(hitColor[1]^2+hitColor[2]^2) with hitColor already multiplied by hw (Residuals.cpp:L217-244)
        wJI2 += hw * hw * (gx * gx + gy * gy);
      }
      }
    }
    clk_stamp<CLK>(clk, 3, __float_as_uint(s.JI00));

    // ---- classification (Residuals.cpp:L260-273) and per-residual outputs
    int newState;
    float newEnergy;
    if (st == RES_NONE) { newState = RES_NONE; newEnergy = 0.f; }
    else if (!live) { newState = RES_OOB; newEnergy = en_old; }  // OOB exits return the old state_energy
    else if (energy > TH || wJI2 < 2.f) { newState = RES_OUTLIER; newEnergy = TH; }
    else { newState = RES_IN; newEnergy = energy; }
    const bool in = (newState == RES_IN);
    if (st != RES_NONE) {
      e_sum = newEnergy;
      n_in = in; n_oob = (newState == RES_OOB); n_outl = (newState == RES_OUTLIER);
    }
    if constexpr (MARG) {
      if (masked) {
        float4* o = reinterpret_cast<float4*>(W.marg_rtz + (size_t)slot * 8);
        o[0] = in ? make_float4(rtz[0], rtz[1], rtz[2], rtz[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
        o[1] = in ? make_float4(rtz[4], rtz[5], rtz[6], rtz[7]) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    if (valid && masked) {
      W.st_new[slot] = (uint8_t)newState;
      W.en_new[slot] = newEnergy;
      const float ewo = (st == RES_NONE || !live) ? -1.f : energy;
      W.en_wo[slot] = ewo;
      if (tc == nf - 1 && W.en_wo_newest_host) W.en_wo_newest_host[p] = ewo;  // zero-copy: the host's percentile needs no D2H call
      const size_t plane = (size_t)MAXF * mp;
      W.cpt[slot] = cKu; W.cpt[plane + slot] = cKv; W.cpt[2 * plane + slot] = new_idepth;
    }

    // ---- EFResidual::takeDataF (EnergyFunctionalStructs.cpp:L39-49), the per-point terms of addPoint (AccumulatedTopHessian.cpp:L131-135)
    // and the residual's part of the point's Schur vector
    float jp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, Hdd = 0.f, bd = 0.f, Hcd0 = 0.f, Hcd1 = 0.f, Hcd2 = 0.f, Hcd3 = 0.f;
    if (in) {
      if constexpr (!MARG) geo_jac(pc, Kl0, Kl1, cu, cv, drescale, new_idepth, fx, fy, fxi, fyi, x, y, ddx, ddy);
      const float J0 = s.JI00 * ddx + s.JI10 * ddy, J1 = s.JI10 * ddx + s.JI11 * ddy;  // JIdx2 * Jpdd
#pragma unroll
      for (int k = 0; k < 6; k++) jp[k] = x[4 + k] * J0 + y[4 + k] * J1;
      jp[6] = s.JabJI00 * ddx + s.JabJI01 * ddy; jp[7] = s.JabJI10 * ddx + s.JabJI11 * ddy;
      Hdd = J0 * ddx + J1 * ddy;
      bd = s.JIr0 * ddx + s.JIr1 * ddy;
      Hcd0 = x[0] * J0 + y[0] * J1; Hcd1 = x[1] * J0 + y[1] * J1; Hcd2 = x[2] * J0 + y[2] * J1; Hcd3 = x[3] * J0 + y[3] * J1;
      if (valid) {
        float4* gj = reinterpret_cast<float4*>(W.jpjd + (size_t)slot * 8);
        gj[0] = make_float4(jp[0], jp[1], jp[2], jp[3]);
        gj[1] = make_float4(jp[4], jp[5], jp[6], jp[7]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 10; k++) { x[k] = 0.f; y[k] = 0.f; }
      s = PixSums{0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    }
    __syncwarp();  // the pair's adjoints staged by this warp above
    if (slot_ok) {
      // host block: adHost(h,t) * JpJdF (summed over targets in phase B); target block: adTarget(h,t) is diagonal
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const float4 a0 = *reinterpret_cast<const float4*>(&S.adH[t][k * 8]), a1 = *reinterpret_cast<const float4*>(&S.adH[t][k * 8 + 4]);
        S.rec[t][k][pl] = a0.x * jp[0] + a0.y * jp[1] + a0.z * jp[2] + a0.w * jp[3] + a1.x * jp[4] + a1.y * jp[5] + a1.z * jp[6] + a1.w * jp[7];
        S.Wv[pl][4 + 8 * t + k] = S.adT[t][k] * jp[k];
      }
      S.rec[t][8][pl] = Hdd; S.rec[t][9][pl] = bd; S.rec[t][10][pl] = Hcd0; S.rec[t][11][pl] = Hcd1; S.rec[t][12][pl] = Hcd2; S.rec[t][13][pl] = Hcd3;
      S.rec[t][14][pl] = in ? 1.f : 0.f;
    }

    // ---- the pair's 13x13 block: 96 (91 used) entries per residual, summed over the pair's P lanes with a transposing butterfly:
    // every step exchanges HALF of the remaining values, so the whole reduction costs 96 shuffles instead of 96 * log2(P)
    float al[10], be[10];
#pragma unroll
    for (int k = 0; k < 10; k++) { al[k] = s.JI00 * x[k] + s.JI10 * y[k]; be[k] = s.JI10 * x[k] + s.JI11 * y[k]; }
    float v[48];
    {
      const bool up = (lane & (P / 2)) != 0;
      static_for<0, 48>([&](auto kc) {
        constexpr int k = decltype(kc)::value;
        const float a = top_entry<k>(x, y, al, be, s), b = top_entry<k + 48>(x, y, al, be, s);
        v[k] = (up ? b : a) + __shfl_xor_sync(0xffffffffu, up ? a : b, P / 2);
      });
    }
    static_for<0, LOGP - 1>([&](auto sc) {  // steps 2..log2(P): 24, 12, 6 (, 3) exchanges
      constexpr int st2 = decltype(sc)::value, hstep = 24 >> st2, m = (P / 4) >> st2;
      const bool up = (lane & m) != 0;
#pragma unroll
      for (int k = 0; k < hstep; k++) v[k] = (up ? v[k + hstep] : v[k]) + __shfl_xor_sync(0xffffffffu, up ? v[k] : v[k + hstep], m);
    });
    if (slot_ok) {  // lane L of the pair's group now holds entries [(96/P) L, (96/P)(L+1))
      constexpr int PER = 96 / P;
#pragma unroll
      for (int k = 0; k < PER; k++) S.pair[t][0][PER * pl + k] = v[k];
    }
  }
  } else {
  // ---------------------------------------------------------------- phase A (LPR = 4): 4 lanes per point-residual, 2 pattern pixels each.
  // The latency-oriented variant for ONE window: the per-residual chain is ~2.5x shorter and the CTA has 4x the warps, at the price of
  // redundant per-residual scalar work in the 4 lanes.  A (host, target) pair = 16 points x 4 lanes = 2 warps.
  static_assert(LPR == 1 || P == 16, "LPR = 4 is written for chunks of 16 points");
  const int r = tid >> 6;                                 // r-th target frame other than h (warp-uniform)
  const int pl = (tid & 63) >> 2, q = tid & 3;            // point of the chunk, lane of the residual
  const int half = (tid >> 5) & 1;                        // which of the pair's two warps
  const bool pair_ok = r < nf - 1;                        // warps beyond the window's pairs shadow a valid pair and write nothing
  const int t = pair_ok ? r + (r >= h ? 1 : 0) : (h == 0 ? 1 : 0);
  {
    const bool valid = pair_ok && pl < ch_count;
    const int p = ch_start + min(pl, ch_count - 1);
    const int slot = t * mp + p;
    const float* pc = it.precalc[h * nf + t];
    const float fx = it.calib[0], fy = it.calib[1], cx = it.calib[2], cy = it.calib[3];
    const float fxi = it.calib[4], fyi = it.calib[5];
    const float TH = fmaxf(it.TH[h], it.TH[t]);
    const float wM3 = (float)(W.w - 3), hM3 = (float)(W.h - 3);
    const float4* __restrict__ img = W.img[t];
    const int iw = W.w;
    const float huber = W.huberTH, oth = W.outlierTHSum;

    // ---- direct loads (all independent: one memory round trip); rows 2q, 2q+1 of the pair's fp32 adjoint for the Schur vector
    int st = valid ? (int)__ldg(W.st_in + slot) : RES_NONE;
    float en_old = __ldg(W.en_in + slot);
    bool masked = true;
    if constexpr (MARG) {
      masked = valid && __ldg(W.marg_mask + p) != 0;
      st = (masked && st != RES_NONE) ? RES_IN : RES_NONE;
      en_old = 0.f;
    }
    const float2 uv = __ldg(W.uv + p);
    const float2 col = __ldg(reinterpret_cast<const float2*>(W.color + (size_t)p * 8) + q);
    const float2 wgt = __ldg(reinterpret_cast<const float2*>(W.weights + (size_t)p * 8) + q);
    float4 ah[4];
#pragma unroll
    for (int u = 0; u < 4; u++) ah[u] = __ldg(reinterpret_cast<const float4*>(&A->adHostF[h * nf + t][q * 16]) + u);
    const float2 at2 = __ldg(reinterpret_cast<const float2*>(&A->adTdiagF[h * nf + t][q * 2]));
    float idepth, idz;
    if (it.have_x) {  // fused resubstituteFPt + point step: lane q of the residual takes targets 2q, 2q+1, two butterfly steps add the 4 lanes'
      // partial sums (commutative pairs: the sum, hence the step, is bit-identical in the 4 lanes and in every pair-warp of the point; it
      // differs in the last bits from the sequential sum of the LPR = 1 path and of resub_point)
      static_assert(MAXF == 8, "4 lanes x 2 targets cover the MAXF frame slots");
      const float4 po0 = __ldg(reinterpret_cast<const float4*>(W.c_pout + (size_t)p * 8));
      const float4 po1 = __ldg(reinterpret_cast<const float4*>(W.c_pout + (size_t)p * 8) + 1);
      const float idb = __ldg(W.idepth_backup + p);
      int stc[2];
      float4 a0[2], a1[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int cs = min(2 * q + u, nf - 1) * mp + p;
        stc[u] = __ldg(W.c_st + cs);
        a0[u] = __ldg(reinterpret_cast<const float4*>(W.c_jpjd + (size_t)cs * 8));
        a1[u] = __ldg(reinterpret_cast<const float4*>(W.c_jpjd + (size_t)cs * 8) + 1);
      }
      float bt = 0.f;
      int ngood = 0;
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int tt = 2 * q + u;
        const bool good = tt < nf && tt != h && stc[u] == RES_IN;
        const float* xa = it.xAd[h * nf + min(tt, nf - 1)];
        const float dot = xa[0] * a0[u].x + xa[1] * a0[u].y + xa[2] * a0[u].z + xa[3] * a0[u].w + xa[4] * a1[u].x + xa[5] * a1[u].y + xa[6] * a1[u].z + xa[7] * a1[u].w;
        bt += good ? dot : 0.f;
        ngood += good;
      }
      bt += __shfl_xor_sync(0xffffffffu, bt, 1);
      bt += __shfl_xor_sync(0xffffffffu, bt, 2);
      ngood += __shfl_xor_sync(0xffffffffu, ngood, 1);
      ngood += __shfl_xor_sync(0xffffffffu, ngood, 2);
      const float b = (po1.w - (it.xc[0] * po0.z + it.xc[1] * po0.w + it.xc[2] * po1.x + it.xc[3] * po1.y)) - bt;
      const float step = ngood > 0 ? -b * po1.z : 0.f;
      idepth = idb + step;
      idz = idepth;
      if (r == 0 && q == 0 && valid) {
        W.step[p] = step;
        W.idepth_out[p] = idepth;
        rs_step2 = step * step; rs_nid = fabsf(idb); rs_cnt = 1.f;
      }
    } else {
      idepth = __ldg(W.idepth + p);
      idz = __ldg(W.idepth_zero + p);
    }
    if (r == 0 && q == 0 && valid) { S.id[pl] = idepth; S.idz[pl] = idz; }
    clk_stamp<CLK>(clk, 2, __float_as_uint(idepth) ^ __float_as_uint(uv.x) ^ (unsigned)st);
    bool live = (st != RES_NONE) && (st != RES_OOB);

    // ---- centre pixel at the FEJ point (every lane)
    const float Kl0 = (uv.x - cx) * fxi, Kl1 = (uv.y - cy) * fyi;
    const float q2 = pc[18] * Kl0 + pc[19] * Kl1 + pc[20] + pc[23] * idz;
    const float drescale = 1.0f / q2;
    const float new_idepth = idz * drescale;
    const float cu = (pc[12] * Kl0 + pc[13] * Kl1 + pc[14] + pc[21] * idz) * drescale;
    const float cv = (pc[15] * Kl0 + pc[16] * Kl1 + pc[17] + pc[22] * idz) * drescale;
    const float cKu = cu * fx + cx, cKv = cv * fy + cy;
    live = live && (drescale > 0.f) && cKu > 1.1f && cKv > 1.1f && cKu < wM3 && cKv < hM3;

    // ---- this lane's two pattern pixels (2q, 2q+1) at the current state
    float Ku[2], Kv[2];
#pragma unroll
    for (int jj = 0; jj < 2; jj++) {
      const float pu = uv.x + (float)c_pattern[2 * q + jj][0], pv = uv.y + (float)c_pattern[2 * q + jj][1];
      const float r2 = pc[6] * pu + pc[7] * pv + pc[8] + pc[11] * idepth;
      Ku[jj] = (pc[0] * pu + pc[1] * pv + pc[2] + pc[9] * idepth) / r2;
      Kv[jj] = (pc[3] * pu + pc[4] * pv + pc[5] + pc[10] * idepth) / r2;
      live = live && Ku[jj] > 1.1f && Kv[jj] > 1.1f && Ku[jj] < wM3 && Kv[jj] < hM3;
    }
    {  // all 8 pixels of the residual must project inside: AND over the 4 lanes
      const unsigned bal = __ballot_sync(0xffffffffu, live);
      live = ((bal >> (lane & ~3)) & 0xfu) == 0xfu;
    }
    float x[10], y[10], ddx = 0.f, ddy = 0.f, jpx = 0.f, jpy = 0.f, dp6 = 0.f, dp7 = 0.f;
    if constexpr (MARG) {
      if (live) {
        geo_jac(pc, Kl0, Kl1, cu, cv, drescale, new_idepth, fx, fy, fxi, fyi, x, y, ddx, ddy);
        const float* dp = W.marg->adHTdelta[h * nf + t];
        const float* cD = W.marg->cDelta;
        const float dlt = idepth - idz;
        jpx = (x[4] * dp[0] + x[5] * dp[1] + x[6] * dp[2] + x[7] * dp[3] + x[8] * dp[4] + x[9] * dp[5]) +
              (x[0] * cD[0] + x[1] * cD[1] + x[2] * cD[2] + x[3] * cD[3]) + ddx * dlt;
        jpy = (y[4] * dp[0] + y[5] * dp[1] + y[6] * dp[2] + y[7] * dp[3] + y[8] * dp[4] + y[9] * dp[5]) +
              (y[0] * cD[0] + y[1] * cD[1] + y[2] * cD[2] + y[3] * cD[3]) + ddy * dlt;
        dp6 = dp[6]; dp7 = dp[7];
      }
    }

    // ---- the lane's 2 x 4 taps, residuals, partial sums
    float sv[17];  // JI00 JI10 JI11 JabJI00 JabJI01 JabJI10 JabJI11 Jab00 Jab01 Jab11 JIr0 JIr1 Jabr0 Jabr1 rr | energy wJI2
#pragma unroll
    for (int k = 0; k < 17; k++) sv[k] = 0.f;
    float rtz[2] = {0.f, 0.f};
    bool fin = true;
    if (live) {
      const bool zA = W.zeroA != 0, zB = W.zeroB != 0;
      float4 tap[2][4];
#pragma unroll
      for (int jj = 0; jj < 2; jj++) {
        const int ix = (int)Ku[jj], iy = (int)Kv[jj];
        const float4* bp = img + (size_t)iy * iw + ix;
        tap[jj][0] = __ldg(bp); tap[jj][1] = __ldg(bp + 1); tap[jj][2] = __ldg(bp + iw); tap[jj][3] = __ldg(bp + iw + 1);
      }
#pragma unroll
      for (int jj = 0; jj < 2; jj++) {
        const int ix = (int)Ku[jj], iy = (int)Kv[jj];
        const float dx = Ku[jj] - ix, dy = Kv[jj] - iy, dxdy = dx * dy;
        const float w11 = dxdy, w10 = dy - dxdy, w01 = dx - dxdy, w00 = 1 - dx - dy + dxdy;
        const float h0 = w11 * tap[jj][3].x + w10 * tap[jj][2].x + w01 * tap[jj][1].x + w00 * tap[jj][0].x;
        const float h1 = w11 * tap[jj][3].y + w10 * tap[jj][2].y + w01 * tap[jj][1].y + w00 * tap[jj][0].y;
        const float h2 = w11 * tap[jj][3].z + w10 * tap[jj][2].z + w01 * tap[jj][1].z + w00 * tap[jj][0].z;
        fin = fin && isfinite(h0);
        const float cj = jj ? col.y : col.x, wj = jj ? wgt.y : wgt.x;
        const float residual = h0 - (pc[24] * cj + pc[25]);
        const float drdA = cj - pc[26];
        float w = sqrtf(oth / (oth + (h1 * h1 + h2 * h2)));
        w = 0.5f * (w + wj);
        const float ar = fabsf(residual);
        float hw = ar < huber ? 1.f : huber / ar;
        sv[15] += w * w * hw * residual * residual * (2.f - hw);
        if (hw < 1.f) hw = sqrtf(hw);
        hw = hw * w;
        const float gx = h1 * hw, gy = h2 * hw;
        const float resF = residual * hw;
        const float ja = drdA * hw, jb = hw;
        const float jaF = zA ? 0.f : ja, jbF = zB ? 0.f : jb;
        float ra = resF;
        if constexpr (MARG) { ra = (((resF - gx * jpx) - gy * jpy) - jaF * dp6) - jbF * dp7; rtz[jj] = ra; }
        sv[0] += gx * gx; sv[2] += gy * gy; sv[1] += gx * gy;
        sv[3] += ja * gx; sv[4] += ja * gy; sv[5] += jb * gx; sv[6] += jb * gy;
        sv[7] += ja * ja; sv[8] += ja * jb; sv[9] += jb * jb;
        sv[10] += ra * gx; sv[11] += ra * gy; sv[12] += ra * jaF; sv[13] += ra * jbF; sv[14] += ra * ra;
        sv[16] += hw * hw * (gx * gx + gy * gy);
      }
    }
    clk_stamp<CLK>(clk, 3, __float_as_uint(sv[0]));
    {  // every sample finite, and the sums of the residual's 8 pixels in all 4 lanes (butterfly over the lane bits 0, 1)
      const unsigned bal = __ballot_sync(0xffffffffu, fin);
      live = live && (((bal >> (lane & ~3)) & 0xfu) == 0xfu);
#pragma unroll
      for (int k = 0; k < 17; k++) {
        sv[k] += __shfl_xor_sync(0xffffffffu, sv[k], 1);
        sv[k] += __shfl_xor_sync(0xffffffffu, sv[k], 2);
      }
    }
    PixSums s = {sv[0], sv[1], sv[2], sv[3], sv[4], sv[5], sv[6], sv[7], sv[8], sv[9], sv[10], sv[11], sv[12], sv[13], sv[14]};
    const float energy = sv[15], wJI2 = sv[16];

    // ---- classification and per-residual outputs (identical in the 4 lanes; lane 0 writes)
    int newState;
    float newEnergy;
    if (st == RES_NONE) { newState = RES_NONE; newEnergy = 0.f; }
    else if (!live) { newState = RES_OOB; newEnergy = en_old; }
    else if (energy > TH || wJI2 < 2.f) { newState = RES_OUTLIER; newEnergy = TH; }
    else { newState = RES_IN; newEnergy = energy; }
    const bool in = (newState == RES_IN);
    if (st != RES_NONE && q == 0) {
      e_sum = newEnergy;
      n_in = in; n_oob = (newState == RES_OOB); n_outl = (newState == RES_OUTLIER);
    }
    if constexpr (MARG) {
      if (masked) *reinterpret_cast<float2*>(W.marg_rtz + (size_t)slot * 8 + 2 * q) = in ? make_float2(rtz[0], rtz[1]) : make_float2(0.f, 0.f);
    }
    if (valid && masked && q == 0) {
      W.st_new[slot] = (uint8_t)newState;
      W.en_new[slot] = newEnergy;
      const float ewo = (st == RES_NONE || !live) ? -1.f : energy;
      W.en_wo[slot] = ewo;
      if (t == nf - 1 && W.en_wo_newest_host) W.en_wo_newest_host[p] = ewo;  // zero-copy: the host's percentile needs no D2H call
      const size_t plane = (size_t)MAXF * mp;
      W.cpt[slot] = cKu; W.cpt[plane + slot] = cKv; W.cpt[2 * plane + slot] = new_idepth;
    }

    // ---- takeDataF, per-point terms, Schur-vector rows (split over the lanes)
    float jp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, Hdd = 0.f, bd = 0.f, Hcd0 = 0.f, Hcd1 = 0.f, Hcd2 = 0.f, Hcd3 = 0.f;
    if (in) {
      if constexpr (!MARG) geo_jac(pc, Kl0, Kl1, cu, cv, drescale, new_idepth, fx, fy, fxi, fyi, x, y, ddx, ddy);
      const float J0 = s.JI00 * ddx + s.JI10 * ddy, J1 = s.JI10 * ddx + s.JI11 * ddy;
#pragma unroll
      for (int k = 0; k < 6; k++) jp[k] = x[4 + k] * J0 + y[4 + k] * J1;
      jp[6] = s.JabJI00 * ddx + s.JabJI01 * ddy; jp[7] = s.JabJI10 * ddx + s.JabJI11 * ddy;
      Hdd = J0 * ddx + J1 * ddy;
      bd = s.JIr0 * ddx + s.JIr1 * ddy;
      Hcd0 = x[0] * J0 + y[0] * J1; Hcd1 = x[1] * J0 + y[1] * J1; Hcd2 = x[2] * J0 + y[2] * J1; Hcd3 = x[3] * J0 + y[3] * J1;
      if (valid && q == 0) {
        float4* gj = reinterpret_cast<float4*>(W.jpjd + (size_t)slot * 8);
        gj[0] = make_float4(jp[0], jp[1], jp[2], jp[3]);
        gj[1] = make_float4(jp[4], jp[5], jp[6], jp[7]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 10; k++) { x[k] = 0.f; y[k] = 0.f; }
      s = PixSums{0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    }
    {  // lane q: rows 2q, 2q+1 of adHost * JpJdF and of the (diagonal) adTarget product; lanes 1..3 also carry the per-point scalars
      const float r0 = ah[0].x * jp[0] + ah[0].y * jp[1] + ah[0].z * jp[2] + ah[0].w * jp[3] + ah[1].x * jp[4] + ah[1].y * jp[5] + ah[1].z * jp[6] + ah[1].w * jp[7];
      const float r1 = ah[2].x * jp[0] + ah[2].y * jp[1] + ah[2].z * jp[2] + ah[2].w * jp[3] + ah[3].x * jp[4] + ah[3].y * jp[5] + ah[3].z * jp[6] + ah[3].w * jp[7];
      const float j0 = (q == 0) ? jp[0] : (q == 1) ? jp[2] : (q == 2) ? jp[4] : jp[6];
      const float j1 = (q == 0) ? jp[1] : (q == 1) ? jp[3] : (q == 2) ? jp[5] : jp[7];
      if (pair_ok) {
        S.rec[t][2 * q][pl] = r0; S.rec[t][2 * q + 1][pl] = r1;
        S.Wv[pl][4 + 8 * t + 2 * q] = at2.x * j0; S.Wv[pl][4 + 8 * t + 2 * q + 1] = at2.y * j1;
      }
      const float e0 = (q == 0) ? Hdd : (q == 1) ? Hcd0 : (q == 2) ? Hcd2 : (in ? 1.f : 0.f);
      const float e1 = (q == 0) ? bd : (q == 1) ? Hcd1 : (q == 2) ? Hcd3 : 0.f;
      const int k0 = (q == 0) ? 8 : (q == 1) ? 10 : (q == 2) ? 12 : 14;
      if (pair_ok) { S.rec[t][k0][pl] = e0; S.rec[t][k0 + 1][pl] = e1; }
    }

    // ---- the pair's 13x13 block, rows split over the 4 lanes: lane q forms rows q, q+4, q+8 of the 10 geometric rows (all columns from the
    // row group's first column on: compile-time register indices; the few sub-diagonal products are discarded) and lane 2 carries the 6
    // (a, b, r) entries; then a transposing butterfly over the warp's 8 points (16 + 8 + 4 exchanges) leaves 4 values per lane
    float v[32];
    {
      const float alq[3] = {s.JI00 * ((q == 0) ? x[0] : (q == 1) ? x[1] : (q == 2) ? x[2] : x[3]) + s.JI10 * ((q == 0) ? y[0] : (q == 1) ? y[1] : (q == 2) ? y[2] : y[3]),
                            s.JI00 * ((q == 0) ? x[4] : (q == 1) ? x[5] : (q == 2) ? x[6] : x[7]) + s.JI10 * ((q == 0) ? y[4] : (q == 1) ? y[5] : (q == 2) ? y[6] : y[7]),
                            s.JI00 * ((q == 0) ? x[8] : (q == 1) ? x[9] : 0.f) + s.JI10 * ((q == 0) ? y[8] : (q == 1) ? y[9] : 0.f)};
      const float beq[3] = {s.JI10 * ((q == 0) ? x[0] : (q == 1) ? x[1] : (q == 2) ? x[2] : x[3]) + s.JI11 * ((q == 0) ? y[0] : (q == 1) ? y[1] : (q == 2) ? y[2] : y[3]),
                            s.JI10 * ((q == 0) ? x[4] : (q == 1) ? x[5] : (q == 2) ? x[6] : x[7]) + s.JI11 * ((q == 0) ? y[4] : (q == 1) ? y[5] : (q == 2) ? y[6] : y[7]),
                            s.JI10 * ((q == 0) ? x[8] : (q == 1) ? x[9] : 0.f) + s.JI11 * ((q == 0) ? y[8] : (q == 1) ? y[9] : 0.f)};
      const float xq[3] = {(q == 0) ? x[0] : (q == 1) ? x[1] : (q == 2) ? x[2] : x[3], (q == 0) ? x[4] : (q == 1) ? x[5] : (q == 2) ? x[6] : x[7],
                           (q == 0) ? x[8] : (q == 1) ? x[9] : 0.f};
      const float yq[3] = {(q == 0) ? y[0] : (q == 1) ? y[1] : (q == 2) ? y[2] : y[3], (q == 0) ? y[4] : (q == 1) ? y[5] : (q == 2) ? y[6] : y[7],
                           (q == 0) ? y[8] : (q == 1) ? y[9] : 0.f};
      // column c of a row: c < 10: al x[c] + be y[c];  c = 10, 11: x_r JabJI(c-10,0) + y_r JabJI(c-10,1);  c = 12: x_r JIr0 + y_r JIr1
      int o = 0;
#pragma unroll
      for (int j = 0; j < 3; j++) {
#pragma unroll
        for (int c = 4 * j; c < 13; c++) {
          float val;
          if (c < 10) val = alq[j] * x[c] + beq[j] * y[c];
          else if (c == 10) val = xq[j] * s.JabJI00 + yq[j] * s.JabJI01;
          else if (c == 11) val = xq[j] * s.JabJI10 + yq[j] * s.JabJI11;
          else val = xq[j] * s.JIr0 + yq[j] * s.JIr1;
          v[o++] = val;   // o: 0..12 (rows 0-3), 13..21 (rows 4-7), 22..26 (rows 8-9)
        }
      }
      if (q == 2) { v[22] = s.Jab00; v[23] = s.Jab01; v[24] = s.Jabr0; v[25] = s.Jab11; v[26] = s.Jabr1; }   // lanes 2, 3 have no third row:
      v[27] = (q == 2) ? s.rr : 0.f;                                                                             // lane 2 carries the bottom block
      if (q == 3) { v[22] = v[23] = v[24] = v[25] = v[26] = 0.f; }
      v[28] = v[29] = v[30] = v[31] = 0.f;
    }
    static_for<0, 3>([&](auto sc) {
      constexpr int st2 = decltype(sc)::value, hstep = 16 >> st2, m = 16 >> st2;   // lane bits 4, 3, 2 = the warp's 8 points
      const bool up = (lane & m) != 0;
#pragma unroll
      for (int k = 0; k < hstep; k++) v[k] = (up ? v[k + hstep] : v[k]) + __shfl_xor_sync(0xffffffffu, up ? v[k] : v[k + hstep], m);
    });
    if (pair_ok) {  // lane (point-in-warp w8, q) holds positions 4 w8 + {0..3} of lane class q: position -> (row, column) -> packed index
      const int w8 = (lane >> 2) & 7;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int pos = 4 * w8 + k;
        int idx = -1;
        if (pos < 13) { const int rr = q, c = pos; if (c >= rr) idx = top_off(rr) + c - rr; }
        else if (pos < 22) { const int rr = q + 4, c = pos - 13 + 4; if (c >= rr) idx = top_off(rr) + c - rr; }
        else if (pos < 28) {
          if (q < 2) { const int rr = q + 8, c = pos - 22 + 8; if (pos < 27 && c >= rr) idx = top_off(rr) + c - rr; }
          else if (q == 2) idx = TOP_TRI + (pos - 22);
        }
        if (idx >= 0) S.pair[t][half][idx] = v[k];
      }
    }
  }
  }
  {  // counters: warp sums
    float es = e_sum, fin = (float)n_in, foob = (float)n_oob, fout = (float)n_outl;
#pragma unroll
    for (int m = 1; m < 32; m <<= 1) {
      es += __shfl_xor_sync(0xffffffffu, es, m);
      fin += __shfl_xor_sync(0xffffffffu, fin, m);
      foob += __shfl_xor_sync(0xffffffffu, foob, m);
      fout += __shfl_xor_sync(0xffffffffu, fout, m);
      rs_step2 += __shfl_xor_sync(0xffffffffu, rs_step2, m);
      rs_nid += __shfl_xor_sync(0xffffffffu, rs_nid, m);
      rs_cnt += __shfl_xor_sync(0xffffffffu, rs_cnt, m);
    }
    if (lane == 0) {
      S.misc[warp][0] = es; S.misc[warp][1] = fin; S.misc[warp][2] = foob; S.misc[warp][3] = fout;
      S.misc[warp][4] = rs_step2; S.misc[warp][5] = rs_nid; S.misc[warp][6] = rs_cnt; S.misc[warp][7] = 0.f;
    }
  }
  cp_async_wait_all();
  __syncthreads();
  clk_stamp<CLK>(clk, 4);

  // ---------------------------------------------------------------- phases B and C: two block-wide passes over regular items, long items
  // first (at P = 16 and up to 7 frames every item of a pass has its own thread).  Every entry keeps the summation order of the formulas quoted below, so the
  // partial blob, the Schur vectors and pout are the same bit for bit however the items are dealt.  Loops over the targets are rolled
  // where unrolling would only add code: this code runs once per chunk and is fetched cold.
  const int nt = nf - 1;  // target slot r <-> frame r + (r >= h)
  double* __restrict__ out = W.part + (size_t)chunk * PART_STRIDE;
  {  // pass 1: G and the target blocks, phase B, H[C,C] / b[C] and the counters: everything that reads only phase A's results
    const int nG = nt * 26;
#pragma unroll 1
    for (int e = tid; e < nG + 9 * P + 28; e += nthreads) {
      if (e < nG) {
        // target t, column c of [P | Q | p](h,t), rows i0..i0+3: [P|Q|p][k][c] = H13[4+k][col], col = 4..11 (P), 0..3 (Q), 12 (p).
        // G(t)[i][c] = sum_k adHost[i][k] [P|Q|p][k][c] (k ascending), and the target's own blocks, which need no adHost:
        // H[t,t] = At P At^T, H[t,C] = At Q, b[t] = At p (AccumulatedTopHessian.cpp:L270-286)
        const int rh = e / 13, c = e - rh * 13, i0 = (rh & 1) * 4;
        const int t = (rh >> 1) + ((rh >> 1) >= h ? 1 : 0);
        const int col = (c < 8) ? 4 + c : (c < 12 ? c - 8 : 12);
        double m[8];
#pragma unroll
        for (int k = 0; k < 8; k++) m[k] = (double)pair_entry<NH>(S.pair[t], 4 + k, col);
        const double dTc = S.dT[t][c & 7];
        // partial-blob slot of target row i in column c: [D 64 | C 32 | b 8] -> first row i0, stride per row
        const int os = (c < 8) ? 8 : (c < 12 ? 4 : 1);
        double* o = out + t * PART_SLOT + ((c < 8) ? 64 + c : (c < 12 ? 120 + c : 160)) + i0 * os;
#pragma unroll
        for (int ii = 0; ii < 4; ii++) {
          const int i = i0 + ii;
          double g = 0.0;
#pragma unroll
          for (int k = 0; k < 8; k++) g += S.AhD[t][i * 8 + k] * m[k];
          S.G[t][i][c] = g;
          double v = S.dT[t][i] * (i0 ? m[4 + ii] : m[ii]);
          if (c < 8) v = v * dTc;
          o[ii * os] = v;
        }
      } else if (e < nG + 9 * P) {  // phase B: per point (AccumulatedSCHessian.cpp:L36-58); lanes = points: conflict-free reads of rec[t][k][.]
        const int k = (e - nG) / P, pl2 = (e - nG) & (P - 1);
        if (pl2 >= ch_count) continue;
        if (k < 8) {  // host block of the Schur vector: sum over the targets, ascending
          float sum = 0.f;
#pragma unroll
          for (int tt = 0; tt < MAXF; tt++) {
            const float v = S.rec[tt][k][pl2];
            if (tt < nf && tt != h) sum += v;
          }
          S.Wv[pl2][4 + 8 * h + k] = sum;
        } else {
          const int p = ch_start + pl2;
          float Hdd = 0.f, bd = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f, ngood = 0.f;
#pragma unroll 1
          for (int r = 0; r < nt; r++) {
            const int tt = r + (r >= h ? 1 : 0);
            Hdd += S.rec[tt][8][pl2]; bd += S.rec[tt][9][pl2]; c0 += S.rec[tt][10][pl2]; c1 += S.rec[tt][11][pl2];
            c2 += S.rec[tt][12][pl2]; c3 += S.rec[tt][13][pl2]; ngood += S.rec[tt][14][pl2];
          }
          float prior = S.prior[pl2];
          bool masked = true;
          if constexpr (MARG) { masked = __ldg(W.marg_mask + p) != 0; prior *= __ldg(&W.marg->priorFac); }
          float HdiF = 0.f, bdSum = 0.f, w0 = 0.f, w1 = 0.f, w2 = 0.f, w3 = 0.f;
          if (ngood > 0.f) {
            float H = Hdd + prior;
            if (H < 1e-10f) H = 1e-10f;
            HdiF = 1.0f / H;
            bdSum = MARG ? bd : bd + prior * (S.id[pl2] - S.idz[pl2]);  // shiftPriorToZero (AccumulatedSCHessian.cpp:L47-50)
            w0 = c0; w1 = c1; w2 = c2; w3 = c3;
          }
          S.Wv[pl2][0] = w0; S.Wv[pl2][1] = w1; S.Wv[pl2][2] = w2; S.Wv[pl2][3] = w3;
          S.Wv[pl2][N] = bdSum;
#pragma unroll 1
          for (int c = N + 1; c < W.NW; c++) S.Wv[pl2][c] = 0.f;  // padding columns of the last 4x4 tiles
          S.hdi[pl2] = HdiF;
          if (masked) {
            float4* po = reinterpret_cast<float4*>(W.pout + (size_t)p * 8);
            po[0] = make_float4(Hdd, bd, c0, c1);
            po[1] = make_float4(c2, c3, HdiF, bdSum);
          }
        }
      } else if (e < nG + 9 * P + 20) {  // H[C,C] (4x4) and b[C] = sum_t Q-block / p of the pair blocks, t ascending
        const int i = (e - nG - 9 * P) / 5, j = (e - nG - 9 * P) - i * 5;
        double val = 0.0;
#pragma unroll 1
        for (int r = 0; r < nt; r++) val += (double)pair_entry<NH>(S.pair[r + (r >= h ? 1 : 0)], i, j < 4 ? j : 12);
        out[PART_CC + (j < 4 ? i * 4 + j : 16 + i)] = val;
      } else {  // the counters: warp sums in warp order, 4 loads in flight
        const int k = e - nG - 9 * P - 20;
        double val = 0.0;
#pragma unroll 1
        for (int wv = 0; wv < nwarps; wv += 4) {
          float v[4];
#pragma unroll
          for (int u = 0; u < 4; u++) v[u] = S.misc[min(wv + u, 15)][k];
#pragma unroll
          for (int u = 0; u < 4; u++)
            if (wv + u < nwarps) val += (double)v[u];
        }
        out[PART_MISC + k] = val;
      }
    }
  }
  __syncthreads();
  {  // pass 2: what needs G, and the Schur vectors -> global.  The 64 H[h,h] items (48-term chains) come first.
    const int nO = nt * 16;
#pragma unroll 1
    for (int e = tid; e < 64 + nO + 8 + P * W.T; e += nthreads) {
      if (e < 64) {  // H[h,h] = sum_t (Ah P) Ah^T: t ascending, then k; the next target's operands load under the current 8-term chain
        const int i = e >> 3, j = e & 7;
        double val = 0.0;
        double2 g[4], a[4];
        const int t0 = (h == 0) ? 1 : 0;
#pragma unroll
        for (int u = 0; u < 4; u++) { g[u] = reinterpret_cast<const double2*>(&S.G[t0][i][0])[u]; a[u] = reinterpret_cast<const double2*>(&S.AhD[t0][j * 8])[u]; }
#pragma unroll 1
        for (int r = 0; r < nt; r++) {
          const int tn = min(r + 1 + (r + 1 >= h ? 1 : 0), MAXF - 1);  // next target (in bounds on the last trip; not used there)
          double2 gn[4], an[4];
#pragma unroll
          for (int u = 0; u < 4; u++) { gn[u] = reinterpret_cast<const double2*>(&S.G[tn][i][0])[u]; an[u] = reinterpret_cast<const double2*>(&S.AhD[tn][j * 8])[u]; }
#pragma unroll
          for (int u = 0; u < 4; u++) { val += g[u].x * a[u].x; val += g[u].y * a[u].y; }
#pragma unroll
          for (int u = 0; u < 4; u++) { g[u] = gn[u]; a[u] = an[u]; }
        }
        out[h * PART_SLOT + 64 + e] = val;
      } else if (e < 64 + nO) {  // H[h,t] = (Ah P) At^T: 4 entries of row i
        const int eo = e - 64, r = eo >> 4, i = (eo >> 1) & 7, j0 = (eo & 1) * 4;
        const int t = r + (r >= h ? 1 : 0);
#pragma unroll
        for (int v = 0; v < 4; v++) out[t * PART_SLOT + i * 8 + j0 + v] = S.G[t][i][j0 + v] * S.dT[t][j0 + v];
      } else if (e < 64 + nO + 8) {  // row i of H[h,C] = sum_t Ah Q and b[h] = sum_t Ah p, t ascending
        const int i = e - 64 - nO;
        double c0 = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0, bh = 0.0;
#pragma unroll 1
        for (int r = 0; r < nt; r++) {
          const int t2 = r + (r >= h ? 1 : 0);
          const double2 q01 = *reinterpret_cast<const double2*>(&S.G[t2][i][8]), q23 = *reinterpret_cast<const double2*>(&S.G[t2][i][10]);
          c0 += q01.x; c1 += q01.y; c2 += q23.x; c3 += q23.y; bh += S.G[t2][i][12];
        }
        double* o = out + h * PART_SLOT;
        o[128 + i * 4] = c0; o[128 + i * 4 + 1] = c1; o[128 + i * 4 + 2] = c2; o[128 + i * 4 + 3] = c3;
        o[160 + i] = bh;
      } else {  // Schur vectors -> global, transposed ([4-column group][point] float4) so that phase E reads them coalesced
        const int ew = e - 64 - nO - 8, g4 = ew / P, pl2 = ew & (P - 1);
        if (pl2 >= ch_count) continue;
        W.wg[(size_t)g4 * mp + ch_start + pl2] = *reinterpret_cast<const float4*>(&S.Wv[pl2][4 * g4]);
        if (g4 == 0) W.hdig[ch_start + pl2] = S.hdi[pl2];
      }
    }
  }
  __syncthreads();  // shared memory is reused by the next chunk (persistent case)
  clk_stamp<CLK>(clk, 5);
}

// phases D / E for one window: the work is split over `ncta` CTAs, this one acting as CTA `vcta`
template <int P, int LPR, bool CLK = false>
__device__ __forceinline__ void fused_reduce(const BAWinDev& W, FusedSmem<P, LPR>& S, bool ok, const int vcta, const int ncta,
                                             unsigned long long* clk = nullptr) {
  const int nf = W.nf, N = W.N, mp = W.mp;
  const int tid = threadIdx.x, nthreads = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;

  const int nH = N * N + N;
  double* __restrict__ R = W.result;
  double* __restrict__ RH = W.result_host;
  const bool xch = W.xc.nranks > 1;
  const double* __restrict__ part = W.part;

  // ---------------------------------------------------------------- phase D: H_top / b_top / counters, 16 lanes per result entry
  // item list: [unordered frame pairs a<b: 64 entries each][diagonal blocks: nf x 64][H[.,C]: nf x 32][b: nf x 8][CC 16][bC 4][counters 7]
  // Usually one pass over the items (16-lane groups in the grid >= items), every lane sums <= 12 chunk partials per segment whose loads
  // are all in flight together, then a 4-step butterfly.  Fixed order => bit-reproducible.
  const int npair = nf * (nf - 1) / 2;
  const int n_off = npair * 64, n_diag = nf * 64, n_c = nf * 32, n_b = nf * 8;
  const int nitems = n_off + n_diag + n_c + n_b + 16 + 4 + (ACC_MISC - 1);  // the last counter slot is the error flag: written on error only
  const int grp = tid >> 4, gl = tid & 15, groups_per_cta = nthreads >> 4;
  const int nch = W.nchunks;
  // with the peer exchange on: pass 0 (sum + push) -> phase E (Gram tiles + push) -> pass 1 (pull) -> phase E pull: the NVLink round trip of
  // the H_top entries overlaps the Gram computation
  // items are dealt from the LAST CTA down: the first CTAs carry the second Schur tile of phase E (tile vcta + ncta), so the two tails
  // land on different CTAs
  const int dcta = ncta - 1 - vcta;
  auto phase_d = [&](const int pass) {
    for (int base = dcta * groups_per_cta; base < nitems; base += ncta * groups_per_cta) {  // CTA-uniform trip count (shuffles below)
      const int item = base + grp;
      const bool act = item < nitems;
      // decode: up to two (offset, chunk range) segments and up to two destinations
      int off0 = 0, lo0 = 0, hi0 = act ? nch : 0, off1 = 0, lo1 = 0, hi1 = 0, d0 = 0, d1 = -1;
      int e = act ? item : nitems - 1;
      if (e < n_off) {
        const int q = e >> 6, ij = e & 63, i = ij >> 3, j = ij & 7;
        int a = 0, rem = q;
        while (rem >= nf - 1 - a) { rem -= nf - 1 - a; a++; }
        const int b = a + 1 + rem;
        off0 = b * PART_SLOT + i * 8 + j; lo0 = W.chunk_beg[a]; hi0 = act ? W.chunk_beg[a + 1] : lo0;
        off1 = a * PART_SLOT + j * 8 + i; lo1 = W.chunk_beg[b]; hi1 = act ? W.chunk_beg[b + 1] : lo1;
        d0 = (4 + 8 * a + i) * N + 4 + 8 * b + j; d1 = (4 + 8 * b + j) * N + 4 + 8 * a + i;
      } else if ((e -= n_off) < n_diag) {
        const int a = e >> 6, ij = e & 63;
        off0 = a * PART_SLOT + 64 + ij;
        d0 = (4 + 8 * a + (ij >> 3)) * N + 4 + 8 * a + (ij & 7);
      } else if ((e -= n_diag) < n_c) {
        const int a = e >> 5, ic = e & 31;
        off0 = a * PART_SLOT + 128 + ic;
        d0 = (4 + 8 * a + (ic >> 2)) * N + (ic & 3); d1 = (ic & 3) * N + 4 + 8 * a + (ic >> 2);
      } else if ((e -= n_c) < n_b) {
        off0 = (e >> 3) * PART_SLOT + 160 + (e & 7);
        d0 = N * N + 4 + e;
      } else if ((e -= n_b) < 16) {
        off0 = PART_CC + e; d0 = (e >> 2) * N + (e & 3);
      } else if ((e -= 16) < 4) {
        off0 = PART_CC + 16 + e; d0 = N * N + e;
      } else {
        e -= 4;
        off0 = PART_MISC + e; d0 = nH + W.ntiles * 16 + e;
      }
      if (pass == 0) {
        double sum = 0.0;
        if (hi0 - lo0 <= 96 && hi1 - lo1 <= 96) {  // both segments in one round trip: <= 6 partials per lane each, summed in the same order
          double v[12];
#pragma unroll
          for (int u = 0; u < 12; u++) {
            const int c = (u < 6 ? lo0 : lo1) + gl + 16 * (u % 6);
            v[u] = (c < (u < 6 ? hi0 : hi1)) ? __ldcg(part + (u < 6 ? off0 : off1) + (size_t)c * PART_STRIDE) : 0.0;
          }
#pragma unroll
          for (int u = 0; u < 12; u++) sum += v[u];
        } else {
#pragma unroll 1
          for (int seg = 0; seg < 2; seg++) {
            const int lo = seg ? lo1 : lo0, hi = seg ? hi1 : hi0;
            const double* __restrict__ src = part + (seg ? off1 : off0);
            for (int c0 = lo + gl; c0 < hi; c0 += 192) {
              double v[12];
#pragma unroll
              for (int u = 0; u < 12; u++) v[u] = (c0 + 16 * u < hi) ? __ldcg(src + (size_t)(c0 + 16 * u) * PART_STRIDE) : 0.0;
#pragma unroll
              for (int u = 0; u < 12; u++) sum += v[u];
            }
          }
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 8);
        sum += __shfl_xor_sync(0xffffffffu, sum, 4);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        if (gl == 0 && act) {
          if (xch) { R[d0] = sum; xchg_push(W.xc, d0, sum); }
          else { R[d0] = sum; if (d1 >= 0) R[d1] = sum; if (RH) { RH[d0] = sum; if (d1 >= 0) RH[d1] = sum; } }
        }
      } else {  // warp-collective: both 16-lane groups of the warp wait together
        const double sum = xchg_pull_sum_group(W.xc, d0, (gl == 0 && act) ? R[d0] : 0.0, act, ok);
        if (gl == 0 && act) {
          R[d0] = sum; if (d1 >= 0) R[d1] = sum;
          if (RH) { RH[d0] = sum; if (d1 >= 0) RH[d1] = sum; }
        }
      }
    }
    };
  phase_d(0);
  clk_stamp<CLK>(clk, 7);

  // ---------------------------------------------------------------- phase E: [H_sc | b_sc] = sum_p HdiF w_p w_p^T as 4x4 tiles over ALL points
  // of the window: a CTA takes tiles vcta, vcta + ncta (both in ONE pass over the points when the grid has fewer CTAs than tiles)
  {
    const int T = W.T, npts = W.npts;
    for (int tile0 = vcta; tile0 < W.ntiles; tile0 += 2 * ncta) {
      const int tile1 = tile0 + ncta;
      const bool two = tile1 < W.ntiles;
      int ti0 = 0, rem = tile0;
      while (rem >= T - ti0) { rem -= T - ti0; ti0++; }
      const int tj0 = ti0 + rem;
      int ti1 = 0;
      rem = two ? tile1 : tile0;
      while (rem >= T - ti1) { rem -= T - ti1; ti1++; }
      const int tj1 = ti1 + rem;
      float a[2][4][4];
#pragma unroll
      for (int q = 0; q < 2; q++)
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) a[q][i][j] = 0.f;
      const float4* __restrict__ wi0 = W.wg + (size_t)ti0 * mp;
      const float4* __restrict__ wj0 = W.wg + (size_t)tj0 * mp;
      const float4* __restrict__ wi1 = W.wg + (size_t)ti1 * mp;
      const float4* __restrict__ wj1 = W.wg + (size_t)tj1 * mp;
#pragma unroll 4
      for (int p = tid; p < npts; p += nthreads) {
        const float sc = __ldcg(W.hdig + p);
        const float4 wi = __ldcg(wi0 + p), wj = __ldcg(wj0 + p);
        const float si[4] = {sc * wi.x, sc * wi.y, sc * wi.z, sc * wi.w};
        const float vj[4] = {wj.x, wj.y, wj.z, wj.w};
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) a[0][i][j] += si[i] * vj[j];
        if (two) {  // CTA-uniform
          const float4 xi = __ldcg(wi1 + p), xj = __ldcg(wj1 + p);
          const float ti[4] = {sc * xi.x, sc * xi.y, sc * xi.z, sc * xi.w};
          const float uj[4] = {xj.x, xj.y, xj.z, xj.w};
#pragma unroll
          for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) a[1][i][j] += ti[i] * uj[j];
        }
      }
      // per-thread fp32 sums over <= npts / nthreads points; transposing warp butterfly in fp32 (31 exchanges for the 32 values: lane L ends with
      // the warp's sum of value L over its <= 160 points; half the instructions of the fp64 form, and this straight-line code is fetched
      // once per CTA, where instruction fetch is the stall), then fp64 across the warps in a fixed order through shared memory
      {
        float d[32];
#pragma unroll
        for (int qq = 0; qq < 2; qq++)
#pragma unroll
          for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) d[qq * 16 + i * 4 + j] = a[qq][i][j];
        static_for<0, 5>([&](auto sc) {
          constexpr int st2 = decltype(sc)::value, hstep = 16 >> st2, m = 16 >> st2;
          const bool up = (lane & m) != 0;
#pragma unroll
          for (int k = 0; k < hstep; k++) d[k] = (up ? d[k + hstep] : d[k]) + __shfl_xor_sync(0xffffffffu, up ? d[k] : d[k + hstep], m);
        });
        S.red[warp][lane] = (double)d[0];   // lane L: value index 16 b4 + 8 b3 + 4 b2 + 2 b1 + b0 = L
      }
      __syncthreads();
      if (tid < 32) {  // the whole first warp (the exchange below is warp-collective)
        const bool own = tid < 16 || two;
        double d = 0.0;
        for (int wv = 0; wv < nwarps; wv++) d += S.red[wv][tid];
        const int idx = nH + (tid < 16 ? tile0 : tile1) * 16 + (tid & 15);
        if (own) {
          R[idx] = d;
          if (xch) xchg_push(W.xc, idx, d);
          else if (RH) RH[idx] = d;
        }
      }
      __syncthreads();
    }
  }
  clk_stamp<CLK>(clk, 8);
  if (xch) {
    phase_d(1);
    if (tid < 32) {  // pull of the Gram tiles: same (tile, lane) ownership as above, so R[idx] is this lane's own earlier store
      for (int tile0 = vcta; tile0 < W.ntiles; tile0 += 2 * ncta) {
        const int tile1 = tile0 + ncta;
        const bool own = tid < 16 || tile1 < W.ntiles;
        const int idx = nH + (tid < 16 ? tile0 : tile1) * 16 + (tid & 15);
        const double d = xchg_pull_sum_lanes(W.xc, idx, own ? R[idx] : 0.0, own, ok);
        if (own) {
          R[idx] = d;
          if (RH) RH[idx] = d;
        }
      }
    }
  }
  if (!__syncthreads_and(ok) && tid == 0) {  // barrier / peer timeout seen by any thread: raise the error slot of the counters (checked by the host)
    R[nH + W.ntiles * 16 + 7] = 1.0;
    if (RH) RH[nH + W.ntiles * 16 + 7] = 1.0;
  }
}

// MARG = true is the marginalisation launch (dmv_ba_marginalize_points): only the points flagged in W.marg_mask take part, their
// residuals are re-linearised from scratch (PointFrameResidual::resetOOB; FullSystem.cpp:L826-838), EFResidual::fixLinearizationF
// (EnergyFunctionalStructs.cpp:L88-114) turns resF into res_toZeroF, and the accumulation is AccumulatedTopHessian::addPoint<2> +
// AccumulatedSCHessian::addPoint(p, shiftPriorToZero = false) with priorF * idepthFixPriorMargFac (EnergyFunctional.cpp:L678-742).
// Two configurations: chunk_points = 16 -> (P = 16, LPR = 4): 448 threads, 4 lanes per residual (the latency-oriented default for ONE window);
//                     chunk_points = 32 -> (P = 32, LPR = 1): 224 threads, one thread per residual (fewest instructions: batches / large windows)
template <int P> struct FusedCfgOf { static constexpr int LPR = (P == 16) ? 4 : 1, TPB = (P == 16) ? 448 : 224; };

// CLK = true: the phase clock (clk_stamp) into clk[gridDim.x][NCLK]; measurement only, launched by launch_fused_kernel_clocked alone
template <int P, bool MARG, bool CLK = false>
__global__ void __launch_bounds__(FusedCfgOf<P>::TPB, 1)
    ba_fused_kernel(const __grid_constant__ BAWinDev W, const __grid_constant__ BAIter it, unsigned long long* clk) {
  constexpr int LPR = FusedCfgOf<P>::LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FusedSmem<P, LPR>& S = *reinterpret_cast<FusedSmem<P, LPR>*>(smem_raw);
  clk_stamp<CLK>(clk, 0);
#pragma unroll 1
  for (int chunk = blockIdx.x; chunk < W.nchunks; chunk += gridDim.x) fused_chunk<P, LPR, MARG, CLK>(W, it, S, chunk, clk);
  const bool ok = grid_barrier(W.bar, W.bar_target);  // every chunk of the window is done
  clk_stamp<CLK>(clk, 6);
  fused_reduce<P, LPR, CLK>(W, S, ok, blockIdx.x, gridDim.x, clk);
}

// Batched variant (SURVEY.md §8d): B independent windows in ONE launch.  Descriptors and per-iteration tables come from global memory;
// work items = (window, chunk) pairs dealt round-robin to the resident CTAs; after the grid barrier every window's reduction is spread
// over all CTAs, rotated per window so that the Schur tiles of different windows land on different CTAs.
template <int P>
__global__ void __launch_bounds__(FusedCfgOf<P>::TPB, P == 32 ? 2 : 1)
    ba_fused_batch_kernel(const BAWinDev* __restrict__ gW, const BAIter* __restrict__ gIt, const __grid_constant__ BABatchHdr hdr) {
  constexpr int LPR = FusedCfgOf<P>::LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FusedSmem<P, LPR>& S = *reinterpret_cast<FusedSmem<P, LPR>*>(smem_raw);
#pragma unroll 1
  for (int item = blockIdx.x; item < hdr.total; item += gridDim.x) {
    int w = 0;
    while (w + 1 < hdr.B && item >= hdr.prefix[w + 1]) w++;
    fused_chunk<P, LPR, false>(gW[w], gIt[w], S, item - hdr.prefix[w]);
  }
  const bool ok = grid_barrier(hdr.bar, hdr.bar_target);
#pragma unroll 1
  for (int w = 0; w < hdr.B; w++) fused_reduce<P, LPR>(gW[w], S, ok, (int)((blockIdx.x + (unsigned)w * 41u) % gridDim.x), gridDim.x);
}

// ---------------------------------------------------------------------------------------------------------------------------
// launch: cooperative (all CTAs resident); shared-memory opt-in and occupancy are cached PER DEVICE (cudaFuncSetAttribute is a
// per-device setting), under a mutex: handles on several devices / threads of one process are fine
// ---------------------------------------------------------------------------------------------------------------------------
struct FusedCfg { bool done = false; int max_ctas = 0; };
static std::mutex g_cfg_mutex;

template <int P, bool MARG, bool CLK = false>
static cudaError_t launch_cfg(BAWinDev& W, const BAIter& it, cudaStream_t s, unsigned* bar_count, unsigned long long* clk = nullptr) {
  static FusedCfg cfg[64];
  constexpr int TPB = FusedCfgOf<P>::TPB;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const int smem = (int)sizeof(FusedSmem<P, FusedCfgOf<P>::LPR>);
  const int threads = TPB;  // fixed block size: the summation orders of phases D / E depend on it, and batched launches must reproduce single ones bit for bit
  int max_ctas;
  {
    std::lock_guard<std::mutex> lk(g_cfg_mutex);
    FusedCfg& c = cfg[dev & 63];
    if (!c.done) {
      e = cudaFuncSetAttribute(ba_fused_kernel<P, MARG, CLK>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (e != cudaSuccess) return e;
      int per_sm = 0, sms = 0;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba_fused_kernel<P, MARG, CLK>, TPB, smem);
      if (e != cudaSuccess) return e;
      e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      if (e != cudaSuccess) return e;
      c.max_ctas = per_sm * sms;
      c.done = true;
    }
    max_ctas = c.max_ctas;
  }
  const int grid = min(W.nchunks, max_ctas);
  *bar_count += (unsigned)grid;   // monotonic arrival counter: every CTA of this launch adds one
  W.bar_target = *bar_count;
  void* args[3] = {(void*)&W, (void*)&it, (void*)&clk};
  return cudaLaunchCooperativeKernel((const void*)ba_fused_kernel<P, MARG, CLK>, dim3(grid), dim3(threads), args, (size_t)smem, s);
}

template <int P>
static cudaError_t launch_batch_cfg(const BAWinDev* gW, const BAIter* gIt, BABatchHdr& hdr, int max_nf, cudaStream_t s, unsigned* bar_count) {
  static FusedCfg cfg[64];
  constexpr int TPB = FusedCfgOf<P>::TPB;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const int smem = (int)sizeof(FusedSmem<P, FusedCfgOf<P>::LPR>);
  const int threads = TPB;
  (void)max_nf;
  int max_ctas;
  {
    std::lock_guard<std::mutex> lk(g_cfg_mutex);
    FusedCfg& c = cfg[dev & 63];
    if (!c.done) {
      e = cudaFuncSetAttribute(ba_fused_batch_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (e != cudaSuccess) return e;
      int per_sm = 0, sms = 0;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba_fused_batch_kernel<P>, TPB, smem);
      if (e != cudaSuccess) return e;
      e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      if (e != cudaSuccess) return e;
      c.max_ctas = per_sm * sms;
      c.done = true;
    }
    max_ctas = c.max_ctas;
  }
  const int grid = min(hdr.total, max_ctas);
  *bar_count += (unsigned)grid;
  hdr.bar_target = *bar_count;
  void* args[3] = {(void*)&gW, (void*)&gIt, (void*)&hdr};
  return cudaLaunchCooperativeKernel((const void*)ba_fused_batch_kernel<P>, dim3(grid), dim3(threads), args, (size_t)smem, s);
}

cudaError_t launch_fused_batch_kernel(int P, const BAWinDev* gW, const BAIter* gIt, BABatchHdr& hdr, int max_nf, cudaStream_t s, unsigned* bar_count) {
  return (P == 32) ? launch_batch_cfg<32>(gW, gIt, hdr, max_nf, s, bar_count) : launch_batch_cfg<16>(gW, gIt, hdr, max_nf, s, bar_count);
}

// W.bar_target is filled in here; *bar_count is the handle's running arrival count
cudaError_t launch_fused_kernel(BAWinDev& W, const BAIter& it, bool marg, cudaStream_t s, unsigned* bar_count) {
  if (W.P == 32) return marg ? launch_cfg<32, true>(W, it, s, bar_count) : launch_cfg<32, false>(W, it, s, bar_count);
  return marg ? launch_cfg<16, true>(W, it, s, bar_count) : launch_cfg<16, false>(W, it, s, bar_count);
}

// the linearisation launch with the phase clock (measurement only): clk holds >= grid x NCLK stamps, *grid receives the CTA count
cudaError_t launch_fused_kernel_clocked(BAWinDev& W, const BAIter& it, cudaStream_t s, unsigned* bar_count, unsigned long long* clk, int* grid) {
  const unsigned before = *bar_count;
  const cudaError_t e = (W.P == 32) ? launch_cfg<32, false, true>(W, it, s, bar_count, clk) : launch_cfg<16, false, true>(W, it, s, bar_count, clk);
  *grid = (int)(*bar_count - before);
  return e;
}

}  // namespace dmv
