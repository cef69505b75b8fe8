// TEST INFRASTRUCTURE ONLY — CPU restatement of the selection half of FullSystem::activatePointsMT (reference FullSystem.cpp:L642-717):
// CoarseDistanceMap::makeDistanceMap (CoarseTracker.cpp:L931-967), growDistBFS (L979-1073), addIntoDistFinal (L1076-1082) and the loop over the
// immature points of every other frame, serial and in the reference's order.  The oracle of dmv_ba_select_activation; pinned to the
// reference's compiled CoarseDistanceMap by ref_activation.cpp (tests/test_ref_pin_activation.py).  Built into liborc.so with the reference's
// flags (-O3, no -march).  Arguments as dmv_ba_select_args (include/dmvio_b200.h); actions 0 keep, 1 delete, 2 optimise.
#include <cmath>
#include <cstdint>
#include <utility>
#include <vector>

namespace {

struct DistMap {
  int w1, h1;
  std::vector<float> d;
  std::vector<int> l1, l2;   // bfsList1 / bfsList2 as (x, y) pairs
  DistMap(int w, int h) : w1(w), h1(h), d((size_t)w * h, 1000.f), l1(2 * (size_t)w * h + 2), l2(2 * (size_t)w * h + 2) {}

  void push(std::vector<int>& L, int& n, int x, int y) { L[2 * n] = x; L[2 * n + 1] = y; n++; }
  void relax(std::vector<int>& L, int& n, int idx, int x, int y, int k) {
    if (d[idx] > k) { d[idx] = k; push(L, n, x, y); }
  }
  void grow(int bfsNum) {
    for (int k = 1; k < 40; k++) {
      const int bfsNum2 = bfsNum;
      std::swap(l1, l2);
      bfsNum = 0;
      for (int i = 0; i < bfsNum2; i++) {
        const int x = l2[2 * i], y = l2[2 * i + 1];
        if (x == 0 || y == 0 || x == w1 - 1 || y == h1 - 1) continue;
        const int idx = x + y * w1;
        relax(l1, bfsNum, idx + 1, x + 1, y, k);
        relax(l1, bfsNum, idx - 1, x - 1, y, k);
        relax(l1, bfsNum, idx + w1, x, y + 1, k);
        relax(l1, bfsNum, idx - w1, x, y - 1, k);
        if (k % 2 != 0) {
          relax(l1, bfsNum, idx + 1 + w1, x + 1, y + 1, k);
          relax(l1, bfsNum, idx - 1 + w1, x - 1, y + 1, k);
          relax(l1, bfsNum, idx - 1 - w1, x - 1, y - 1, k);
          relax(l1, bfsNum, idx + 1 - w1, x + 1, y - 1, k);
        }
      }
    }
  }
  void add(int u, int v) {
    l1[0] = u; l1[1] = v;
    d[u + w1 * v] = 0;
    grow(1);
  }
};

// Vec3f ptp = KRKi * Vec3f(u, v, 1) + Kt * x;  int u = ptp[0] / ptp[2] + 0.5f (x86-64: cvttss2si)
inline bool project(const float* T, float u, float v, float x, int w1, int h1, int& iu, int& iv, float& p0) {
  float ptp[3];
  for (int k = 0; k < 3; k++) ptp[k] = ((T[3 * k] * u + T[3 * k + 1] * v) + T[3 * k + 2] * 1.0f) + T[9 + k] * x;
  iu = ptp[0] / ptp[2] + 0.5f;
  iv = ptp[1] / ptp[2] + 0.5f;
  p0 = ptp[0];
  return iu > 0 && iv > 0 && iu < w1 && iv < h1;
}

}  // namespace

extern "C" {

// returns the size of toOptimize; opt must hold imm_offset[nf] entries; map (w1*h1) may be NULL
int orc_act_select(int w1, int h1, int nf, int newest, const float* tab12, const uint8_t* flagged, int na, const float* au, const float* av,
                   const float* aid, const int32_t* ah, const int32_t* off, const float* u, const float* v, const float* idmin, const float* idmax,
                   const int32_t* status, const float* interval, const float* quality, const float* type, float minActDist, float minTraceQuality,
                   int32_t* action, int32_t* opt, float* map) {
  DistMap M(w1, h1);
  if (na > w1 * h1) { M.l1.resize(2 * (size_t)na + 2); M.l2.resize(2 * (size_t)na + 2); }   // makeDistanceMap lists every seed, duplicates included
  int numItems = 0;
  for (int f = 0; f < nf; f++) {   // makeDistanceMap: frames in order, each frame's points in order
    if (f == newest) continue;
    for (int p = 0; p < na; p++) {
      if (ah[p] != f) continue;
      int iu, iv;
      float p0;
      if (!project(tab12 + 12 * f, au[p], av[p], aid[p], w1, h1, iu, iv, p0)) continue;
      M.d[iu + w1 * iv] = 0;
      M.push(M.l1, numItems, iu, iv);
    }
  }
  M.grow(numItems);
  int nopt = 0;
  for (int f = 0; f < nf; f++) {
    for (int i = off[f]; i < off[f + 1]; i++) action[i] = 0;
    if (f == newest) continue;
    for (int i = off[f]; i < off[f + 1]; i++) {
      if (!std::isfinite(idmax[i]) || status[i] == 2) { action[i] = 1; continue; }
      const int st = status[i];
      const bool canActivate = (st == 0 || st == 3 || st == 4 || st == 1) && interval[i] < 8 && quality[i] > minTraceQuality && (idmax[i] + idmin[i]) > 0;
      if (!canActivate) {
        if (flagged[f] || st == 1) action[i] = 1;
        continue;
      }
      int iu, iv;
      float p0;
      if (project(tab12 + 12 * f, u[i], v[i], 0.5f * (idmax[i] + idmin[i]), w1, h1, iu, iv, p0)) {
        const float dist = M.d[iu + w1 * iv] + (p0 - floorf((float)(p0)));
        if (dist >= minActDist * type[i]) {
          M.add(iu, iv);
          action[i] = 2;
          opt[nopt++] = i;
        }
      } else {
        action[i] = 1;
      }
    }
  }
  if (map)
    for (size_t c = 0; c < M.d.size(); c++) map[c] = M.d[c];
  return nopt;
}

// addIntoDistFinal for each cell of a list in order, on a map (w1*h1, in/out): the flood alone, for tests/test_ref_pin_activation.py
void orc_act_grow(int w1, int h1, float* map, int nadd, const int32_t* add_xy) {
  DistMap M(w1, h1);
  for (size_t c = 0; c < M.d.size(); c++) M.d[c] = map[c];
  for (int s = 0; s < nadd; s++) M.add(add_xy[2 * s], add_xy[2 * s + 1]);
  for (size_t c = 0; c < M.d.size(); c++) map[c] = M.d[c];
}
}
