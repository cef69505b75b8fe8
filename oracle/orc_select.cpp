// TEST INFRASTRUCTURE ONLY — CPU restatement of PixelSelector (FullSystem/PixelSelector2.cpp) and of the raster loop of
// FullSystem::makeNewTraces (FullSystem.cpp:L1640-1667), the oracle of dmv_ct_make_new_traces.  select() stays the reference's literal
// serial loop; it additionally counts the "mixed" pot-blocks it meets (a level-0 candidate under some of the 16 directions but not all),
// the blocks the device resolves on its serial chain.  The ImmaturePoint constructor is the existing restatement (orc.ip_init, applied in
// oracle/select.py).  Built into liborc.so with the reference's flags.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct Settings {
  float minGradHistCut, minGradHistAdd, gradDownweightPerLevel;
  int selectDirectionDistribution, gammaWeightsPixelSelect;
};

// glibc random_r.c, TYPE_3: srand(seed) seeds r[0..30] with the Park-Miller recurrence (Schrage's method), r[31..33] = r[0..2], discards 310
// outputs; rand() = (r[i-31] + r[i-3]) >> 1 in 32-bit arithmetic
void random_pattern(unsigned seed, size_t n, unsigned char* out) {
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
  for (size_t k = 0; k < n; k++) out[k] = (unsigned char)((int)((uint32_t)r[344 + k] >> 1) & 0xFF);
}

struct Frame {
  int w[3], h[3];
  const float* dI[3];          // [I, dx, dy] per pixel
  std::vector<float> asg[3];   // absSquaredGrad
};

// FrameHessian::makeImages' absSquaredGrad (HessianBlocks.cpp:L169-189) from the given [I, dx, dy] levels; rows 0 and h-1, which the reference
// never writes, are 0
float getBGradOnly(const float* B, float color) {   // HessianBlocks.h:L394-400
  int c = color + 0.5f;
  if (c < 5) c = 5;
  if (c > 250) c = 250;
  return B[c + 1] - B[c];
}
void make_asg(Frame& F, const float* B, int gammaW) {
  for (int l = 0; l < 3; l++) {
    const int wl = F.w[l], hl = F.h[l];
    F.asg[l].assign((size_t)wl * hl, 0.f);
    for (int idx = wl; idx < wl * (hl - 1); idx++) {
      const float dx = F.dI[l][3 * idx + 1], dy = F.dI[l][3 * idx + 2];
      F.asg[l][idx] = dx * dx + dy * dy;
      if (gammaW == 1) {
        const float gw = getBGradOnly(B, F.dI[l][3 * idx]);
        F.asg[l][idx] *= gw * gw;
      }
    }
  }
}

int computeHistQuantil(int* hist, float below) {   // L82-91
  int th = hist[0] * below + 0.5f;
  for (int i = 0; i < 90; i++) {
    th -= hist[i + 1];
    if (th < 0) return i;
  }
  return 90;
}

struct Selector {
  int w, h, bW = 16, bH = 16, nbW, nbH, thsStep;
  std::vector<unsigned char> randomPattern;
  std::vector<int> gradHist;
  std::vector<float> ths, thsSmoothed;
  Settings S;
  long long nMixed = 0;

  void makeHists(const Frame& F) {   // L94-157
    const float* mapmax0 = F.asg[0].data();
    int w32 = nbW, h32 = nbH;
    thsStep = w32;
    for (int y = 0; y < h32; y++)
      for (int x = 0; x < w32; x++) {
        const float* map0 = mapmax0 + bW * x + bH * y * w;
        int* hist0 = gradHist.data();
        std::memset(hist0, 0, sizeof(int) * 50);
        for (int j = 0; j < bH; j++)
          for (int i = 0; i < bW; i++) {
            int it = i + bW * x, jt = j + bH * y;
            if (it > w - 2 || jt > h - 2 || it < 1 || jt < 1) continue;
            int g = sqrtf(map0[i + j * w]);
            if (g > 48) g = 48;
            hist0[g + 1]++;
            hist0[0]++;
          }
        ths[x + y * w32] = computeHistQuantil(hist0, S.minGradHistCut) + S.minGradHistAdd;
      }
    for (int y = 0; y < h32; y++)
      for (int x = 0; x < w32; x++) {
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
        thsSmoothed[x + y * w32] = (sum / num) * (sum / num);
      }
  }

  // L311-454
  void select(const Frame& F, float* map_out, int pot, float thFactor, int n[3]) {
    const float* map0 = F.dI[0];
    const float *mapmax0 = F.asg[0].data(), *mapmax1 = F.asg[1].data(), *mapmax2 = F.asg[2].data();
    const int w1 = F.w[1], w2 = F.w[2];
    static const float directions[16][2] = {{0, 1.0000},      {0.3827, 0.9239},  {0.1951, 0.9808},  {0.9239, 0.3827},  {0.7071, 0.7071},
                                            {0.3827, -0.9239}, {0.8315, 0.5556},  {0.8315, -0.5556}, {0.5556, -0.8315}, {0.9808, 0.1951},
                                            {0.9239, -0.3827}, {0.7071, -0.7071}, {0.5556, 0.8315},  {0.9808, -0.1951}, {1.0000, 0.0000},
                                            {0.1951, -0.9808}};
    auto dotabs = [](const float* g, const float* d) { float s = 0.f; s += g[0] * d[0]; s += g[1] * d[1]; return fabsf(s); };   // Vec2f::dot
    std::memset(map_out, 0, sizeof(float) * w * h);
    float dw1 = S.gradDownweightPerLevel;
    float dw2 = dw1 * dw1;
    int n3 = 0, n2 = 0, n4 = 0;
    for (int y4 = 0; y4 < h; y4 += (4 * pot))
      for (int x4 = 0; x4 < w; x4 += (4 * pot)) {
        int my3 = std::min((4 * pot), h - y4);
        int mx3 = std::min((4 * pot), w - x4);
        int bestIdx4 = -1; float bestVal4 = 0;
        const float* dir4 = directions[randomPattern[n2] & 0xF];
        for (int y3 = 0; y3 < my3; y3 += (2 * pot))
          for (int x3 = 0; x3 < mx3; x3 += (2 * pot)) {
            int x34 = x3 + x4, y34 = y3 + y4;
            int my2 = std::min((2 * pot), h - y34);
            int mx2 = std::min((2 * pot), w - x34);
            int bestIdx3 = -1; float bestVal3 = 0;
            const float* dir3 = directions[randomPattern[n2] & 0xF];
            for (int y2 = 0; y2 < my2; y2 += pot)
              for (int x2 = 0; x2 < mx2; x2 += pot) {
                int x234 = x2 + x34, y234 = y2 + y34;
                int my1 = std::min(pot, h - y234);
                int mx1 = std::min(pot, w - x234);
                int bestIdx2 = -1; float bestVal2 = 0;
                const float* dir2 = directions[randomPattern[n2] & 0xF];
                unsigned mask = 0;   // not in the reference: the directions under which this pot-block has a level-0 candidate
                for (int y1 = 0; y1 < my1; y1 += 1)
                  for (int x1 = 0; x1 < mx1; x1 += 1) {
                    int idx = x1 + x234 + w * (y1 + y234);
                    int xf = x1 + x234, yf = y1 + y234;
                    if (xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4) continue;
                    float pixelTH0 = thsSmoothed[xf / bW + (yf / bH) * thsStep];
                    float pixelTH1 = pixelTH0 * dw1;
                    float pixelTH2 = pixelTH1 * dw2;
                    const float* ag0d = map0 + 3 * idx + 1;
                    float ag0 = mapmax0[idx];
                    if (ag0 > pixelTH0 * thFactor) {
                      for (int d = 0; d < 16; d++)
                        if ((S.selectDirectionDistribution ? dotabs(ag0d, directions[d]) : ag0) > 0) mask |= 1u << d;
                      float dirNorm = dotabs(ag0d, dir2);
                      if (!S.selectDirectionDistribution) dirNorm = ag0;
                      if (dirNorm > bestVal2) { bestVal2 = dirNorm; bestIdx2 = idx; bestIdx3 = -2; bestIdx4 = -2; }
                    }
                    if (bestIdx3 == -2) continue;
                    float ag1 = mapmax1[(int)(xf * 0.5f + 0.25f) + (int)(yf * 0.5f + 0.25f) * w1];
                    if (ag1 > pixelTH1 * thFactor) {
                      float dirNorm = dotabs(ag0d, dir3);
                      if (!S.selectDirectionDistribution) dirNorm = ag1;
                      if (dirNorm > bestVal3) { bestVal3 = dirNorm; bestIdx3 = idx; bestIdx4 = -2; }
                    }
                    if (bestIdx4 == -2) continue;
                    float ag2 = mapmax2[(int)(xf * 0.25f + 0.125) + (int)(yf * 0.25f + 0.125) * w2];
                    if (ag2 > pixelTH2 * thFactor) {
                      float dirNorm = dotabs(ag0d, dir4);
                      if (!S.selectDirectionDistribution) dirNorm = ag2;
                      if (dirNorm > bestVal4) { bestVal4 = dirNorm; bestIdx4 = idx; }
                    }
                  }
                if (mask != 0 && mask != 0xFFFFu) nMixed++;
                if (bestIdx2 > 0) { map_out[bestIdx2] = 1; bestVal3 = 1e10; n2++; }
              }
            if (bestIdx3 > 0) { map_out[bestIdx3] = 2; bestVal4 = 1e10; n3++; }
          }
        if (bestIdx4 > 0) { map_out[bestIdx4] = 4; n4++; }
      }
    n[0] = n2; n[1] = n3; n[2] = n4;
  }

  // L158-307 (the FAST branch is commented out in the reference; plot = false); the histogram is rebuilt on every call
  int makeMaps(const Frame& F, float* map_out, float density, int recursionsLeft, float thFactor, int& currentPotential, bool hists, float& quotiaOut) {
    float numHave = 0, numWant = density, quotia;
    int idealPotential = currentPotential;
    if (hists) makeHists(F);
    int n[3];
    select(F, map_out, currentPotential, thFactor, n);
    numHave = n[0] + n[1] + n[2];
    quotia = numWant / numHave;
    float K = numHave * (currentPotential + 1) * (currentPotential + 1);
    idealPotential = sqrtf(K / numWant) - 1;
    if (idealPotential < 1) idealPotential = 1;
    if (recursionsLeft > 0 && quotia > 1.25 && currentPotential > 1) {
      if (idealPotential >= currentPotential) idealPotential = currentPotential - 1;
      currentPotential = idealPotential;
      return makeMaps(F, map_out, density, recursionsLeft - 1, thFactor, currentPotential, false, quotiaOut);
    } else if (recursionsLeft > 0 && quotia < 0.25) {
      if (idealPotential <= currentPotential) idealPotential = currentPotential + 1;
      currentPotential = idealPotential;
      return makeMaps(F, map_out, density, recursionsLeft - 1, thFactor, currentPotential, false, quotiaOut);
    }
    quotiaOut = quotia;
    int numHaveSub = numHave;
    if (quotia < 0.95) {
      int wh = w * h, rn = 0;
      unsigned char charTH = 255 * quotia;
      for (int i = 0; i < wh; i++)
        if (map_out[i] != 0) {
          if (randomPattern[rn] > charTH) { map_out[i] = 0; numHaveSub--; }
          rn++;
        }
    }
    currentPotential = idealPotential;
    return numHaveSub;
  }
};

}  // namespace

extern "C" {

void orc_sel_random_pattern(unsigned seed, int n, unsigned char* out) { random_pattern(seed, (size_t)n, out); }

// one makeMaps call: dI0/1/2 = levels 0-2 as [I, dx, dy]; s = {minGradHistCut, minGradHistAdd, gradDownweightPerLevel}, si = {selectDirectionDistribution,
// gammaWeightsPixelSelect}; *potential in/out; *n_mixed = mixed pot-blocks met; *quotia = the last select's numWant / numHave.  Returns numHaveSub.
int orc_sel_make_maps(int w, int h, const float* dI0, const float* dI1, const float* dI2, const float* B, const float* s, const int* si, float density,
                      int recursionsLeft, float thFactor, int* potential, float* map_out, long long* n_mixed, float* quotia) {
  Frame F;
  const float* lv[3] = {dI0, dI1, dI2};
  for (int l = 0; l < 3; l++) { F.w[l] = w >> l; F.h[l] = h >> l; F.dI[l] = lv[l]; }
  Selector P;
  P.w = w; P.h = h; P.nbW = w / 16; P.nbH = h / 16;
  P.S = Settings{s[0], s[1], s[2], si[0], si[1]};
  make_asg(F, B, P.S.gammaWeightsPixelSelect);
  P.randomPattern.resize((size_t)w * h);
  random_pattern(3141592, (size_t)w * h, P.randomPattern.data());
  P.gradHist.assign(100 * (1 + P.nbW) * (1 + P.nbH), 0);
  P.ths.assign(P.nbW * P.nbH + 100, 0.f);
  P.thsSmoothed.assign(P.nbW * P.nbH + 100, 0.f);
  const int r = P.makeMaps(F, map_out, density, recursionsLeft, thFactor, *potential, true, *quotia);
  *n_mixed = P.nMixed;
  return r;
}

// makeNewTraces' raster loop (L1652-1657): the pixels an ImmaturePoint is constructed for, in push_back order
int orc_sel_trace_pixels(int w, int h, const float* map, int32_t* u, int32_t* v, float* type) {
  const int patternPadding = 2;
  int n = 0;
  for (int y = patternPadding + 1; y < h - patternPadding - 2; y++)
    for (int x = patternPadding + 1; x < w - patternPadding - 2; x++) {
      int i = x + y * w;
      if (map[i] == 0) continue;
      u[n] = x; v[n] = y; type[n] = map[i]; n++;
    }
  return n;
}

}  // extern "C"
