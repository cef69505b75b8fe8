// TEST INFRASTRUCTURE ONLY — CPU restatement of the per-frame part of Undistort::undistort<T> (src/dso/util/Undistort.cpp:L385-482)
// with PhotometricUndistorter::processFrame (L213-252), on the same tables the reference builds once per sequence (remapX / remapY,
// G, vignetteMapInv).  Same two passes and operation order as the reference: the photometric map over the whole raw image, then the
// bilinear remap.  Built with the reference's flags (-O3, no -march: scalar SSE2, no FMA) into oracle/liborc.so.
#include <cstring>
#include <vector>

template <typename T>
static void undistort_t(int w, int h, int wOrg, int hOrg, const float* remapX, const float* remapY, const float* G, const float* vigInv, int mode,
                        const T* image_in, float exposure, float factor, float* out) {
  const int wh = wOrg * hOrg;
  std::vector<float> data(wh);
  if (!G || exposure <= 0 || mode == 0) {  // L222-230
    for (int i = 0; i < wh; i++) data[i] = factor * image_in[i];
  } else {  // L231-246
    for (int i = 0; i < wh; i++) data[i] = G[image_in[i]];
    if (mode == 2)
      for (int i = 0; i < wh; i++) data[i] *= vigInv[i];
  }
  if (!remapX) {  // passthrough, L474-477
    std::memcpy(out, data.data(), sizeof(float) * w * h);
    return;
  }
  const float* in_data = data.data();
  for (int idx = w * h - 1; idx >= 0; idx--) {  // L421-465 (no benchmark noise)
    float xx = remapX[idx];
    float yy = remapY[idx];
    if (xx < 0)
      out[idx] = 0;
    else {
      int xxi = xx;
      int yyi = yy;
      xx -= xxi;
      yy -= yyi;
      float xxyy = xx * yy;
      const float* src = in_data + xxi + yyi * wOrg;
      out[idx] = xxyy * src[1 + wOrg] + (yy - xxyy) * src[wOrg] + (xx - xxyy) * src[1] + (1 - xx - yy + xxyy) * src[0];
    }
  }
}

extern "C" {
// raw: wOrg*hOrg pixels of bpp bytes (1 = uint8, 2 = uint16); out: w*h floats.  remapX = NULL: passthrough (w = wOrg, h = hOrg).
// G = NULL: no photometric calibration (PhotometricUndistorter::valid == false).
void orc_undistort(int w, int h, int wOrg, int hOrg, const float* remapX, const float* remapY, const float* G, const float* vigInv, int mode,
                   const void* raw, int bpp, float exposure, float factor, float* out) {
  if (bpp == 1)
    undistort_t(w, h, wOrg, hOrg, remapX, remapY, G, vigInv, mode, static_cast<const unsigned char*>(raw), exposure, factor, out);
  else
    undistort_t(w, h, wOrg, hOrg, remapX, remapY, G, vigInv, mode, static_cast<const unsigned short*>(raw), exposure, factor, out);
}
}
