// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement of cv::resize(src, dst, Size(), f, f) with the default INTER_LINEAR on float 1-channel images, the
// resize CreateObjFromDisparityEquirect.cpp:59-62 applies for --scale < 1 (resize.cpp resizeGeneric_ with HResizeLinear /
// VResizeLinear).  Pinned to the cv2 4.13.0 wheel of this image by tests/golden/linear_vectors.npz (generator
// tests/golden/gen_linear_vectors.py, test tests/test_eqr_obj.py): <= 2.5e-7 absolute on (0, 1] data, not bit-exact —
// cv2's operation order is not fully restated.  Used by both equirect-mesh checkers (eqrmesh.mk): the OpenCV stand-in
// of refshim/ has no INTER_LINEAR, so the reference's glue calls this in place of cv::resize.
#pragma once

#include <algorithm>
#include <vector>

#include "cvprims.h"

namespace oracle {

// dsize = cvRound(size * f); a dsize equal to the source size is a copy; an empty one is cv::Exception (false here).
// Sample position p = (d + 0.5) / f - 0.5 in double, s = floor(p), weight a = float(p - s), taps (1.f - a, a).
// Columns: s < 0 -> (0, weight 0); s >= size - 1 -> a copy of column size - 1 (no product).  Rows: no clamp of the
// weight, only of the row index.  Every value is two fp32 products and one fp32 sum, unfused.
inline bool resizeLinearScaledF32(const float* src, int sw, int sh, double f, std::vector<float>& dst, int* dw, int* dh) {
  const int w = cvRoundD(sw * f), h = cvRoundD(sh * f);
  if (w < 1 || h < 1) return false;
  *dw = w;
  *dh = h;
  dst.resize((size_t)w * h);
  if (w == sw && h == sh) {
    std::copy(src, src + (size_t)sw * sh, dst.begin());
    return true;
  }
  const double inv = 1. / f;
  std::vector<float> rows((size_t)sh * w);
  for (int x = 0; x < w; ++x) {
    const double p = (x + 0.5) * inv - 0.5;
    int s = cvFloorD(p);
    float a = (float)(p - s);
    if (s < 0) s = 0, a = 0.f;
    const bool copy = s + 1 >= sw;
    if (copy) s = sw - 1;
    for (int y = 0; y < sh; ++y) {
      const float* S = src + (size_t)y * sw;
      rows[(size_t)y * w + x] = copy ? S[s] : S[s] * (1.f - a) + S[s + 1] * a;
    }
  }
  for (int y = 0; y < h; ++y) {
    const double p = (y + 0.5) * inv - 0.5;
    const int s = cvFloorD(p);
    const float b = (float)(p - s);
    const float* R0 = rows.data() + (size_t)std::min(std::max(s, 0), sh - 1) * w;
    const float* R1 = rows.data() + (size_t)std::min(std::max(s + 1, 0), sh - 1) * w;
    for (int x = 0; x < w; ++x) dst[(size_t)y * w + x] = R0[x] * (1.f - b) + R1[x] * b;
  }
  return true;
}

// the mesh grid of derp_equirect_mesh_size (include/derp_eqrmesh.h), shared by both checkers
inline bool equirectGrid(int width, int height, double scale, int* W, int* H) {
  if (width < 1 || height < 1 || !(scale > 0)) return false;
  const int w = scale < 1 ? cvRoundD(width * scale) : width, h = scale < 1 ? cvRoundD(height * scale) : height;
  if (w < 2 || h < 2 || (size_t)w * h * 2 >= (1ull << 31)) return false;
  *W = w;
  *H = h;
  return true;
}

}  // namespace oracle
