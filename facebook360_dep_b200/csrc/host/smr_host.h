// SimpleMeshRenderer's host-side image steps (source/render/SimpleMeshRenderer.cpp): the background compositing, the
// stereo layouts and the png conversion.  Header-only and free of GL and CUDA, so that the app and the CPU checker
// (tests/canopy_oracle.cpp, which exports them for the numpy and cv2 pins) run the same code.  Images are float
// B, G, R, A, row-major, top row first.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace smr {

// posForwardUp's rotation in fp32 as Eigen forms it: with right = up.cross(-forward), the rows of forwardUp(f, u) for
// f = forward.normalized(), u = right.cross(forward).normalized() are u.cross(-f), u, -f (row-major R[9]).  False when
// the rows are not unitary within 0.001 (forwardUp's CHECK).
inline bool forwardUp(const float* forward, const float* up, float* R) {
  auto cross = [](const float* a, const float* b, float* r) {
    r[0] = a[1] * b[2] - a[2] * b[1];
    r[1] = a[2] * b[0] - a[0] * b[2];
    r[2] = a[0] * b[1] - a[1] * b[0];
  };
  auto normalized = [](const float* a, float* r) {
    const float n = std::sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]);
    for (int c = 0; c < 3; ++c) r[c] = a[c] / n;
  };
  const float negF[3] = {-forward[0], -forward[1], -forward[2]};
  float right[3], u0[3], f[3], u[3];
  cross(up, negF, right);
  cross(right, forward, u0);
  normalized(forward, f);
  normalized(u0, u);
  const float nf[3] = {-f[0], -f[1], -f[2]};
  cross(u, nf, R);
  for (int c = 0; c < 3; ++c) {
    R[3 + c] = u[c];
    R[6 + c] = nf[c];
  }
  for (int r = 0; r < 3; ++r)
    for (int q = 0; q < 3; ++q) {
      const float dot = (R[3 * r] * R[3 * q] + R[3 * r + 1] * R[3 * q + 1]) + R[3 * r + 2] * R[3 * q + 2];
      if (!(std::fabs(dot - (r == q ? 1.0f : 0.0f)) <= 0.001f)) return false;
    }
  return true;
}

// alphaBlend: alpha * fore + (1 - alpha) * back, alpha + (1 - alpha) * back.a; a NaN alpha takes the background
inline void alphaBlend(float* fore, const float* back, size_t n) {
  for (size_t i = 0; i < n; ++i) {
    float* f = fore + 4 * i;
    const float* b = back + 4 * i;
    const float alpha = f[3];
    if (std::isnan(alpha)) {
      std::memcpy(f, b, 4 * sizeof(float));
      continue;
    }
    for (int c = 0; c < 3; ++c) f[c] = alpha * f[c] + (1 - alpha) * b[c];
    f[3] = alpha + (1 - alpha) * b[3];
  }
}

// backgroundEquirect: every pixel of a snapshot-sized image whose alpha is not 1 is blended over the background
// equirect's nearest texel in the direction of the pixel centre at the near plane.  fwdUp is posForwardUp's rotation
// (rows right, up, -forward); its inverse is the transpose, and the inverse's translation is `position`.  The reference
// formula (lon = atan2(-y, -x): -X in the centre column, +Y to its right, +Z in the top row) can index one past the last
// column or row at lon = -pi or lat = -pi/2, and takes asin of a normalised z that rounding can push past 1: both are
// clamped here.
inline void backgroundEquirect(float* fore, int width, int height, const float* equi, int ew, int eh,
                               const float* fwdUp, const float* position, double horizontalFovDeg) {
  const float kNearZ = 0.1f, kNearInfinity = 1e4f;
  const float xMax = (float)((double)kNearZ * std::tan(horizontalFovDeg / 180 * M_PI / 2));
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      float* f = fore + 4 * ((size_t)y * width + x);
      const float alpha = f[3];
      if (alpha == 1) continue;
      const float pixel[3] = {((x + 0.5f) / width * 2 - 1) * xMax, -((y + 0.5f) / height * 2 - 1) * xMax * height / width,
                              -kNearZ};
      float world[3];
      for (int r = 0; r < 3; ++r)
        world[r] = ((fwdUp[0 * 3 + r] * (kNearInfinity * pixel[0]) + fwdUp[1 * 3 + r] * (kNearInfinity * pixel[1])) +
                    fwdUp[2 * 3 + r] * (kNearInfinity * pixel[2])) +
                   position[r];
      const float lon = std::atan2(-world[1], -world[0]);
      const float norm = std::sqrt((world[0] * world[0] + world[1] * world[1]) + world[2] * world[2]);
      const float z = world[2] / norm;
      const float lat = std::asin(z > 1 ? 1.0f : (z < -1 ? -1.0f : z));
      const float equiX = (-lon / M_PI + 1) / 2 * ew;
      const float equiY = (-lat / M_PI + 0.5) * eh;
      const int ix = std::min(ew - 1, std::max(0, (int)equiX)), iy = std::min(eh - 1, std::max(0, (int)equiY));
      const float* b = equi + 4 * ((size_t)iy * ew + ix);
      if (std::isnan(alpha)) {
        std::memcpy(f, b, 4 * sizeof(float));
        continue;
      }
      for (int c = 0; c < 3; ++c) f[c] = alpha * f[c] + (1 - alpha) * b[c];
      f[3] = alpha + (1 - alpha) * b[3];
    }
}

// cv_util::convertImage<cv::Vec3w> (channels = 3) or <cv::Vec4w> (channels = 4) of a Vec4f image: convertTo(CV_16U,
// 65535) (saturate_cast of cvRound(v * 65535): round half to even, NaN -> 0), with BGRA -> BGR for 3 channels
inline std::vector<uint16_t> toPng16(const float* bgra, size_t n, int channels = 3) {
  std::vector<uint16_t> out(n * channels);
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < channels; ++c) {
      const float v = bgra[4 * i + c] * 65535.0f;
      uint16_t u = 0;
      if (v > -2147483648.0f && v < 2147483648.0f) {
        const long r = std::lrintf(v);
        u = (uint16_t)(r < 0 ? 0 : r > 65535 ? 65535 : r);
      }
      out[channels * i + c] = u;
    }
  return out;
}

// stereo layouts: tbstereo stacks the eyes vertically; lr180 puts the centre half (columns [w / 4, w / 4 + w / 2)) of
// each eye side by side; tb3dof stacks colour over disparity (the same as tbstereo's stacking)
inline std::vector<float> stackVertical(const std::vector<float>& top, const std::vector<float>& bottom) {
  std::vector<float> out(top);
  out.insert(out.end(), bottom.begin(), bottom.end());
  return out;
}

inline std::vector<float> lr180(const std::vector<float>& left, const std::vector<float>& right, int w, int h) {
  const int x0 = w / 4, cw = w / 2;
  std::vector<float> out((size_t)2 * cw * h * 4);
  for (int y = 0; y < h; ++y)
    for (int e = 0; e < 2; ++e)
      std::memcpy(&out[((size_t)y * 2 * cw + (size_t)e * cw) * 4], &(e == 0 ? left : right)[((size_t)y * w + x0) * 4],
                  (size_t)cw * 4 * sizeof(float));
  return out;
}

}  // namespace smr
