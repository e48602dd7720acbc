// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// oracle/libeqrmesh_oracle.so: a CPU restatement of include/derp_eqrmesh.h, the mesh of CreateObjFromDisparityEquirect
// (source/conversion/CreateObjFromDisparityEquirect.cpp:56-71) before simplification: cv::resize INTER_LINEAR
// (cvprims_linear.h), mesh_util::getVertexesEquirect and getFaces(wrapHorizontally = true, isRigCoordinates = true)
// (source/render/MeshUtil.h:167-313), written from the reference's text.  Checked against the reference's own MeshUtil.h
// (oracle/_ref/libeqrmesh_ref.so, ref_bridge_eqrmesh.cpp) by tests/test_eqr_obj.py.  Recipe: eqrmesh.mk.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <tuple>
#include <vector>

#include "../include/derp_eqrmesh.h"
#include "cvprims_linear.h"

namespace {

thread_local std::string g_err;

int fail(const char* msg) {
  g_err = msg;
  return DERP_EINVAL;
}

// getTriangleMask, MeshUtil.h:167-220, with the corner distances given
unsigned triangleMask(const std::vector<double>& d, int base, int width, float tearRatio) {
  const double tl = d[base], tr = d[base + 1], bl = d[base + width], br = d[base + width + 1];
  std::vector<std::tuple<double, int>> v = {std::make_tuple(tl, 0), std::make_tuple(tr, 1), std::make_tuple(bl, 2),
                                            std::make_tuple(br, 3)};
  std::sort(v.begin(), v.end());  // literal: with NaN distances the order is whatever libstdc++'s insertion sort leaves
  if (std::get<0>(v.front()) / std::get<0>(v.back()) > tearRatio) {
    if (std::abs(tl - br) < std::abs(tr - bl)) return 1 << 1 | 1 << 2;
    return 1 << 0 | 1 << 3;
  }
  const double lo = std::get<0>(v.front()) / std::get<0>(v[2]);
  const double hi = std::get<0>(v[1]) / std::get<0>(v.back());
  if (lo >= tearRatio && lo > hi) return 1 << (std::get<1>(v.back()) ^ 0x3);
  if (hi >= tearRatio) return 1 << (std::get<1>(v.front()) ^ 0x3);
  return 0;
}

// addTriangle, MeshUtil.h:222-247
void triangle(int which, int base, int width, uint32_t* f) {
  switch (which) {
    case 0: f[0] = base + width, f[1] = base + 1, f[2] = base; break;
    case 1: f[0] = base, f[1] = base + width + 1, f[2] = base + 1; break;
    case 2: f[0] = base + width + 1, f[1] = base, f[2] = base + width; break;
    default: f[0] = base + 1, f[1] = base + width, f[2] = base + width + 1; break;
  }
}

}  // namespace

extern "C" {

const char* derp_last_error(void) { return g_err.c_str(); }

int derp_equirect_mesh_size(int width, int height, double scale, int* mesh_width, int* mesh_height) {
  if (!mesh_width || !mesh_height || !oracle::equirectGrid(width, height, scale, mesh_width, mesh_height))
    return fail("derp_equirect_mesh_size: bad arguments");
  return DERP_OK;
}

int derp_equirect_mesh(int /*device*/, const float* disparity, int width, int height, double scale, double max_depth,
                       float tear_ratio, double* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces) {
  int W = 0, H = 0;
  if (!oracle::equirectGrid(width, height, scale, &W, &H) || !disparity || !vertexes || !faces || !num_vertexes ||
      !num_faces)
    return fail("derp_equirect_mesh: bad arguments");
  std::vector<float> disp(disparity, disparity + (size_t)width * height);
  if (scale < 1) {  // cv::resize(disp, disp, Size(), scale, scale), INTER_LINEAR
    std::vector<float> small;
    int w2, h2;
    oracle::resizeLinearScaledF32(disp.data(), width, height, scale, small, &w2, &h2);
    disp.swap(small);
  }
  // getVertexesEquirect, MeshUtil.h:298-313
  const float maxDepth = (float)max_depth;
  const size_t n = (size_t)W * H;
  std::vector<double> norm(n);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const float u = float(x + 0.5) / float(W);
      const float v = float(y + 0.5) / float(H);
      const float theta = u * 2.0f * M_PI;
      const float phi = v * M_PI;
      const float depth = std::fmin(maxDepth, 1.0f / disp[(size_t)y * W + x]);
      const float c[3] = {std::sin(phi) * std::cos(theta), std::cos(phi), std::sin(phi) * std::sin(theta)};
      double* p = vertexes + ((size_t)y * W + x) * 3;
      for (int k = 0; k < 3; ++k) p[k] = (double)depth * (double)c[k];
      norm[(size_t)y * W + x] = std::sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);  // isRigCoordinates: the norm
    }
  // getFaces(wrapHorizontally = true, isRigCoordinates = true), MeshUtil.h:264-296
  size_t nf = 0;
  for (int y = 0; y < H - 1; ++y)
    for (int x = 0; x < W - 1; ++x) {
      const int base = y * W + x;
      const unsigned m = triangleMask(norm, base, W, tear_ratio);
      for (int t = 0; t < 4; ++t)
        if ((m >> t) & 1) triangle(t, base, W, faces + 3 * nf++);
    }
  for (int y = 0; y < H - 1; ++y) {
    const uint32_t base = (uint32_t)(y * W), w = (uint32_t)W;
    const uint32_t f[6] = {base + w, base, base + w - 1, base + w - 1, base + 2 * w - 1, base + w};
    std::memcpy(faces + nf * 3, f, sizeof f);
    nf += 2;
  }
  *num_vertexes = n;
  *num_faces = nf;
  return DERP_OK;
}

// As for the camera mesh, the simplifier is checked against the reference's own MeshSimplifier.cpp (oracle/_ref) only.
int derp_equirect_mesh_simplified(int, const float*, int, int, double, double, float, int, float, double*, uint32_t*,
                                  uint64_t*, uint64_t*) {
  return fail("derp_equirect_mesh_simplified: the oracle restatement stops before simplification; use oracle/_ref");
}

// test hook: the INTER_LINEAR restatement; dst holds the cvRound(size * scale) grid
void oracle_resize_linear_f32(const float* src, int sw, int sh, double scale, float* dst) {
  std::vector<float> out;
  int dw, dh;
  if (oracle::resizeLinearScaledF32(src, sw, sh, scale, out, &dw, &dh)) std::copy(out.begin(), out.end(), dst);
}

}  // extern "C"
