// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// Bridges of the two sweep-view checkers (sweepview.mk): the reference's OWN GenerateCameraOverlaps.cpp and
// GenerateEquirect.cpp, compiled where they lie (main renamed), each into its own library because both define main and
// same-named gflags globals.  This file is compiled twice, with -DSWEEP_OVERLAPS or -DSWEEP_EQUIRECT, and exports the
// entry points of include/derp_sweepview.h that its app implements by calling the app's own functions:
//   libsweep_overlaps_ref.so  derp_sweep_overlaps -> projectSrcsToDst
//   libsweep_equirect_ref.so  derp_sweep_crop_bounds / derp_sweep_equirect -> createEquirect / createCroppedEquirect
//                             (bounds from createCroppedEquirect's own loop), derp_sweep_center_rig -> centerRig
// Cameras are built from the descriptors through the reference's JSON loader (%.17g round trip), ids "cam<i>".
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <opencv2/opencv.hpp>

#include "source/util/Camera.h"

#include "../include/derp_sweepview.h"

using namespace fb360_dep;
using Image = cv::Mat_<cv::Vec4f>;

#ifdef SWEEP_OVERLAPS
Image projectSrcsToDst(const Camera& camDst, const Camera::Rig& rigSrc, const std::vector<Image>& imagesSrc,
                       const float disparity);
#endif
#ifdef SWEEP_EQUIRECT
extern bool FLAGS_black_bg;
extern uint64_t FLAGS_height;
Image createEquirect(const Camera::Rig& rig, const std::vector<Image>& images, const size_t height, const size_t width,
                     const float depth);
Image createCroppedEquirect(const Camera::Rig& rig, const std::vector<Image>& images, const size_t height,
                            const size_t width, const float depth);
void centerRig(Camera::Rig& rig, std::string camera_id);
Camera::Vector3 getEquirectPoint(const double x, const double y, const double depth, const double width,
                                 const double height);
#endif

// SystemUtil.cpp is not linked: the renamed mains are never called
namespace fb360_dep::system_util {
void initDep(int&, char**&, const std::string) { std::abort(); }
}  // namespace fb360_dep::system_util

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& m) {
  g_err = m;
  return code;
}
std::string num17(double v) {
  char b[64];
  snprintf(b, sizeof b, "%.17g", v);
  return b;
}
std::string vecJson(const double* v, int n) {
  std::string s = "[";
  for (int i = 0; i < n; ++i) s += (i ? "," : "") + num17(v[i]);
  return s + "]";
}
Camera::Rig rigOf(const DerpCameraDesc* cams, int n) {
  static const char* kTypes[] = {"FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"};
  std::string json = "{\"cameras\":[";
  for (int i = 0; i < n; ++i) {
    const DerpCameraDesc& d = cams[i];
    json += std::string(i ? "," : "") + "{\"version\":1,\"type\":\"" + kTypes[d.type] + "\",\"id\":\"cam" +
            std::to_string(i) + "\",\"origin\":" + vecJson(d.origin, 3) + ",\"forward\":" + vecJson(d.forward, 3) +
            ",\"up\":" + vecJson(d.up, 3) + ",\"right\":" + vecJson(d.right, 3) +
            ",\"resolution\":" + vecJson(d.resolution, 2) + ",\"focal\":" + vecJson(d.focal, 2);
    if (d.has_principal) json += ",\"principal\":" + vecJson(d.principal, 2);
    json += ",\"distortion\":" + vecJson(d.distortion, 3);
    if (d.has_fov) json += ",\"fov\":" + num17(d.fov);
    json += "}";
  }
  return Camera::loadRigFromJsonString(json + "]}");
}
std::vector<Image> imagesOf(const float* const* images, const int32_t* sizes, int n) {
  std::vector<Image> out;
  for (int i = 0; i < n; ++i) {
    Image m(sizes[2 * i + 1], sizes[2 * i]);
    std::memcpy(m.data, images[i], (size_t)sizes[2 * i] * sizes[2 * i + 1] * sizeof(cv::Vec4f));
    out.push_back(m);
  }
  return out;
}
template <class F>
int guarded(F&& f) {
  try {
    return f();
  } catch (const std::exception& e) {
    return fail(DERP_EINVAL, e.what());
  }
}
}  // namespace

extern "C" {

const char* derp_backend(void) { return "reference-cpu"; }
const char* derp_last_error(void) { return g_err.c_str(); }

#ifdef SWEEP_OVERLAPS
int derp_sweep_overlaps(int, const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                        const int32_t* image_sizes, int dst, const float* disparities, int num_slices, float* out) {
  return guarded([&] {
    const Camera::Rig rig = rigOf(cams, num_cams);
    const std::vector<Image> images = imagesOf(images_bgra, image_sizes, num_cams);
    for (int k = 0; k < num_slices; ++k) {
      const Image m = projectSrcsToDst(rig[dst], rig, images, disparities[k]);
      const size_t bytes = (size_t)m.rows * m.cols * sizeof(cv::Vec4f);
      std::memcpy(reinterpret_cast<char*>(out) + k * bytes, m.data, bytes);
    }
    return DERP_OK;
  });
}
#endif

#ifdef SWEEP_EQUIRECT
// createCroppedEquirect's bounding-box loop (GenerateEquirect.cpp:139-156) is not a function of its own; this is that
// loop over the reference's getEquirectPoint and Camera::sees.
int derp_sweep_crop_bounds(int, const DerpCameraDesc* cams, int num_cams, int center, uint64_t height,
                           const float* depths, int num_depths, double* bounds) {
  return guarded([&] {
    Camera::Rig rig = rigOf(cams, num_cams);
    if (center >= 0) centerRig(rig, "cam" + std::to_string(center));
    const size_t width = 2 * height;
    for (int k = 0; k < num_depths; ++k) {
      const float depth = depths[k];
      double minX = width, maxX = 0, minY = height, maxY = 0;
      for (double x = 0; x < width; x++)
        for (double y = 0; y < height; y++) {
          const Camera::Vector3 p = getEquirectPoint(x, y, depth, width, height);
          for (int c = 0; c < int(rig.size()); c++) {
            Camera::Vector2 px;
            if (rig[c].sees(p, px)) {
              minX = floor(std::min(minX, x));
              maxX = ceil(std::max(maxX, x));
              minY = floor(std::min(minY, y));
              maxY = ceil(std::max(maxY, y));
            }
          }
        }
      bounds[4 * k] = minX;
      bounds[4 * k + 1] = maxX;
      bounds[4 * k + 2] = minY;
      bounds[4 * k + 3] = maxY;
    }
    return DERP_OK;
  });
}

// bounds == NULL: createEquirect; otherwise createCroppedEquirect, which recomputes its own box (the caller's bounds
// only select the mode; the test compares derp_sweep_crop_bounds separately)
int derp_sweep_equirect(int, const DerpCameraDesc* cams, int num_cams, int center, const float* const* images_bgra,
                        const int32_t* image_sizes, uint64_t height, const float* depths, int num_depths,
                        const double* bounds, int black_bg, float* const* out) {
  return guarded([&] {
    Camera::Rig rig = rigOf(cams, num_cams);
    if (center >= 0) centerRig(rig, "cam" + std::to_string(center));
    const std::vector<Image> images = imagesOf(images_bgra, image_sizes, num_cams);
    FLAGS_black_bg = black_bg != 0;
    FLAGS_height = height;
    for (int k = 0; k < num_depths; ++k) {
      const Image m = bounds ? createCroppedEquirect(rig, images, height, 2 * height, depths[k])
                             : createEquirect(rig, images, height, 2 * height, depths[k]);
      std::memcpy(out[k], m.data, (size_t)m.rows * m.cols * sizeof(cv::Vec4f));
    }
    return DERP_OK;
  });
}

int derp_sweep_center_rig(const DerpCameraDesc* cams, int num_cams, int center, DerpCameraDesc* out, double* rotation9) {
  return guarded([&] {
    Camera::Rig rig = rigOf(cams, num_cams);
    centerRig(rig, "cam" + std::to_string(center));
    for (int i = 0; i < num_cams; ++i) {
      out[i] = cams[i];
      for (int k = 0; k < 3; ++k) {
        out[i].origin[k] = rig[i].position[k];
        out[i].forward[k] = rig[i].forward()[k];
        out[i].up[k] = rig[i].up()[k];
        out[i].right[k] = rig[i].right()[k];
      }
      if (rotation9)
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) rotation9[9 * i + 3 * r + c] = rig[i].rotation(r, c);
    }
    return DERP_OK;
  });
}
#endif

}  // extern "C"
