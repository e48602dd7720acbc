// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// Bridge of the ProjectEquirectsToCameras checker (eqrproject.mk): the reference's OWN ProjectEquirectsToCameras.cpp,
// compiled where it lies (main renamed), linked with the reference's Camera.o and ImageUtil.o.  Exports
//   derp_project_equirect_masks  the app's per-pixel loop (ProjectEquirectsToCameras.cpp:99-124) over the reference's
//                                Camera::rig and image_util::worldToEquirect
//   ref_eqrproject_rescale       the app's own rescaleCameras at a given --width
// The loop is restated because it is not a function of its own in the app; its one deviation is the NaN guard: the
// reference converts a NaN equirect coordinate (acos of z > 1 near a pole) to int and indexes the mask with it, which
// is undefined, so here such a pixel is left unset, as the product library defines it.
// Cameras are built from the descriptors through the reference's JSON loader (%.17g round trip), ids "cam<i>".
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <opencv2/opencv.hpp>

#include "source/util/Camera.h"
#include "source/util/ImageUtil.h"

#include "../include/derp_sweepview.h"

using namespace fb360_dep;

extern int32_t FLAGS_width;
void rescaleCameras(Camera::Rig& rig);

// SystemUtil.cpp is not linked: the renamed main is never called
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

int derp_project_equirect_masks(int, const DerpCameraDesc* cams, int num_cams, double depth,
                                const uint8_t* const* eqr_masks, const int32_t* mask_sizes, uint8_t* const* out) {
  return guarded([&] {
    const Camera::Rig rig = rigOf(cams, num_cams);
    for (int i = 0; i < num_cams; ++i) {
      const Camera& cam = rig[i];
      cv::Mat_<bool> camMask(cam.resolution.y(), cam.resolution.x(), false);
      const int rows = mask_sizes[2 * i + 1], cols = mask_sizes[2 * i];
      for (int y = 0; y < camMask.rows; ++y) {
        for (int x = 0; x < camMask.cols; ++x) {
          const Camera::Vector3 world = cam.rig({x + 0.5, y + 0.5}, depth);
          const Camera::Vector2 pEqr = image_util::worldToEquirect(world, cols, rows);
          if (pEqr.x() < 0 || pEqr.y() < 0 || pEqr.x() >= cols || pEqr.y() >= rows) {
            continue;
          }
          if (std::isnan(pEqr.x()) || std::isnan(pEqr.y())) {
            continue;  // the deviation: see the header
          }
          if (eqr_masks[i][(size_t)int(pEqr.y()) * cols + int(pEqr.x())]) {
            camMask(y, x) = true;
          }
        }
      }
      for (int k = 0; k < camMask.rows * camMask.cols; ++k) out[i][k] = camMask.data[k] ? 255 : 0;
    }
    return DERP_OK;
  });
}

// rescaleCameras at --width: out[i] receives camera i's resolution, principal and focal after it
int ref_eqrproject_rescale(const DerpCameraDesc* cams, int num_cams, int width, DerpCameraDesc* out) {
  return guarded([&] {
    Camera::Rig rig = rigOf(cams, num_cams);
    FLAGS_width = width;
    rescaleCameras(rig);
    for (int i = 0; i < num_cams; ++i) {
      out[i] = cams[i];
      for (int k = 0; k < 2; ++k) {
        out[i].resolution[k] = rig[i].resolution[k];
        out[i].principal[k] = rig[i].principal[k];
        out[i].focal[k] = rig[i].focal[k];
      }
      out[i].has_principal = 1;
    }
    return DERP_OK;
  });
}

}  // extern "C"
