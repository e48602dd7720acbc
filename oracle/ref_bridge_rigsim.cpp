// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// Bridge of the RigSimulator checker (rigsim.mk): the reference's OWN source/rig/RigSimulator.cpp, compiled where it
// lies (main renamed), linked with the reference's Camera.o.  Nothing here restates the simulator; every
// export calls the app's own functions with its FLAGS_ set from the arguments:
//   ref_rigsim_build          srand(seed), then main's scene, selfIdx binding and makeBVH(triangles, 20, 5, 0, 50)
//   ref_rigsim_triangles      the scene's Triangles: v0, v1, v2, e1, e2, normal, color (21 floats each)
//   ref_rigsim_bvh            the BVH flattened in preorder: per node its sphere (cx, cy, cz, r) and {first, count,
//                             escape} (count = 0 for inner nodes, escape = the preorder index after its subtree), and
//                             the selfIdx of the leaf triangles in preorder
//   ref_rigsim_rand           the next rand() value (the stream position after the scene and the BVH)
//   ref_rigsim_trace          traceRayToGetColor on given fp32 rays: B, G, R, depth
//   ref_rigsim_render_camera  renderCamera (downscale and corruptImageWithNoise included), continuing the rand() stream
//                             where the build left it, as the app does
//   ref_rigsim_render_mono / ref_rigsim_render_stereo   renderMonoEquirect / renderStereoEquirect
//   ref_rigsim_area           the app's downscale (cv::resize INTER_AREA by an integer factor) of a float image
//   ref_rigsim_set_ceiling    --ceiling_path / _position / _width / _depth; the image is the caller's 8-bit BGR
//   ref_rigsim_save_rig       main's rig of a camera --mode (ringOfClones, makeHorizontalRingOf*, addTopCamera,
//                             make{Dodeca,Icosa}hedronOfFThetaCameras) written by Camera::saveRig(path, rig, {}, digits)
//                             (10 as the app's --rig_out; 0: folly's shortest round-trip doubles)
// The skybox is the caller's 8-bit BGR image.  This bridge is the checker's image decoder: cv_util::imreadExceptionOnFail
// (CvUtil.cpp, not linked here) returns the ceiling image the caller registered, which traceRayToGetColor loads once
// per process into its function-local static, so one process sees one ceiling image.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include <opencv2/opencv.hpp>

// RaytracingPrimitives.h defines its two intersection functions out of line; the app's object holds them, so this
// translation unit's copies get other names (it only needs the types)
#define rayIntersectTriangle bridge_unused_rayIntersectTriangle
#define rayIntersectSphereYesNo bridge_unused_rayIntersectSphereYesNo
#include "source/render/BoundingVolumeHierarchy.h"
#include "source/render/RaytracingPrimitives.h"
#undef rayIntersectTriangle
#undef rayIntersectSphereYesNo
#include "source/util/Camera.h"
#include "source/util/CvUtil.h"

#include "../include/derp_b200.h"

using namespace fb360_dep;
using namespace fb360_dep::render;

extern int32_t FLAGS_anti_alias_supersample;
extern double FLAGS_ground_plane_dist_m;
extern double FLAGS_interpupillary_radius;
extern bool FLAGS_marble;
extern double FLAGS_marble_scale;
extern double FLAGS_max_icosahedron_dist;
extern double FLAGS_max_icosahedron_radius;
extern double FLAGS_min_icosahedron_dist;
extern double FLAGS_min_icosahedron_radius;
extern double FLAGS_noise_amplitude;
extern int32_t FLAGS_num_random_icosahedrons;
extern bool FLAGS_red_triangle;
extern std::string FLAGS_ceiling_path;
extern double FLAGS_ceiling_position, FLAGS_ceiling_width, FLAGS_ceiling_depth;
extern int32_t FLAGS_num_cams_in_ring, FLAGS_ftheta_width, FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius;
extern int32_t FLAGS_pinhole_width, FLAGS_pinhole_height;
extern double FLAGS_rig_radius, FLAGS_ftheta_image_circle_fov, FLAGS_pinhole_fov_horizontal, FLAGS_pinhole_aspect_ratio;
extern double FLAGS_top_cam_vertical_offset;

void makeIcosahedronScene(std::vector<Triangle>& triangles);
void makeCubesScene(std::vector<Triangle>& triangles);
void makeGroundPlaneScene(std::vector<Triangle>& triangles);
cv::Vec4f traceRayToGetColor(const Ray& ray, const std::vector<Triangle>& triangles, const BoundingVolumeHierarchy& bvh,
                             const cv::Mat_<cv::Vec3b>& skybox);
std::pair<cv::Mat_<cv::Vec3f>, cv::Mat_<float>> renderMonoEquirect(const std::vector<Triangle>& triangles,
                                                                   const BoundingVolumeHierarchy& bvh, const int w,
                                                                   const int h, const cv::Mat_<cv::Vec3b>& skybox);
std::pair<cv::Mat_<cv::Vec3f>, cv::Mat_<cv::Vec3f>> renderStereoEquirect(const std::vector<Triangle>& triangles,
                                                                         const BoundingVolumeHierarchy& bvh,
                                                                         const int w, const int h,
                                                                         const cv::Mat_<cv::Vec3b>& skybox);
void renderCamera(const Camera& cam, const std::vector<Triangle>& triangles, const BoundingVolumeHierarchy& bvh,
                  const cv::Mat_<cv::Vec3b>& skybox, cv::Mat_<cv::Vec3f>& destImage, cv::Mat_<float>& destDepthMap);

std::vector<Camera> makeHorizontalRingOfPinholeCameras(const int numCameras, const float cameraArrayRadius,
                                                       const int pixelWidth, const int pixelHeight,
                                                       const float fovHorizontalDegrees, const float aspectRatioWoverH);
std::vector<Camera> makeHorizontalRingOfFThetaCameras(const int numCameras, const float cameraArrayRadius,
                                                      const int pixelWidth, const int pixelHeight,
                                                      const int imageCircleRadius, const float circleFov);
void addTopCamera(Camera::Rig& rig, const int pixelWidth, const int pixelHeight, const int imageCircleRadius,
                  const float circleFov);
std::vector<Camera> makeDodecahedronOfFThetaCameras(const float cameraSphereRadius, const int pixelWidth,
                                                    const int pixelHeight, const int imageCircleRadius,
                                                    const float circleFov);
std::vector<Camera> makeIcosahedronOfFThetaCameras(const float cameraSphereRadius, const int pixelWidth,
                                                   const int pixelHeight, const int imageCircleRadius,
                                                   const float circleFov);

namespace {
cv::Mat g_ceiling;
}  // namespace

// CvUtil.cpp is not linked: the ceiling is the one image the app reads after main; the writers are only reached from
// main and renderCamerasThreaded, which the bridge never calls
namespace fb360_dep::cv_util {
cv::Mat imreadExceptionOnFail(const filesystem::path&, const int) {
  if (g_ceiling.empty()) std::abort();
  return g_ceiling;
}
void imwriteExceptionOnFail(const filesystem::path&, const cv::Mat&, const std::vector<int>&) { std::abort(); }
void writeCvMat32FC1ToPFM(const filesystem::path&, const cv::Mat_<float>&) { std::abort(); }
}  // namespace fb360_dep::cv_util

// SystemUtil.cpp is not linked: the renamed main is never called
namespace fb360_dep::system_util {
void initDep(int&, char**&, const std::string) { std::abort(); }
}  // namespace fb360_dep::system_util

namespace {
std::vector<Triangle> g_tris;
BoundingVolumeHierarchy g_bvh;
cv::Mat_<cv::Vec3b> g_sky;

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
// One camera through the reference's JSON loader (%.17g round trip)
Camera cameraOf(const DerpCameraDesc& d) {
  static const char* kTypes[] = {"FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"};
  std::string json = std::string("{\"cameras\":[{\"version\":1,\"type\":\"") + kTypes[d.type] +
                     "\",\"id\":\"0\",\"origin\":" + vecJson(d.origin, 3) + ",\"forward\":" + vecJson(d.forward, 3) +
                     ",\"up\":" + vecJson(d.up, 3) + ",\"right\":" + vecJson(d.right, 3) +
                     ",\"resolution\":" + vecJson(d.resolution, 2) + ",\"focal\":" + vecJson(d.focal, 2);
  if (d.has_principal) json += ",\"principal\":" + vecJson(d.principal, 2);
  json += ",\"distortion\":" + vecJson(d.distortion, 3);
  if (d.has_fov) json += ",\"fov\":" + num17(d.fov);
  return Camera::loadRigFromJsonString(json + "}]}")[0];
}

void put3(float* o, const cv::Vec3f& v) {
  o[0] = v[0];
  o[1] = v[1];
  o[2] = v[2];
}

void flatten(const BoundingVolumeHierarchy& b, std::vector<float>& spheres, std::vector<int>& nodes,
             std::vector<int>& leafTris) {
  const size_t me = nodes.size() / 3;
  spheres.insert(spheres.end(), {b.sphere.center[0], b.sphere.center[1], b.sphere.center[2], b.sphere.radius});
  nodes.insert(nodes.end(), {(int)leafTris.size(), b.isLeaf ? (int)b.leafTriangles.size() : 0, -1});
  if (b.isLeaf)
    for (const Triangle& t : b.leafTriangles) leafTris.push_back(t.selfIdx);
  else
    for (const BoundingVolumeHierarchy& c : b.children) flatten(c, spheres, nodes, leafTris);
  nodes[3 * me + 2] = (int)(nodes.size() / 3);
}
}  // namespace

extern "C" {

int ref_rigsim_build(const char* scene, int num_icosahedrons, double min_dist, double max_dist, double min_radius,
                     double max_radius, int red_triangle, double ground_plane_dist, unsigned seed) {
  FLAGS_num_random_icosahedrons = num_icosahedrons;
  FLAGS_min_icosahedron_dist = min_dist;
  FLAGS_max_icosahedron_dist = max_dist;
  FLAGS_min_icosahedron_radius = min_radius;
  FLAGS_max_icosahedron_radius = max_radius;
  FLAGS_red_triangle = red_triangle != 0;
  FLAGS_ground_plane_dist_m = ground_plane_dist;
  srand(seed);
  g_tris.clear();
  const std::string s(scene);
  if (s == "icosahedron") {
    makeIcosahedronScene(g_tris);
  } else if (s == "cube") {
    makeCubesScene(g_tris);
  } else if (s == "ground_plane") {
    makeGroundPlaneScene(g_tris);
  } else {
    return -1;
  }
  for (int i = 0; i < int(g_tris.size()); ++i) g_tris[i].selfIdx = i;  // RigSimulator.cpp:682-684
  g_bvh = BoundingVolumeHierarchy::makeBVH(g_tris, 20, 5, 0, 50);       // RigSimulator.cpp:688-696
  return (int)g_tris.size();
}

void ref_rigsim_triangles(float* out) {
  for (const Triangle& t : g_tris) {
    for (const cv::Vec3f* v : {&t.v0, &t.v1, &t.v2, &t.e1, &t.e2, &t.normal, &t.color}) put3(out, *v), out += 3;
  }
}

// Sizes first (spheres == NULL), then the arrays
void ref_rigsim_bvh(int* num_nodes, int* num_leaf_tris, float* spheres, int* nodes, int* leaf_tris) {
  std::vector<float> s;
  std::vector<int> n, l;
  flatten(g_bvh, s, n, l);
  *num_nodes = (int)(n.size() / 3);
  *num_leaf_tris = (int)l.size();
  if (!spheres) return;
  std::memcpy(spheres, s.data(), s.size() * sizeof(float));
  std::memcpy(nodes, n.data(), n.size() * sizeof(int));
  std::memcpy(leaf_tris, l.data(), l.size() * sizeof(int));
}

int ref_rigsim_rand(void) { return rand(); }

void ref_rigsim_set_render(int aas, int marble, double marble_scale, double noise_amplitude,
                           double interpupillary_radius) {
  FLAGS_anti_alias_supersample = aas;
  FLAGS_marble = marble != 0;
  FLAGS_marble_scale = marble_scale;
  FLAGS_noise_amplitude = noise_amplitude;
  FLAGS_interpupillary_radius = interpupillary_radius;
}

void ref_rigsim_set_skybox(const uint8_t* bgr, int w, int h) {
  g_sky = cv::Mat_<cv::Vec3b>(h, w);
  std::memcpy(g_sky.data, bgr, (size_t)w * h * 3);
}

// rays: n x {ox, oy, oz, dx, dy, dz}; out: n x {B, G, R, depth}
void ref_rigsim_trace(const float* rays, int n, float* out) {
  for (int i = 0; i < n; ++i) {
    const float* r = rays + 6 * i;
    const cv::Vec4f c = traceRayToGetColor(Ray(cv::Vec3f(r[0], r[1], r[2]), cv::Vec3f(r[3], r[4], r[5])), g_tris, g_bvh,
                                           g_sky);
    for (int k = 0; k < 4; ++k) out[4 * i + k] = c[k];
  }
}

// image: [res.y][res.x][3] (255 * BGR), depth: [res.y][res.x]
int ref_rigsim_render_camera(const DerpCameraDesc* cam, float* image, float* depth) {
  try {
    const Camera c = cameraOf(*cam);
    cv::Mat_<cv::Vec3f> img;
    cv::Mat_<float> dep;
    renderCamera(c, g_tris, g_bvh, g_sky, img, dep);
    std::memcpy(image, img.data, img.total() * sizeof(cv::Vec3f));
    std::memcpy(depth, dep.data, dep.total() * sizeof(float));
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ref_rigsim_render_camera: %s\n", e.what());
    return -1;
  }
}

void ref_rigsim_render_mono(int w, int h, float* image, float* inv_depth) {
  const auto r = renderMonoEquirect(g_tris, g_bvh, w, h, g_sky);
  std::memcpy(image, r.first.data, r.first.total() * sizeof(cv::Vec3f));
  std::memcpy(inv_depth, r.second.data, r.second.total() * sizeof(float));
}

void ref_rigsim_render_stereo(int w, int h, float* left, float* right) {
  const auto r = renderStereoEquirect(g_tris, g_bvh, w, h, g_sky);
  std::memcpy(left, r.first.data, r.first.total() * sizeof(cv::Vec3f));
  std::memcpy(right, r.second.data, r.second.total() * sizeof(cv::Vec3f));
}

void ref_rigsim_set_ceiling(const uint8_t* bgr, int w, int h, double position, double width, double depth) {
  if (g_ceiling.empty()) {
    g_ceiling = cv::Mat_<cv::Vec3b>(h, w);
    std::memcpy(g_ceiling.data, bgr, (size_t)w * h * 3);
  }
  FLAGS_ceiling_path = "ceiling.png";
  FLAGS_ceiling_position = position;
  FLAGS_ceiling_width = width;
  FLAGS_ceiling_depth = depth;
}

void ref_rigsim_clear_ceiling(void) { FLAGS_ceiling_path = ""; }

// mode: pinhole_ring, ftheta_ring, dodecahedron or icosahedron, with main's arguments (RigSimulator.cpp:724-771)
int ref_rigsim_save_rig(const char* mode, const char* path, int num_cams, double rig_radius, int ftheta_w, int ftheta_h,
                        int circle_radius, double circle_fov, int pinhole_w, int pinhole_h, double pinhole_fov,
                        double pinhole_aspect, double top_offset, int digits) {
  FLAGS_num_cams_in_ring = num_cams;
  FLAGS_rig_radius = rig_radius;
  FLAGS_ftheta_width = ftheta_w;
  FLAGS_ftheta_height = ftheta_h;
  FLAGS_ftheta_image_circle_radius = circle_radius;
  FLAGS_ftheta_image_circle_fov = circle_fov;
  FLAGS_pinhole_width = pinhole_w;
  FLAGS_pinhole_height = pinhole_h;
  FLAGS_pinhole_fov_horizontal = pinhole_fov;
  FLAGS_pinhole_aspect_ratio = pinhole_aspect;
  FLAGS_top_cam_vertical_offset = top_offset;
  const std::string m(mode);
  std::vector<Camera> cameras;
  if (m == "pinhole_ring") {
    cameras = makeHorizontalRingOfPinholeCameras(FLAGS_num_cams_in_ring, FLAGS_rig_radius, FLAGS_pinhole_width,
                                                 FLAGS_pinhole_height, FLAGS_pinhole_fov_horizontal,
                                                 FLAGS_pinhole_aspect_ratio);
  } else if (m == "ftheta_ring") {
    cameras = makeHorizontalRingOfFThetaCameras(FLAGS_num_cams_in_ring, FLAGS_rig_radius, FLAGS_ftheta_width,
                                                FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius,
                                                FLAGS_ftheta_image_circle_fov);
    addTopCamera(cameras, FLAGS_ftheta_width, FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius,
                 FLAGS_ftheta_image_circle_fov);
  } else if (m == "dodecahedron") {
    cameras = makeDodecahedronOfFThetaCameras(FLAGS_rig_radius, FLAGS_ftheta_width, FLAGS_ftheta_height,
                                              FLAGS_ftheta_image_circle_radius, FLAGS_ftheta_image_circle_fov);
  } else if (m == "icosahedron") {
    cameras = makeIcosahedronOfFThetaCameras(FLAGS_rig_radius, FLAGS_ftheta_width, FLAGS_ftheta_height,
                                             FLAGS_ftheta_image_circle_radius, FLAGS_ftheta_image_circle_fov);
  } else {
    return -1;
  }
  try {
    Camera::saveRig(path, cameras, {}, digits);
  } catch (const std::exception& e) {
    fprintf(stderr, "ref_rigsim_save_rig: %s\n", e.what());
    return -1;
  }
  return 0;
}

// src: [h][w][cn] floats (cn 1 or 3); dst: [h / k][w / k][cn]
void ref_rigsim_area(const float* src, int w, int h, int cn, int k, float* dst) {
  cv::Mat m(h, w, cn == 3 ? CV_32FC3 : CV_32FC1);
  std::memcpy(m.data, src, (size_t)w * h * cn * sizeof(float));
  cv::Mat out;
  cv::resize(m, out, cv::Size(w / k, h / k), 0, 0, cv::INTER_AREA);
  std::memcpy(dst, out.data, (size_t)(w / k) * (h / k) * cn * sizeof(float));
}

}  // extern "C"
