// RigSimulator — drop-in for source/rig/RigSimulator.cpp.  Renders the synthetic scene (random icosahedrons, two
// cubes or a ground plane under a skybox) as seen by a simulated rig or as mono / stereo equirects, with ground-truth
// depth.  The scene, its BVH and the renders run in libderp_b200.so (include/derp_rigsim.h); the rigs, the noise and
// the image files are built here.  See INTEGRATION.md for what differs from the reference.
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "../../../include/derp_rigsim.h"
#include "../derp_camera.cuh"
#include "io.h"
#include "rig_json.h"

const std::string kUsage = R"(
  - Render an artificial scene as seen by the specified rig.

  - Example:
    ./RigSimulator \
    --mode=pinhole_ring \
    --skybox_path=/path/to/skybox.png
)";

DEFINE_int32(
    anti_alias_supersample,
    1,
    "1 = no supersampling, 2 or higher = anti-alias supersampling");
DEFINE_double(ceiling_depth, 0, "depth of ceiling texture (m)");
DEFINE_string(ceiling_path, "", "path to image to use for ceiling");
DEFINE_double(ceiling_position, 0, "how far up the ceiling is (m)");
DEFINE_double(ceiling_width, 0, "width of ceiling texture (m)");
DEFINE_string(
    dest_cam_images,
    "",
    "path to directory to write camera images for multi-camera rigs");
DEFINE_string(dest_left, "", "path to left-eye image");
DEFINE_string(dest_mono, "", "path to mono image");
DEFINE_string(dest_mono_depth, "", "path to mono 1/depthmap (intensity = 1 / depth in meters)");
DEFINE_string(dest_right, "", "path to right-eye image");
DEFINE_string(dest_stereo, "", "path to right-eye image");
DEFINE_int32(eqr_height, 1540, "height of equirect output");
DEFINE_int32(eqr_width, 3080, "width of equirect output");
DEFINE_int32(ftheta_height, 400, "height of ftheta camera output");
DEFINE_double(
    ftheta_image_circle_fov,
    166.667,
    "ftheta FOV, i.e. number of degrees spanned at the image circle");
DEFINE_int32(
    ftheta_image_circle_radius,
    250,
    "image circle radius corresponding to specified ftheta FOV");
DEFINE_int32(ftheta_width, 300, "width of ftheta camera output");
DEFINE_double(
    ground_plane_dist_m,
    1.70,
    "for 'ground_plane' scene, distance from camera to ground");
DEFINE_double(interpupillary_radius, 3.2, "half distance between eyes");
DEFINE_bool(
    marble,
    false,
    "if true, adds a marble (perlin noise) texture to the objects in the scene");
DEFINE_double(marble_scale, 0.1, "scale applied to marble texture");
DEFINE_double(
    max_icosahedron_dist,
    250,
    "maximum distance from origin that a randomly generated icosahedron can spawn");
DEFINE_double(max_icosahedron_radius, 50, "max radius of a randomly generated icosahedron");
DEFINE_double(
    min_icosahedron_dist,
    100,
    "minimum distance from a center of camera to the closest point on a randomly generated icosahedron");
DEFINE_double(min_icosahedron_radius, 20, "min radius of a randomly generated icosahedron");
DEFINE_string(
    mode,
    "",
    "mono_eqr,stereo_eqr,pinhole_ring,ftheta_ring,dodecahedron,icosahedron,rig_from_json (required)");
DEFINE_double(
    noise_amplitude,
    0.0,
    "amount of noise to be added to pixels (to simulate real camera noise). pixel intensities are scaled in 0...255");
DEFINE_int32(num_cams_in_ring, 14, "number of cameras in simulated rings of cameras");
DEFINE_int32(num_random_icosahedrons, 250, "number of icosahedrons to generate");
DEFINE_double(
    pinhole_aspect_ratio,
    1.0,
    "aspect ratio of pinhole lens = horizontal fov / vertical fov");
DEFINE_double(pinhole_fov_horizontal, 77.7, "horizontal FOV of pinhole lens (degrees)");
DEFINE_int32(pinhole_height, 512, "height of pinhole camera output");
DEFINE_int32(pinhole_width, 512, "width of pinhole camera output");
DEFINE_bool(red_triangle, false, "add a red triangle at (0,0)");
DEFINE_string(rig_in, "", "path to read json rig file if mode = rig_from_json");
DEFINE_string(rig_out, "", "path to write json description of multi-camera rig");
DEFINE_double(
    rig_radius,
    0.218,
    "radius of the rig/sphere of cameras (m). distance from center to lens exit pupil.");
DEFINE_string(scene, "icosahedron", "scene to draw: 'icosahedron', 'cube', 'ground_plane'");
DEFINE_string(skybox_path, "res/skybox.jpg", "path to image to use as background/skybox");
DEFINE_double(top_cam_vertical_offset, 13.0, "distance from center plane to top camera");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                    \
  do {                                                                     \
    const int rc_ = (expr);                                                \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

namespace {

// ---- rigs (RigSimulator.cpp:360-491) --------------------------------------------------------------------------------
struct SimCamera {
  DerpCameraDesc d{};
  std::string id, group;
};

float toRadians(float deg) { return deg * static_cast<float>(M_PI) / 180.0f; }  // MathUtil.h:27-29

void cross(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// Camera(type, resolution, focal): principal = resolution / 2, default distortion and fov
SimCamera generic(int type, double w, double h, double fx, double fy) {
  SimCamera c;
  c.d.type = type;
  c.d.resolution[0] = w;
  c.d.resolution[1] = h;
  c.d.focal[0] = fx;
  c.d.focal[1] = fy;
  c.d.forward[2] = -1;  // rotation = identity: forward -z, up +y, right +x
  c.d.up[1] = 1;
  c.d.right[0] = 1;
  return c;
}

// Camera::setRotation(forward, up): right = forward x up; the re-unitarised rotation is what forward() returns
void setRotation(SimCamera& c, const double* fwd, const double* up) {
  for (int k = 0; k < 3; ++k) {
    c.d.forward[k] = fwd[k];
    c.d.up[k] = up[k];
  }
  cross(fwd, up, c.d.right);
}
void forwardOf(const SimCamera& c, double* f) {
  derp::DevCamera dc;
  CHECK(derp::host::makeCamera(c.d, &dc)) << "rotation is not close to unitary";
  for (int k = 0; k < 3; ++k) f[k] = -dc.rot[6 + k];
}

std::vector<SimCamera> ringOfClones(const SimCamera& camera, int count, double radius) {
  std::vector<SimCamera> result(count, camera);
  for (int i = 0; i < count; ++i) {
    const double theta = -2.0 * M_PI * double(i) / double(count);
    SimCamera& clone = result[i];
    const double fwd[3] = {cos(theta), sin(theta), 0}, up[3] = {0, 0, 1};
    setRotation(clone, fwd, up);
    double f[3];
    forwardOf(clone, f);
    for (int k = 0; k < 3; ++k) clone.d.origin[k] = radius * f[k];
    clone.id = std::to_string(i);
    clone.group = "side camera";
  }
  return result;
}

SimCamera genericFTheta(int w, int h, int imageCircleRadius, float circleFov) {
  const double f = 2 * imageCircleRadius / toRadians(circleFov);  // float, then Vector2(1, 1) in double
  return generic(DERP_CAM_FTHETA, w, h, f, f);
}

std::vector<SimCamera> pinholeRing(int n, float radius, int w, int h, float fovDeg, float aspect) {
  const float tanHalfFov = std::tan(toRadians(fovDeg) / 2);
  const SimCamera g = generic(DERP_CAM_RECTILINEAR, w, h, (w / 2.0) / tanHalfFov, (h / 2.0) / (tanHalfFov / aspect));
  return ringOfClones(g, n, radius);
}

std::vector<SimCamera> fthetaRing(int n, float radius, int w, int h, int circleRadius, float circleFov) {
  return ringOfClones(genericFTheta(w, h, circleRadius, circleFov), n, radius);
}

void addTopCamera(std::vector<SimCamera>& rig, int w, int h, int circleRadius, float circleFov) {
  SimCamera top = genericFTheta(w, h, circleRadius, circleFov);
  top.d.origin[2] = FLAGS_top_cam_vertical_offset;
  const double fwd[3] = {0, 0, 1}, up[3] = {1, 0, 0};
  setRotation(top, fwd, up);
  top.id = std::to_string(rig.size());
  rig.push_back(top);
}

// The unit icosahedron of the scene, as float (the same table as derp_rigsim.cuh), read as double
constexpr float kIcoX = 0.525731112119133696f, kIcoZ = 0.850650808352039932f;
const float kIcoVertex[12][3] = {
    {-kIcoX, 0, kIcoZ}, {kIcoX, 0, kIcoZ}, {-kIcoX, 0, -kIcoZ}, {kIcoX, 0, -kIcoZ}, {0, kIcoZ, kIcoX}, {0, kIcoZ, -kIcoX},
    {0, -kIcoZ, kIcoX}, {0, -kIcoZ, -kIcoX}, {kIcoZ, kIcoX, 0}, {-kIcoZ, kIcoX, 0}, {kIcoZ, -kIcoX, 0}, {-kIcoZ, -kIcoX, 0}};
const int kIcoFace[20][3] = {{1, 4, 0},  {4, 9, 0},  {4, 5, 9},  {8, 5, 4},  {1, 8, 4},  {1, 10, 8}, {10, 3, 8},
                             {8, 3, 5},  {3, 2, 5},  {3, 7, 2},  {3, 10, 7}, {10, 6, 7}, {6, 11, 7}, {6, 0, 11},
                             {6, 1, 0},  {10, 1, 6}, {11, 0, 9}, {2, 11, 9}, {5, 2, 9},  {11, 2, 7}};

void normalized(double* v) {  // Eigen's normalized(): v / sqrt(squaredNorm)
  const double n = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  for (int k = 0; k < 3; ++k) v[k] = v[k] / n;
}

// makeFThetaCameraOnSphere: position = imageCircleRadius * normal (the reference ignores the sphere radius)
SimCamera fthetaOnSphere(const double* normal, int w, int h, int circleRadius, float circleFov, const std::string& id) {
  SimCamera c = genericFTheta(w, h, circleRadius, circleFov);
  for (int k = 0; k < 3; ++k) c.d.origin[k] = circleRadius * normal[k];
  const double worldUp[3] = {0, 0, 1};
  double right[3], minusRight[3], up[3];
  cross(normal, worldUp, right);
  normalized(right);
  for (int k = 0; k < 3; ++k) minusRight[k] = -right[k];
  cross(normal, minusRight, up);
  setRotation(c, normal, up);
  c.id = id;
  return c;
}

std::vector<SimCamera> dodecahedron(int w, int h, int circleRadius, float circleFov) {
  std::vector<SimCamera> cams;
  for (int i = 0; i < 12; ++i) {
    const double n[3] = {kIcoVertex[i][0], kIcoVertex[i][1], kIcoVertex[i][2]};
    cams.push_back(fthetaOnSphere(n, w, h, circleRadius, circleFov, std::to_string(cams.size())));
  }
  return cams;
}

std::vector<SimCamera> icosahedron(int w, int h, int circleRadius, float circleFov) {
  std::vector<SimCamera> cams;
  for (const auto& f : kIcoFace) {
    double m[3];
    for (int k = 0; k < 3; ++k)
      m[k] = (double)kIcoVertex[f[0]][k] + (double)kIcoVertex[f[1]][k] + (double)kIcoVertex[f[2]][k];
    normalized(m);
    cams.push_back(fthetaOnSphere(m, w, h, circleRadius, circleFov, std::to_string(cams.size())));
  }
  return cams;
}

// ---- --rig_out: Camera::saveRig with sorted keys and doubleNumDigits = 10 (folly's FIXED mode) ------------------------
void saveRig(const std::string& path, const std::vector<SimCamera>& cams) {
  std::vector<rigjson::Camera> out(cams.size());
  for (size_t i = 0; i < cams.size(); ++i) {
    derp::DevCamera dc;
    CHECK(derp::host::makeCamera(cams[i].d, &dc)) << "invalid camera " << cams[i].id;
    out[i].d = cams[i].d;
    std::copy(dc.rot, dc.rot + 9, out[i].rot);
    out[i].id = cams[i].id;
    out[i].group = cams[i].group;
  }
  rigjson::saveRig(path, out, {}, false);
}

// ---- images -----------------------------------------------------------------------------------------------------------
bool isPng(const std::string& path) {
  const std::string ext = fs::path(path).extension().string();
  return ext == ".png" || ext == ".PNG";
}

// imread(path, IMREAD_COLOR) of a PNG: 8-bit B, G, R (io::readPng hands out B, G, R(, A) like OpenCV; grey replicated,
// alpha dropped, 16-bit samples' high byte)
std::vector<uint8_t> loadBgr8(const std::string& path, int* w, int* h) {
  CHECK(isPng(path)) << "unsupported image " << path << ": this build reads PNG only (no JPEG decoder)";
  CHECK(fs::exists(path)) << "failed to load image: " << path;
  const io::Image im = io::readPng(path);
  CHECK(im.bits == 8 || im.bits == 16) << "unsupported PNG " << path;
  *w = im.w;
  *h = im.h;
  std::vector<uint8_t> bgr((size_t)im.w * im.h * 3);
  const int cn = im.channels, shift = im.bits == 16 ? 8 : 0;
  for (size_t p = 0; p < (size_t)im.w * im.h; ++p) {
    const uint16_t* s = &im.u[p * cn];
    const int b = s[0] >> shift, g = s[cn >= 3 ? 1 : 0] >> shift, r = s[cn >= 3 ? 2 : 0] >> shift;
    bgr[3 * p] = (uint8_t)b;
    bgr[3 * p + 1] = (uint8_t)g;
    bgr[3 * p + 2] = (uint8_t)r;
  }
  return bgr;
}

// imwrite of a float Mat to PNG: convertTo(CV_8U) (saturate_cast: round half to even, clamp, NaN -> 0)
void writePng8(const std::string& path, const float* v, int w, int h, int channels) {
  CHECK(isPng(path)) << "unsupported output " << path << ": this build writes PNG only";
  std::vector<uint8_t> b((size_t)w * h * channels);
  for (size_t i = 0; i < b.size(); ++i) b[i] = io::saturateU8(v[i]);
  if (!fs::path(path).parent_path().empty()) fs::create_directories(fs::path(path).parent_path());
  io::writePng8(path, b.data(), w, h, channels);
}

inline float randf0to1() { return float(rand()) / float(RAND_MAX); }  // MathUtil.h:23-25

// corruptImageWithNoise (RigSimulator.cpp:494-508); the three draws of one pixel are made last channel first, the order
// g++ evaluates the arguments of the reference's cv::Vec3f(...)
void corruptImageWithNoise(std::vector<float>& image) {
  const float a = FLAGS_noise_amplitude;
  if (a == 0.0f) return;
  for (size_t p = 0; p < image.size() / 3; ++p) {
    float v[3];
    for (int c = 2; c >= 0; --c) {
      const float x = image[3 * p + c] + 2.0f * a * (randf0to1() - 0.5f);
      v[c] = x < 0 ? 0 : x > 255.0f ? 255.0f : x;  // math_util::clamp<float>
    }
    for (int c = 0; c < 3; ++c) image[3 * p + c] = v[c];
  }
}

}  // namespace

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);

  CHECK_NE(FLAGS_mode, "");
  CHECK_NE(FLAGS_skybox_path, "");
  CHECK_GE(FLAGS_anti_alias_supersample, 1) << "--anti_alias_supersample must be at least 1";

  // the outputs are PNG files (no other encoder is built): refused before any work
  for (const std::string* dest : {&FLAGS_dest_mono, &FLAGS_dest_mono_depth, &FLAGS_dest_left, &FLAGS_dest_right,
                                  &FLAGS_dest_stereo})
    CHECK(dest->empty() || isPng(*dest)) << "unsupported output " << *dest << ": this build writes PNG only";

  int skyW = 0, skyH = 0, ceilW = 0, ceilH = 0;
  const std::vector<uint8_t> skybox = loadBgr8(FLAGS_skybox_path, &skyW, &skyH);
  std::vector<uint8_t> ceiling;
  if (!FLAGS_ceiling_path.empty()) ceiling = loadBgr8(FLAGS_ceiling_path, &ceilW, &ceilH);

  DerpRigsimSceneParams sp{};
  if (FLAGS_scene == "icosahedron") {
    sp.scene = DERP_RIGSIM_ICOSAHEDRON;
  } else if (FLAGS_scene == "cube") {
    sp.scene = DERP_RIGSIM_CUBE;
  } else if (FLAGS_scene == "ground_plane") {
    sp.scene = DERP_RIGSIM_GROUND_PLANE;
  } else {
    CHECK(false) << "unexpected scene: " << FLAGS_scene;
  }
  sp.num_random_icosahedrons = FLAGS_num_random_icosahedrons;
  sp.red_triangle = FLAGS_red_triangle;
  sp.min_icosahedron_dist = FLAGS_min_icosahedron_dist;
  sp.max_icosahedron_dist = FLAGS_max_icosahedron_dist;
  sp.min_icosahedron_radius = FLAGS_min_icosahedron_radius;
  sp.max_icosahedron_radius = FLAGS_max_icosahedron_radius;
  sp.ground_plane_dist_m = FLAGS_ground_plane_dist_m;
  LOG(INFO) << "building BVH";
  DerpRigsimScene* scene = nullptr;
  DERP_CALL(derp_rigsim_scene_create(&sp, &scene));

  DerpRigsimRender ro{};
  ro.anti_alias_supersample = FLAGS_anti_alias_supersample;
  ro.marble = FLAGS_marble;
  ro.marble_scale = FLAGS_marble_scale;
  ro.interpupillary_radius = FLAGS_interpupillary_radius;
  ro.skybox_bgr = skybox.data();
  ro.skybox_width = skyW;
  ro.skybox_height = skyH;
  ro.ceiling_bgr = ceiling.empty() ? nullptr : ceiling.data();
  ro.ceiling_cols = ceilW;
  ro.ceiling_rows = ceilH;
  ro.ceiling_position = FLAGS_ceiling_position;
  ro.ceiling_width = FLAGS_ceiling_width;
  ro.ceiling_depth = FLAGS_ceiling_depth;

  const int W = FLAGS_eqr_width, H = FLAGS_eqr_height;
  if (FLAGS_mode == "mono_eqr") {
    CHECK_NE(FLAGS_dest_mono, "");
    CHECK_NE(FLAGS_dest_mono_depth, "");
    std::vector<float> image((size_t)W * H * 3), invDepth((size_t)W * H);
    DERP_CALL(derp_rigsim_render_equirect(FLAGS_gpu, scene, &ro, 0, W, H, image.data(), invDepth.data()));
    writePng8(FLAGS_dest_mono, image.data(), W, H, 3);
    for (float& v : invDepth) v = v * 255.0f;  // monoEquirectInvDepth * 255.0: convertTo with (float)255
    writePng8(FLAGS_dest_mono_depth, invDepth.data(), W, H, 1);
  } else if (FLAGS_mode == "stereo_eqr") {
    CHECK_NE(FLAGS_dest_left, "");
    CHECK_NE(FLAGS_dest_right, "");
    CHECK_NE(FLAGS_dest_stereo, "");
    std::vector<float> stereo((size_t)W * H * 3 * 2);  // vconcat(left, right)
    float* left = stereo.data();
    float* right = stereo.data() + (size_t)W * H * 3;
    DERP_CALL(derp_rigsim_render_equirect(FLAGS_gpu, scene, &ro, 1, W, H, left, right));
    writePng8(FLAGS_dest_left, left, W, H, 3);
    writePng8(FLAGS_dest_right, right, W, H, 3);
    writePng8(FLAGS_dest_stereo, stereo.data(), W, 2 * H, 3);
  } else {
    std::vector<SimCamera> cams;
    if (FLAGS_mode == "pinhole_ring") {
      cams = pinholeRing(FLAGS_num_cams_in_ring, FLAGS_rig_radius, FLAGS_pinhole_width, FLAGS_pinhole_height,
                         FLAGS_pinhole_fov_horizontal, FLAGS_pinhole_aspect_ratio);
    } else if (FLAGS_mode == "ftheta_ring") {
      cams = fthetaRing(FLAGS_num_cams_in_ring, FLAGS_rig_radius, FLAGS_ftheta_width, FLAGS_ftheta_height,
                        FLAGS_ftheta_image_circle_radius, FLAGS_ftheta_image_circle_fov);
      addTopCamera(cams, FLAGS_ftheta_width, FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius,
                   FLAGS_ftheta_image_circle_fov);
    } else if (FLAGS_mode == "dodecahedron") {
      cams = dodecahedron(FLAGS_ftheta_width, FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius,
                          FLAGS_ftheta_image_circle_fov);
    } else if (FLAGS_mode == "icosahedron") {
      cams = icosahedron(FLAGS_ftheta_width, FLAGS_ftheta_height, FLAGS_ftheta_image_circle_radius,
                         FLAGS_ftheta_image_circle_fov);
    } else if (FLAGS_mode == "rig_from_json") {
      CHECK_NE(FLAGS_rig_in, "");
      const io::Rig rig = io::loadRig(FLAGS_rig_in);
      for (size_t i = 0; i < rig.cams.size(); ++i) {
        SimCamera c;
        c.d = rig.cams[i];
        c.id = rig.ids[i];
        cams.push_back(c);
      }
    } else {
      CHECK(false) << "unexpected mode: " << FLAGS_mode;
    }
    if (!FLAGS_rig_out.empty()) saveRig(FLAGS_rig_out, cams);
    if (!FLAGS_dest_cam_images.empty()) {
      const int n = (int)cams.size();
      std::vector<DerpCameraDesc> descs(n);
      std::vector<std::vector<float>> images(n), depths(n);
      std::vector<float*> ip(n), dp(n);
      for (int i = 0; i < n; ++i) {
        LOG(INFO) << "------ rendering camera " << i;
        descs[i] = cams[i].d;
        const size_t px = (size_t)(int)descs[i].resolution[0] * (int)descs[i].resolution[1];
        images[i].resize(3 * px);
        depths[i].resize(px);
        ip[i] = images[i].data();
        dp[i] = depths[i].data();
      }
      DERP_CALL(derp_rigsim_render_cameras(FLAGS_gpu, scene, &ro, descs.data(), n, ip.data(), dp.data()));
      fs::create_directories(FLAGS_dest_cam_images);
      for (int i = 0; i < n; ++i) {
        corruptImageWithNoise(images[i]);
        const int w = (int)descs[i].resolution[0], h = (int)descs[i].resolution[1];
        const std::string stem = FLAGS_dest_cam_images + "/" + cams[i].id;
        writePng8(stem + ".png", images[i].data(), w, h, 3);
        writePng8(stem + "_depth.png", depths[i].data(), w, h, 1);
        io::writePfm(stem + "_depth.pfm", depths[i].data(), w, h);
      }
    }
  }
  derp_rigsim_scene_destroy(scene);
  return EXIT_SUCCESS;
}
