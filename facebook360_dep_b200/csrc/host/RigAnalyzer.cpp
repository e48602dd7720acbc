// RigAnalyzer — drop-in for source/rig/RigAnalyzer.cpp.  Builds or edits a rig, prints how many cameras see each
// direction at 20 distances, and writes the rig's overlap maps (equirect, one camera's pixels, a cross-section) as PPM
// text, the rig as an OBJ and as rig JSON.  The coverage counts run in libderp_b200.so (include/derp_riganalysis.h);
// the rig edits, the report and the files are made here.  See INTEGRATION.md for what differs from the reference.
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iomanip>
#include <sstream>

#include "../../../include/derp_riganalysis.h"
#include "../derp_camera.cuh"
#include "io.h"
#include "rig_json.h"

const std::string kUsage = R"(
   - Miscellaneous analysis utilities for a rig. Various output formats are supported to
   visualize the rig setup (e.g. equirect projection).

   - Example:
     ./RigAnalyzer \
     --rig=/path/to/rigs/rig.json \
     --output_equirect=/path/to/output/equirect.png
 )";

struct Camera {  // Camera::kNearInfinity (Camera.cpp), the default of --overlap_distance
  static constexpr double kNearInfinity = 1.0e4;
};

DEFINE_double(custom, -1, "custom angle away from north");
DEFINE_double(discard_poles, 0, "degrees from poles to ignore");
DEFINE_string(eulers, "", "create from eulers file");
DEFINE_double(min_distance, 0.50, "min distance to test");
DEFINE_double(
    overlap_distance,
    Camera::kNearInfinity,
    "distance to visualize equirect overlap, default is INF");
DEFINE_bool(one_based_indexing, false, "enable to index cameras starting at 1 instead of 0");
DEFINE_string(output_camera, "", "path to output camera .ppm file");
DEFINE_string(output_camera_id, "", "output camera id");
DEFINE_string(output_cross_section, "", "path to output cross section .ppm file");
DEFINE_string(output_equirect, "", "path to output equirect .ppm file");
DEFINE_string(output_obj, "", "path to output rig .obj file");
DEFINE_string(output_rig, "", "path to output rig .json file");
DEFINE_bool(perturb_cameras, false, "");
DEFINE_double(perturb_focals, 0, "pertub focals");
DEFINE_double(perturb_positions, 0, "perturb positions (cm)");
DEFINE_double(perturb_principals, 0, "pertub principals (pixels)");
DEFINE_double(perturb_rotations, 0, "perturb rotations (radians)");
DEFINE_int32(perturb_seed, 1, "seed for perturb cameras. Default: 1, same as no seed");
DEFINE_double(radius, 0, "change rig radius");
DEFINE_string(
    rearrange,
    "",
    "create specific arrangement (ballcam24, tetra, ring4, cube, carbon0, carbon1, diamond)");
DEFINE_string(revolve, "", "create from angle file");
DEFINE_string(rig, "", "path to rig .json file (required)");
DEFINE_string(rotate, "", "rotate rig by euler angles");
DEFINE_string(rotate_cam_z, "", "rotate camera to align with z");
DEFINE_int32(sample_count, 100000, "number of samples");
DEFINE_double(scale_resolution, 1, "scale camera resolutions");
DEFINE_bool(show_timing, false, "visualize time as well as spatial overlap");
DEFINE_bool(z_is_down, false, "modify rig from y-is-up to z-is-down");
DEFINE_bool(z_is_up, false, "modify rig from y-is-up to z-is-up");
DEFINE_double(scale_rig, 1, "scale rig space, e.g., by 1e-2 to convert from cm to m");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                    \
  do {                                                                     \
    const int rc_ = (expr);                                                \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

namespace {

using Cam = rigjson::Camera;
using Rig = std::vector<Cam>;
using derp::host::Quat;

// ---- Eigen's geometry, in the operation order of the reference's Eigen calls ---------------------------------------
struct V3 {
  double v[3];
};
V3 mul(const double* m, const V3& x) {  // Matrix3 * Vector3
  V3 r;
  derp::host::mulMV(m, x.v, r.v);
  return r;
}
double norm(const V3& a) { return std::sqrt(a.v[0] * a.v[0] + a.v[1] * a.v[1] + a.v[2] * a.v[2]); }
V3 scaled(const V3& a, double s) { return V3{{a.v[0] * s, a.v[1] * s, a.v[2] * s}}; }
V3 forward(const Cam& c) { return V3{{-c.rot[6], -c.rot[7], -c.rot[8]}}; }
V3 up(const Cam& c) { return V3{{c.rot[3], c.rot[4], c.rot[5]}}; }
V3 right(const Cam& c) { return V3{{c.rot[0], c.rot[1], c.rot[2]}}; }
V3 position(const Cam& c) { return V3{{c.d.origin[0], c.d.origin[1], c.d.origin[2]}}; }
void setPosition(Cam& c, const V3& p) {
  for (int k = 0; k < 3; ++k) c.d.origin[k] = p.v[k];
}

// Camera::setRotation(forward, up, right): right-handed and unitary within 0.001, then re-unitarised
void setRotation(Cam& c, const V3& f, const V3& u, const V3& r) {
  for (int k = 0; k < 3; ++k) {
    c.d.forward[k] = f.v[k];
    c.d.up[k] = u.v[k];
    c.d.right[k] = r.v[k];
  }
  CHECK(derp::host::reunitarise(f.v, u.v, r.v, c.rot)) << "rotation must be right-handed and close to unitary";
}
// Camera::getRotation (Camera.cpp:103-112)
V3 getRotation(const Cam& c) {
  double angle, axis[3];
  derp::host::angleAxisOf(c.rot, &angle, axis);
  if (angle > M_PI) {
    angle = 2 * M_PI - angle;
    for (double& a : axis) a = -a;
  }
  return V3{{angle * axis[0], angle * axis[1], angle * axis[2]}};
}
// Camera::setRotation(angleAxis) (Camera.cpp:93-101): no re-unitarisation
void setRotationAngleAxis(Cam& c, const V3& aa) {
  const double angle = norm(aa);
  V3 axis{{aa.v[0] / angle, aa.v[1] / angle, aa.v[2] / angle}};
  if (angle == 0) axis = V3{{1, 0, 0}};
  derp::host::rotationOf(angle, axis.v, c.rot);
  for (int k = 0; k < 3; ++k) {  // the desc's vectors follow the rotation (the library takes c.rot as is)
    c.d.right[k] = c.rot[k];
    c.d.up[k] = c.rot[3 + k];
    c.d.forward[k] = -c.rot[6 + k];
  }
}

// (xyz ? z * y * x : y * x * z).toRotationMatrix() of AngleAxis about the unit axes
void rotationMatrixFromEulers(const V3& e, bool xyz, double* R) {
  using derp::host::quatMul;
  using derp::host::quatOf;
  const Quat x = quatOf(e.v[0], 0), y = quatOf(e.v[1], 1), z = quatOf(e.v[2], 2);
  derp::host::quatToRotation(xyz ? quatMul(quatMul(z, y), x) : quatMul(quatMul(y, x), z), R);
}

// ---- rig builders (RigAnalyzer.cpp:96-259) --------------------------------------------------------------------------
Rig makeRigFromEulers(const Cam& model, const std::vector<V3>& eulers, bool xyz) {
  Rig result;
  for (V3 euler : eulers) {
    euler = scaled(euler, M_PI / 180);
    double m[9];
    rotationMatrixFromEulers(euler, xyz, m);
    Cam camera = model;
    setRotation(camera, V3{{m[2], m[5], m[8]}}, V3{{m[1], m[4], m[7]}}, V3{{-m[0], -m[3], -m[6]}});
    const V3 f = forward(camera);
    setPosition(camera, scaled(f, norm(position(model))));
    camera.id = "cam" + std::to_string(result.size() + (FLAGS_one_based_indexing ? 1 : 0));
    result.push_back(camera);
  }
  return result;
}

Rig revolveRig(const Rig& rig, const std::vector<V3>& eulers) {
  Rig result;
  for (int frame = 0; frame < int(eulers.size()); ++frame) {
    double xform[9];
    rotationMatrixFromEulers(eulers[frame], true, xform);
    for (Cam camera : rig) {
      setRotation(camera, mul(xform, forward(camera)), mul(xform, up(camera)), mul(xform, right(camera)));
      setPosition(camera, mul(xform, position(camera)));
      if (eulers.size() > 1) camera.id += '_' + std::to_string(frame);
      result.push_back(camera);
    }
  }
  return result;
}

Rig makeNamedArrangement(const std::string& name, const Cam& model, double custom) {
  auto eulers = [&](std::initializer_list<V3> e, bool xyz) { return makeRigFromEulers(model, e, xyz); };
  if (name == "ballcam24") {
    return eulers({{{22.998, -36.1543, 132.267}},    {{-2.89381, -156.601, 168.482}},
                   {{-50.2907, -68.7384, 139.028}},  {{-80.2662, 172.721, 113.889}},
                   {{57.5173, 87.6811, 161.596}},    {{6.46204, 162.32, 70.7419}},
                   {{21.8577, 118.439, 114.195}},    {{77.4316, -95.0674, -100.379}},
                   {{-20.2739, 41.1554, -135.466}},  {{-38.2009, 172.776, -171.825}},
                   {{-0.841465, -110.909, 57.8619}}, {{-39.8563, -128.178, 46.3619}},
                   {{-54.3882, 8.6561, -13.3586}},   {{24.3104, 51.5133, -20.0308}},
                   {{35.7198, -82.6713, 160.228}},   {{-48.4447, 85.1941, 93.5637}},
                   {{48.4425, 165.464, 19.7297}},    {{-3.41527, 84.0526, 56.5226}},
                   {{-20.5666, -24.4286, 14.2745}},  {{35.8214, -139.006, -27.4138}},
                   {{-8.22831, -69.3313, -46.6214}}, {{51.5282, 4.18718, -133.303}},
                   {{6.61383, 8.24745, -72.7674}},   {{-22.4038, 126.995, 13.7087}}},
                  false);
  } else if (name == "tetra") {
    const double a = custom == -1 ? acos(-1 / 3.0) * 180 / M_PI : custom;
    return eulers({{{a, 0, 0}}, {{a, 0, 120}}, {{a, 0, -120}}, {{0, 0, 0}}}, true);
  } else if (name == "tetratilted") {
    return eulers({{{-35.2644, 45, -65.1818}}, {{-35.2644, -135, -137.834}}, {{35.2644, -45, -45.0048}},
                   {{35.2644, 135, -104.664}}},
                  false);
  } else if (name == "ring4") {
    const double a = custom == -1 ? 90 : custom;
    return eulers({{{a, 0, 0}}, {{a, 0, 90}}, {{a, 0, 180}}, {{a, 0, 270}}}, true);
  } else if (name == "cube") {
    const double a = custom == -1 ? 90 : custom;
    return eulers({{{a, 0, 0}}, {{a, 0, 90}}, {{a, 0, 180}}, {{a, 0, 270}}, {{0, 0, 0}}, {{180, 0, 0}}}, true);
  } else if (name == "carbon0") {
    return eulers({{{-35.2644, 3.89537e-15, 112.232}}, {{-35.2644, 120, -67.3096}}, {{-35.2644, -120, 155.867}},
                   {{35.2644, 180, 21.9328}}, {{35.2644, -60, 14.0236}}, {{35.2644, 60, 66.2737}}},
                  false);
  } else if (name == "carbon1") {
    return eulers({{{-35.2644, 1.94768e-15, 133.504}}, {{-35.2644, 120, -179.989}}, {{-35.2644, -120, -134.51}},
                   {{35.2644, 180, 89.7419}}, {{35.2644, -60, 43.7899}}, {{35.2644, 60, -45.1612}}},
                  false);
  }
  CHECK_EQ(name, "diamond") << "unknown arrangement";
  const double a = custom == -1 ? 90 : custom;
  return eulers({{{a, 0, 0}}, {{a, 0, 120}}, {{a, 0, 240}}, {{0, 0, 0}}, {{180, 0, 0}}}, true);
}

std::vector<V3> readVectorFile(const std::string& filename) {
  std::vector<V3> result;
  std::ifstream file(filename);
  for (std::string line; getline(file, line);) {
    if (line.find("===") == 0) continue;  // ignore lines beginning with '==='
    std::istringstream s(line);
    V3 angles;
    s >> angles.v[0] >> angles.v[1] >> angles.v[2];
    CHECK(s) << "bad line <" << line << "> in file " << filename;
    result.push_back(angles);
  }
  return result;
}

// Camera::perturbCameras (Camera.cpp:260-280) after std::srand(seed): position, angle-axis, principal, focal
double randOffset(double amount) { return amount * 2 * (std::rand() / double(RAND_MAX) - 0.5); }
void perturbCameras(Rig& rig, double pos, double rot, double principal, double focal) {
  for (size_t i = 0; i < rig.size(); ++i) {
    Cam& camera = rig[i];
    if (i != 0) {
      for (double& p : camera.d.origin) p += randOffset(pos);
      V3 aa = getRotation(camera);
      for (double& a : aa.v) a += randOffset(rot);
      setRotationAngleAxis(camera, aa);
    }
    for (double& p : camera.d.principal) p += randOffset(principal);
    if (focal != 0) {
      CHECK_EQ(camera.d.focal[0], -camera.d.focal[1]) << "pixels are not square";
      double scalar = camera.d.focal[0];
      scalar += randOffset(focal);
      camera.d.focal[0] = scalar;
      camera.d.focal[1] = -scalar;
    }
  }
}

const Cam& findCameraById(const std::string& id, const Rig& rig) {
  for (const Cam& c : rig)
    if (c.id == id) return c;
  LOG(FATAL) << "Camera id " << id << " not found";
  std::abort();
}

// Eigen's << of a column vector: one coefficient per line, right-aligned to the widest
std::string eigenColumn(const V3& a) {
  std::string s[3];
  size_t w = 0;
  for (int k = 0; k < 3; ++k) {
    std::ostringstream o;
    o << a.v[k];
    s[k] = o.str();
    w = std::max(w, s[k].size());
  }
  return std::string(w - s[0].size(), ' ') + s[0] + "\n" + std::string(w - s[1].size(), ' ') + s[1] + "\n" +
         std::string(w - s[2].size(), ' ') + s[2];
}

// ---- samples (RigAnalyzer.cpp:67-94) -------------------------------------------------------------------------------
std::vector<double> fibonacciUnits(int count, double discardRadians) {
  const double threshold = cos(discardRadians);
  std::vector<double> out;
  for (int i = 0; i < count; ++i) {
    const double y = (i + 0.5) / count * 2 - 1;
    const double r = sqrt(1 - y * y);
    const double phi = (1 + sqrt(5)) / 2;
    const double roty = i / phi * 2 * M_PI;
    const double p[3] = {sin(roty) * r, y, cos(roty) * r};
    if (std::abs(p[2]) < threshold) out.insert(out.end(), p, p + 3);
  }
  return out;
}

// ---- outputs --------------------------------------------------------------------------------------------------------
// PPM P2 text as the reference's ofstream writes it: "P2", the size and the maximum on their own lines, then each row's
// values followed by a space, each row ended by a newline
class Ppm {
 public:
  Ppm(int w, int h, long long maxValue) {
    out_ = "P2\n" + std::to_string(w) + " " + std::to_string(h) + "\n" + std::to_string(maxValue) + "\n";
    out_.reserve(out_.size() + (size_t)w * h * 3 + h);
  }
  void value(int v) {
    char b[16];
    const auto r = std::to_chars(b, b + sizeof b, v);
    out_.append(b, r.ptr);
    out_ += ' ';
  }
  void endRow() { out_ += '\n'; }
  void write(const std::string& path) const {
    std::ofstream f(path, std::ios::binary);
    f.write(out_.data(), (std::streamsize)out_.size());
  }

 private:
  std::string out_;
};

struct RigArrays {
  std::vector<DerpCameraDesc> descs;
  std::vector<double> rot;
};
RigArrays arrays(const Rig& rig) {
  RigArrays a;
  for (const Cam& c : rig) {
    a.descs.push_back(c.d);
    a.rot.insert(a.rot.end(), c.rot, c.rot + 9);
  }
  return a;
}

void saveEquirect(const std::string& filename, const Rig& rig) {
  const int kDimX = 360 * 5, kDimY = 180 * 5;
  const RigArrays a = arrays(rig);
  std::vector<int32_t> counts((size_t)kDimX * kDimY);
  std::vector<float> timing(counts.size());
  DERP_CALL(derp_rig_equirect_coverage(FLAGS_gpu, a.descs.data(), a.rot.data(), (int)rig.size(), kDimX, kDimY,
                                       FLAGS_overlap_distance, counts.data(), timing.data()));
  Ppm ppm(kDimX, kDimY, FLAGS_show_timing ? 256 : (long long)rig.size());
  double holes = 0, maxMin = 0, aveMin = 0;
  for (int y = 0; y < kDimY; ++y) {
    for (int x = 0; x < kDimX; ++x) {
      const size_t at = (size_t)y * kDimX + x;
      const double minTimingDiff = timing[at];
      maxMin = std::max(maxMin, minTimingDiff);
      aveMin += minTimingDiff;
      ppm.value(FLAGS_show_timing ? int((1.0 - minTimingDiff) * 255.0) : counts[at]);
      holes += (0 == counts[at]) ? 1 : 0;
    }
    ppm.endRow();
  }
  ppm.write(filename);
  const float kFrameRate = 60.0f;
  const float kFrameTime = 1000.0f / kFrameRate;
  LOG(INFO) << "Holes found (in pixels) = " << holes;
  LOG(INFO) << "Max of min timing distance = " << kFrameTime * maxMin << "ms";
  LOG(INFO) << "Ave of min timing distance = " << kFrameTime * aveMin / (kDimX * kDimY) << "ms";
}

void saveCamera(const std::string& filename, const std::string& camId, const Rig& rig) {
  const RigArrays a = arrays(rig);
  for (size_t i = 0; i < rig.size(); ++i) {
    if (rig[i].id != camId) continue;
    const int kDimX = rig[i].d.resolution[0], kDimY = rig[i].d.resolution[1];
    std::vector<int32_t> counts((size_t)std::max(kDimX, 0) * std::max(kDimY, 0));
    if (!counts.empty())
      DERP_CALL(derp_rig_camera_coverage(FLAGS_gpu, a.descs.data(), a.rot.data(), (int)rig.size(), (int)i,
                                         FLAGS_overlap_distance, counts.data()));
    Ppm ppm(kDimX, kDimY, (long long)rig.size());
    for (int y = 0; y < kDimY; ++y) {
      for (int x = 0; x < kDimX; ++x) ppm.value(counts[(size_t)y * kDimX + x]);
      ppm.endRow();
    }
    ppm.write(filename);
  }
}

void saveCrossSection(const std::string& filename, const Rig& rig) {
  const int kDim = 400;
  const RigArrays a = arrays(rig);
  std::vector<int32_t> counts((size_t)kDim * kDim);
  DERP_CALL(derp_rig_cross_section(FLAGS_gpu, a.descs.data(), a.rot.data(), (int)rig.size(), kDim, counts.data()));
  Ppm ppm(kDim, kDim, (long long)rig.size());
  for (int y = 0; y < kDim; ++y) {
    for (int x = 0; x < kDim; ++x) ppm.value(counts[(size_t)y * kDim + x]);
    ppm.endRow();
  }
  ppm.write(filename);
}

// saveRigObj (RigAnalyzer.cpp:271-344) with the ostream's default formatting
void writeVertexObj(std::ostream& file, const V3& color, const V3& p) {
  const double kScale = 1000;  // CAD wants mm, json is meters
  file << "v";
  for (int i = 0; i < 3; ++i) file << " " << kScale * p.v[i];
  for (int i = 0; i < 3; ++i) file << " " << color.v[i];
  file << "\n";
}
void writeFaceObj(std::ostream& file, const V3& color, const std::vector<V3>& positions) {
  for (const V3& p : positions) writeVertexObj(file, color, p);
  for (int order = 0; order < 2; ++order) {
    file << "f";
    for (int i = 0; i < int(positions.size()); ++i) file << " " << (order ? -int(positions.size()) + i : -1 - i);
    file << "\n";
  }
}
V3 add(const V3& a, const V3& b) { return V3{{a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]}}; }
V3 sub(const V3& a, const V3& b) { return V3{{a.v[0] - b.v[0], a.v[1] - b.v[1], a.v[2] - b.v[2]}}; }
void writeArrowObj(std::ostream& file, const V3& color, const V3& base, const V3& dir, const V3& t0, const V3& t1,
                   double length = 0.01, double radius = 0.001) {
  writeFaceObj(file, color, {add(base, scaled(dir, length)), add(base, scaled(t0, radius)), sub(base, scaled(t0, radius))});
  writeFaceObj(file, color, {add(base, scaled(dir, length)), add(base, scaled(t1, radius)), sub(base, scaled(t1, radius))});
}
void writeCameraObj(std::ostream& file, const V3& p, const V3& f, const V3& r, const V3& u) {
  writeArrowObj(file, {{1, 1, 1}}, p, f, r, u, 0.02);
  writeArrowObj(file, {{0, 1, 0}}, p, r, u, f);
  writeArrowObj(file, {{0, 0, 1}}, p, u, f, r);
}
void saveRigObj(const std::string& filename, const Rig& rig) {
  std::ostringstream file;
  for (int i = 0; i < int(rig.size()); ++i) {
    const V3 p = position(rig[i]), f = forward(rig[i]), r = right(rig[i]), u = up(rig[i]);
    writeCameraObj(file, p, f, r, u);
    for (int tri = 0; tri < i; ++tri) {
      const double kSize = 0.002;
      const V3 v = sub(p, scaled(r, kSize * tri));
      writeFaceObj(file, {{1, 0, 0}}, {v, sub(v, scaled(r, kSize)), sub(v, scaled(u, kSize))});
    }
  }
  writeArrowObj(file, {{1, 1, 0}}, {{0, 0, -1}}, {{0, 0, 1}}, {{1, 0, 0}}, {{0, 1, 0}}, 1.0, 0.01);
  std::ofstream out(filename);
  out << file.str();
}

}  // namespace

int main(int argc, char** argv) {
  std::string commandLine;  // gflags::GetArgv(): the arguments joined by spaces
  for (int i = 0; i < argc; ++i) commandLine += (i ? " " : "") + std::string(argv[i]);
  flags::initDep(argc, argv, kUsage);

  CHECK_NE(FLAGS_rig, "");
  // the reference's coverage report is undefined without samples (maxCoeff of an empty vector): refused before any work
  CHECK_GE(FLAGS_sample_count, 1) << "--sample_count must be at least 1";
  const std::vector<double> samples = fibonacciUnits(FLAGS_sample_count, FLAGS_discard_poles * M_PI / 180);
  CHECK(!samples.empty()) << "--discard_poles " << FLAGS_discard_poles << " leaves no samples";

  const io::Rig loaded = io::loadRig(FLAGS_rig);
  CHECK(!loaded.cams.empty()) << "the rig has no cameras";
  Rig rig;
  for (size_t i = 0; i < loaded.cams.size(); ++i) {
    Cam c;
    c.d = loaded.cams[i];
    if (!c.d.has_principal) {  // Camera(json): principal = resolution / 2
      c.d.has_principal = 1;
      c.d.principal[0] = c.d.resolution[0] / 2;
      c.d.principal[1] = c.d.resolution[1] / 2;
    }
    derp::DevCamera dc;
    CHECK(derp::host::makeCamera(c.d, &dc)) << "invalid camera " << loaded.ids[i];
    std::copy(dc.rot, dc.rot + 9, c.rot);
    c.id = loaded.ids[i];
    c.group = loaded.groups[i];
    rig.push_back(c);
  }

  // Modify rig
  if (!FLAGS_rearrange.empty()) {
    rig = makeNamedArrangement(FLAGS_rearrange, rig[0], FLAGS_custom);
  } else if (!FLAGS_eulers.empty()) {
    rig = makeRigFromEulers(rig[0], readVectorFile(FLAGS_eulers), false);
  } else if (!FLAGS_revolve.empty()) {
    rig = revolveRig(rig, readVectorFile(FLAGS_revolve));
  } else if (FLAGS_perturb_cameras) {
    std::srand(FLAGS_perturb_seed);
    perturbCameras(rig, FLAGS_perturb_positions, FLAGS_perturb_rotations, FLAGS_perturb_principals,
                   FLAGS_perturb_focals);
  }

  if (!FLAGS_rotate_cam_z.empty()) {
    const Cam zCam = findCameraById(FLAGS_rotate_cam_z, rig);
    const V3 zp = position(zCam);
    const double angle = acos(zp.v[0] * 0.0 + zp.v[1] * 0.0 + zp.v[2] * 1.0);
    V3 axis{{zp.v[1] * 1.0 - zp.v[2] * 0.0, zp.v[2] * 0.0 - zp.v[0] * 1.0, zp.v[0] * 0.0 - zp.v[1] * 0.0}};  // cross
    const double sq = axis.v[0] * axis.v[0] + axis.v[1] * axis.v[1] + axis.v[2] * axis.v[2];
    if (sq > 0) axis = V3{{axis.v[0] / std::sqrt(sq), axis.v[1] / std::sqrt(sq), axis.v[2] / std::sqrt(sq)}};  // normalize()
    double rot[9];
    derp::host::rotationOf(angle, axis.v, rot);
    for (Cam& camera : rig) {
      LOG(INFO) << eigenColumn(forward(camera));
      LOG(INFO) << eigenColumn(mul(rot, forward(camera)));
      setPosition(camera, mul(rot, position(camera)));
      setRotation(camera, mul(rot, forward(camera)), mul(rot, up(camera)), mul(rot, right(camera)));
    }
  }

  if (FLAGS_z_is_up || FLAGS_z_is_down || !FLAGS_rotate.empty()) {
    double m[9];
    if (FLAGS_z_is_up) {
      const double z[9] = {1, 0, 0, 0, 0, -1, 0, 1, 0};
      std::copy(z, z + 9, m);
    } else if (FLAGS_z_is_down) {
      const double z[9] = {1, 0, 0, 0, 0, 1, 0, -1, 0};
      std::copy(z, z + 9, m);
    } else {
      V3 euler;
      std::istringstream s(FLAGS_rotate);
      s >> euler.v[0] >> euler.v[1] >> euler.v[2];
      CHECK(s.eof() && !s.fail()) << "bad --rotate vector " << FLAGS_rotate;
      rotationMatrixFromEulers(euler, true, m);
    }
    for (Cam& camera : rig) {
      setPosition(camera, mul(m, position(camera)));
      setRotation(camera, mul(m, forward(camera)), mul(m, up(camera)), mul(m, right(camera)));
    }
  }

  if (FLAGS_scale_rig != 1) {
    LOG(INFO) << "scaling rig by " << FLAGS_scale_rig;
    for (Cam& camera : rig) setPosition(camera, scaled(position(camera), FLAGS_scale_rig));
  }

  if (FLAGS_radius > 0) {
    for (Cam& camera : rig) {
      V3 p = position(camera);
      const double n = norm(p);
      if (n > 0) p = V3{{p.v[0] / n, p.v[1] / n, p.v[2] / n}};  // normalized()
      setPosition(camera, scaled(p, FLAGS_radius));
    }
  }

  if (FLAGS_scale_resolution != 1) {  // Camera::rescale(scale * resolution)
    for (Cam& camera : rig) {
      for (int i = 0; i < 2; ++i) {
        const double newRes = camera.d.resolution[i] * FLAGS_scale_resolution;
        camera.d.principal[i] *= newRes / camera.d.resolution[i];
        camera.d.focal[i] *= newRes / camera.d.resolution[i];
        camera.d.resolution[i] = newRes;
      }
    }
  }

  // Go through N distances from min_distance to kNearInfinity
  const int kN = 20;
  const int n = (int)rig.size(), numSamples = (int)(samples.size() / 3);
  std::vector<double> distances(kN);
  for (int i = 0; i < kN; ++i) distances[i] = FLAGS_min_distance / (1 - i / double(kN));
  std::vector<uint64_t> hist((size_t)kN * (n + 1));
  {
    const RigArrays a = arrays(rig);
    DERP_CALL(derp_rig_coverage(FLAGS_gpu, a.descs.data(), a.rot.data(), n, samples.data(), numSamples,
                                distances.data(), kN, hist.data()));
  }
  for (int i = 0; i < kN; ++i) {
    const uint64_t* h = &hist[(size_t)i * (n + 1)];
    int minC = 0, maxC = 0;
    while (h[minC] == 0) ++minC;
    for (int c = 0; c <= n; ++c)
      if (h[c]) maxC = c;
    const double quality = minC + (numSamples - (long long)h[minC]) / double(numSamples);
    std::string histogram;
    for (int c = 0; c <= maxC; ++c) histogram += "h[" + std::to_string(c) + "] = " + std::to_string(h[c]) + ", ";
    char head[128];
    snprintf(head, sizeof head, "distance: %.2f quality: %.2f samples: %d ", distances[i], quality, numSamples);
    std::cout << head << histogram << std::endl;
  }

  if (!FLAGS_output_rig.empty()) rigjson::saveRig(FLAGS_output_rig, rig, {"command line:", commandLine}, true);
  if (!FLAGS_output_obj.empty()) saveRigObj(FLAGS_output_obj, rig);
  if (!FLAGS_output_equirect.empty()) saveEquirect(FLAGS_output_equirect, rig);
  if (!FLAGS_output_camera.empty() && !FLAGS_output_camera_id.empty())
    saveCamera(FLAGS_output_camera, FLAGS_output_camera_id, rig);
  if (!FLAGS_output_cross_section.empty()) saveCrossSection(FLAGS_output_cross_section, rig);
  return EXIT_SUCCESS;
}
