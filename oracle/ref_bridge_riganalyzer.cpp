// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// Bridge of the RigAnalyzer checker (riganalyzer.mk): the reference's OWN source/rig/RigAnalyzer.cpp, compiled where it
// lies (main renamed), linked with the reference's Camera.o.  Nothing here restates the analyzer; every export calls
// the app's own functions with its FLAGS_ set by the caller:
//   ref_ra_set_flag   sets FLAGS_<name> from its text (every flag of the app's DEFINE_ lines)
//   ref_ra_main       runs main with the given arguments (argv[0] first) and std::cout captured into out; returns the
//                     number of bytes main printed.  gflags::GetArgv() returns the arguments joined by spaces.  The rig
//                     state after main's edits is what --output_rig writes (the stand-in folly writes 17 significant
//                     digits, which round-trip every double)
//   ref_ra_samples    getFibonacciUnits(count), then discardPoles(samples, degrees * M_PI / 180): x, y, z per sample
//   ref_ra_save       saveRigObj (0), saveEquirect (1), saveCamera (2, camera id cam_id) or saveCrossSection (3) of
//                     the rig loaded from a rig JSON file by Camera::loadRig
//   ref_ra_count      per point, the number of cameras of the loaded rig whose Camera::sees is true
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "source/util/Camera.h"

using namespace fb360_dep;

namespace gflags {
std::string g_refArgv;
}  // namespace gflags
namespace fb360_dep::system_util {
void initDep(int&, char**&, const std::string) {}
}  // namespace fb360_dep::system_util

extern double FLAGS_custom, FLAGS_discard_poles, FLAGS_min_distance, FLAGS_overlap_distance, FLAGS_perturb_focals,
    FLAGS_perturb_positions, FLAGS_perturb_principals, FLAGS_perturb_rotations, FLAGS_radius, FLAGS_scale_resolution,
    FLAGS_scale_rig;
extern bool FLAGS_one_based_indexing, FLAGS_perturb_cameras, FLAGS_show_timing, FLAGS_z_is_down, FLAGS_z_is_up;
extern int32_t FLAGS_perturb_seed, FLAGS_sample_count;
extern std::string FLAGS_eulers, FLAGS_output_camera, FLAGS_output_camera_id, FLAGS_output_cross_section,
    FLAGS_output_equirect, FLAGS_output_obj, FLAGS_output_rig, FLAGS_rearrange, FLAGS_revolve, FLAGS_rig, FLAGS_rotate,
    FLAGS_rotate_cam_z;

int ref_rig_analyzer_main(int argc, char* argv[]);
std::vector<Camera::Vector3> getFibonacciUnits(int count);
std::vector<Camera::Vector3> discardPoles(const std::vector<Camera::Vector3>& samples, const Camera::Real radians);
void saveRigObj(const std::string& filename, const Camera::Rig& rig);
void saveCamera(const std::string& filename, const std::string& camId, const Camera::Rig& rig);
void saveEquirect(const std::string& filename, const Camera::Rig& rig);
void saveCrossSection(const std::string& filename, const Camera::Rig& rig);

namespace {
struct Flag {
  const char* name;
  char type;  // d(ouble), b(ool), i(nt32), s(tring)
  void* p;
};
const Flag kFlags[] = {
    {"custom", 'd', &FLAGS_custom},
    {"discard_poles", 'd', &FLAGS_discard_poles},
    {"eulers", 's', &FLAGS_eulers},
    {"min_distance", 'd', &FLAGS_min_distance},
    {"overlap_distance", 'd', &FLAGS_overlap_distance},
    {"one_based_indexing", 'b', &FLAGS_one_based_indexing},
    {"output_camera", 's', &FLAGS_output_camera},
    {"output_camera_id", 's', &FLAGS_output_camera_id},
    {"output_cross_section", 's', &FLAGS_output_cross_section},
    {"output_equirect", 's', &FLAGS_output_equirect},
    {"output_obj", 's', &FLAGS_output_obj},
    {"output_rig", 's', &FLAGS_output_rig},
    {"perturb_cameras", 'b', &FLAGS_perturb_cameras},
    {"perturb_focals", 'd', &FLAGS_perturb_focals},
    {"perturb_positions", 'd', &FLAGS_perturb_positions},
    {"perturb_principals", 'd', &FLAGS_perturb_principals},
    {"perturb_rotations", 'd', &FLAGS_perturb_rotations},
    {"perturb_seed", 'i', &FLAGS_perturb_seed},
    {"radius", 'd', &FLAGS_radius},
    {"rearrange", 's', &FLAGS_rearrange},
    {"revolve", 's', &FLAGS_revolve},
    {"rig", 's', &FLAGS_rig},
    {"rotate", 's', &FLAGS_rotate},
    {"rotate_cam_z", 's', &FLAGS_rotate_cam_z},
    {"sample_count", 'i', &FLAGS_sample_count},
    {"scale_resolution", 'd', &FLAGS_scale_resolution},
    {"show_timing", 'b', &FLAGS_show_timing},
    {"z_is_down", 'b', &FLAGS_z_is_down},
    {"z_is_up", 'b', &FLAGS_z_is_up},
    {"scale_rig", 'd', &FLAGS_scale_rig},
};
}  // namespace

extern "C" {

int ref_ra_set_flag(const char* name, const char* value) {
  for (const Flag& f : kFlags) {
    if (std::strcmp(f.name, name) != 0) continue;
    const std::string v(value);
    switch (f.type) {
      case 'd': *static_cast<double*>(f.p) = std::strtod(value, nullptr); break;
      case 'b': *static_cast<bool*>(f.p) = v == "true" || v == "1"; break;
      case 'i': *static_cast<int32_t*>(f.p) = (int32_t)std::strtol(value, nullptr, 10); break;
      default: *static_cast<std::string*>(f.p) = v;
    }
    return 0;
  }
  return -1;
}

long ref_ra_main(const char* const* args, int argc, char* out, long cap) {
  std::vector<std::string> store(args, args + argc);
  std::vector<char*> argv;
  gflags::g_refArgv.clear();
  for (int i = 0; i < argc; ++i) {
    argv.push_back(&store[i][0]);
    gflags::g_refArgv += (i ? " " : "") + store[i];
  }
  argv.push_back(nullptr);
  std::ostringstream captured;
  std::streambuf* old = std::cout.rdbuf(captured.rdbuf());
  ref_rig_analyzer_main(argc, argv.data());
  std::cout.rdbuf(old);
  const std::string s = captured.str();
  if ((long)s.size() <= cap) std::memcpy(out, s.data(), s.size());
  return (long)s.size();
}

int ref_ra_samples(int count, double degrees, double* out, int cap) {
  const std::vector<Camera::Vector3> s = discardPoles(getFibonacciUnits(count), degrees * M_PI / 180);
  for (int i = 0; i < (int)s.size() && i < cap; ++i)
    for (int k = 0; k < 3; ++k) out[3 * i + k] = s[i][k];
  return (int)s.size();
}

int ref_ra_save(int kind, const char* rig_path, const char* out_path, const char* cam_id) {
  const Camera::Rig rig = Camera::loadRig(rig_path);
  if (kind == 0) saveRigObj(out_path, rig);
  else if (kind == 1) saveEquirect(out_path, rig);
  else if (kind == 2) saveCamera(out_path, cam_id, rig);
  else if (kind == 3) saveCrossSection(out_path, rig);
  else return -1;
  return 0;
}

int ref_ra_count(const char* rig_path, const double* points, int n, int32_t* out) {
  const Camera::Rig rig = Camera::loadRig(rig_path);
  for (int i = 0; i < n; ++i) {
    const Camera::Vector3 p(points[3 * i], points[3 * i + 1], points[3 * i + 2]);
    int count = 0;
    for (const Camera& c : rig) count += c.sees(p) ? 1 : 0;
    out[i] = count;
  }
  return 0;
}

}  // extern "C"
