// CreateObjFromDisparityEquirect — drop-in for source/conversion/CreateObjFromDisparityEquirect.cpp.  A disparity equirect
// (e.g. SimpleMeshRenderer --format eqrdisp) becomes an OBJ mesh: the resize, the vertexes and the faces run in
// libderp_b200.so on the GPU (derp_equirect_mesh*, csrc/derp_mesh.cuh), the quadric simplification on the host inside
// the library.  See INTEGRATION.md for what differs from the reference (--create_mtl).
#include <cmath>
#include <cstdio>
#include <fstream>

#include "../../../include/derp_eqrmesh.h"
#include "io.h"

const std::string kUsage = R"(
  - Creates an OBJ (optionally with texturing) from a disparity equirect.

  - Example:
    ./CreateObjFromDisparityEquirect \
    --input_png_color=/path/to/equirects/color.png \
    --input_png_disp=/path/to/equirects/disparity.png \
    --output_obj=/path/to/output/test.obj
  )";

DEFINE_bool(create_mtl, false, "cerate MTL file and attach to OBJ");
DEFINE_string(input_png_color, "", "path to input color png (required)");
DEFINE_string(input_png_disp, "", "path to input disparity png (required)");
DEFINE_double(max_depth, 700.0, "maximum depth. Use something like 20 to visualize");
DEFINE_int32(num_faces, 200000, "number of output faces");
DEFINE_string(output_obj, "", "path to output obj file (required)");
DEFINE_double(scale, 1.0, "depth map resolution before decimation");
DEFINE_double(strictness, 0.8, "[0, 1] mesh simplification aggressiveness. 0 = no simplification");
DEFINE_double(tear_ratio, 0.95, "depth ratio that causes mesh to tear");
DEFINE_int32(threads, 12, "number of threads");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                    \
  do {                                                                     \
    const int rc_ = (expr);                                                \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

// mesh_util::writeMtl (MeshUtil.h:131-144): the .mtl next to the OBJ, the colour path relative to the OBJ's directory;
// returns the .mtl's file name
static std::string writeMtl(const fs::path& obj, const fs::path& color) {
  const std::string rel = fs::relative(color, obj.parent_path()).string();
  fs::path mtl(obj);
  mtl.replace_extension(".mtl");
  std::ofstream f(mtl.string());
  f << "newmtl material" << std::endl;
  f << "illum 0" << std::endl;
  f << "Kd 1 1 1" << std::endl;
  f << "map_Kd " << rel << std::endl;
  return mtl.filename().string();
}

// mesh_util::writeObj (MeshUtil.h:91-129); with a material, every vertex is followed by its texture coordinate from
// mesh_util::addTextureCoordinatesEquirect (MeshUtil.h:408-418), in fp64 with the host's atan2
static void writeObj(const std::vector<double>& v, const std::vector<uint32_t>& f, const fs::path& path,
                     const std::string& mtl) {
  FILE* fp = fopen(path.c_str(), "w");
  CHECK(fp) << "file open failed: " << path;
  if (!mtl.empty()) fprintf(fp, "mtllib %s\nusemtl material\n", mtl.c_str());
  for (size_t i = 0; i + 2 < v.size(); i += 3) {
    const double x = v[i], y = v[i + 1], z = v[i + 2];
    fprintf(fp, "v %g %g %g\n", x, y, z);
    if (!mtl.empty()) {
      const double xzNorm = std::sqrt(x * x + z * z);
      fprintf(fp, "vt %g %g\n", std::atan2(-z, -x) * 0.5 / M_PI + 0.5, -std::atan2(-y, xzNorm) / M_PI + 0.5);
    }
  }
  for (size_t i = 0; i + 2 < f.size(); i += 3) {
    const int a = (int)f[i] + 1, b = (int)f[i + 1] + 1, c = (int)f[i + 2] + 1;
    if (mtl.empty())
      fprintf(fp, "f %d %d %d\n", a, b, c);
    else
      fprintf(fp, "f %d/%d %d/%d %d/%d\n", a, a, b, b, c, c);
  }
  fclose(fp);
}

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_input_png_disp, "");
  CHECK_NE(FLAGS_input_png_color, "");
  CHECK_NE(FLAGS_output_obj, "");
  CHECK(0 <= FLAGS_strictness && FLAGS_strictness <= 1) << "strictness must be between 0 and 1";

  LOG(INFO) << "Reading disparity image...";
  int w = 0, h = 0;
  const std::vector<float> disp = io::loadFloat(FLAGS_input_png_disp, &w, &h);
  int mw = 0, mh = 0;
  DERP_CALL(derp_equirect_mesh_size(w, h, FLAGS_scale, &mw, &mh));

  LOG(INFO) << "Generating mesh...";
  std::vector<double> vertexes((size_t)mw * mh * 3);
  std::vector<uint32_t> faces((size_t)mw * mh * 6);
  uint64_t nv = 0, nf = 0;
  if (FLAGS_strictness > 0) {
    // --threads only splits the reference's independent per-face work: the result does not depend on it
    LOG(INFO) << "Mesh simplification...";
    DERP_CALL(derp_equirect_mesh_simplified(FLAGS_gpu, disp.data(), w, h, FLAGS_scale, FLAGS_max_depth,
                                            (float)FLAGS_tear_ratio, FLAGS_num_faces, (float)FLAGS_strictness,
                                            vertexes.data(), faces.data(), &nv, &nf));
  } else {
    DERP_CALL(derp_equirect_mesh(FLAGS_gpu, disp.data(), w, h, FLAGS_scale, FLAGS_max_depth, (float)FLAGS_tear_ratio,
                                 vertexes.data(), faces.data(), &nv, &nf));
  }
  vertexes.resize(nv * 3);
  faces.resize(nf * 3);
  // the reference prints Eigen's size() (rows x columns)
  LOG(INFO) << "Num vertexes: " << nv * 3 << ", num faces: " << nf * 3;

  LOG(INFO) << "Creating OBJ...";
  const std::string mtl = FLAGS_create_mtl ? writeMtl(FLAGS_output_obj, FLAGS_input_png_color) : "";
  writeObj(vertexes, faces, FLAGS_output_obj, mtl);
  return EXIT_SUCCESS;
}
