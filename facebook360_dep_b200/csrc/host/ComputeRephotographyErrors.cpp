// ComputeRephotographyErrors — drop-in for source/render/ComputeRephotographyErrors.cpp without OpenGL.
// For each camera: the cubemap rendered from its own disparity and colour at its centre (the reference image) and the
// cubemap rendered from all other cameras, compared with MSSIM or NCC inside the reference's coverage.  Rendering and
// scoring run in libderp_b200.so (derp_rephoto_cubemap / derp_rephoto_score, csrc/derp_rephoto.cuh), under documented
// rasterisation and filtering rules instead of a GL driver's: see INTEGRATION.md for what differs from a GL run.
#include "../../../include/derp_rephoto.h"
#include "io.h"
#include "rephoto_plot.h"

const std::string kUsage = R"(
   - Computes rephotography error for a set of frames. Rephotography error for a single frame is
   computed by generating cubemaps for both the reference and the rendered data, translating the
   cubemap origin to the center of the reference camera, and computing the MSSIM for each camera.

   - Example:
     ./ComputeRephotographyErrors \
     --first=000000 \
     --last=000000 \
     --output=/path/to/output \
     --rig=/path/to/rigs/rig.json \
     --color=/path/to/video/color \
     --disparity=/path/to/output/disparity
 )";

DEFINE_string(cameras, "", "comma-separated cameras to render (empty for all)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_string(disparity, "", "path to disparity images (required)");
DEFINE_string(first, "", "first frame to process (lexical) (required)");
DEFINE_string(last, "", "last frame to process (lexical) (required)");
DEFINE_string(method, "MSSIM", "MSSIM or NCC");
DEFINE_string(output, "", "path to output directory (required)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_int32(stat_radius, 1, "local statistics window radius");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

// rephoto_util::formatResults: R, G, B from a B, G, R scalar
static std::string formatResults(const double* s) {
  char buf[128];
  std::snprintf(buf, sizeof(buf), "R %.2f%%, G %.2f%%, B %.2f%%", 100 * s[2], 100 * s[1], 100 * s[0]);
  return buf;
}

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_color, "");
  CHECK_NE(FLAGS_disparity, "");
  CHECK_NE(FLAGS_rig, "");
  CHECK_NE(FLAGS_output, "");
  CHECK_NE(FLAGS_first, "");
  CHECK_NE(FLAGS_last, "");
  CHECK_GT(FLAGS_stat_radius, 0);
  CHECK(FLAGS_method == "MSSIM" || FLAGS_method == "NCC") << "invalid method " << FLAGS_method;

  const io::Rig rig = io::loadRig(FLAGS_rig);
  const int S = (int)rig.cams.size();
  CHECK_GT(S, 0);
  const int first = std::stoi(FLAGS_first), last = std::stoi(FLAGS_last);
  io::verifyImagePaths(FLAGS_color, rig, first, last, "");
  io::verifyImagePaths(FLAGS_disparity, rig, first, last, ".pfm");
  LOG(INFO) << "backend " << derp_backend();

  const fs::path rephotoDir = fs::path(FLAGS_output) / "rephoto";
  for (const std::string& id : rig.ids) fs::create_directories(rephotoDir / id);
  std::vector<std::string> cameras;
  if (!FLAGS_cameras.empty()) {
    std::stringstream ss(FLAGS_cameras);
    std::string c;
    while (std::getline(ss, c, ',')) cameras.push_back(c);
  }
  const int method = FLAGS_method == "NCC" ? DERP_REPHOTO_NCC : DERP_REPHOTO_MSSIM;
  double totalScore[3] = {0, 0, 0};
  const int numFrames = last - first + 1;
  CHECK_GT(numFrames, 0);
  for (int iFrame = 0; iFrame < numFrames; ++iFrame) {
    const std::string frameName = io::zeroPad(iFrame + first);
    LOG(INFO) << "Processing frame " << frameName << "...";
    LOG(INFO) << "Loading color and disparity images...";
    std::vector<std::vector<float>> disps(S), colors(S);
    int W = 0, H = 0;
    for (int i = 0; i < S; ++i) {
      int w, h;
      disps[i] = io::readPfm(fs::path(FLAGS_disparity) / rig.ids[i] / (frameName + ".pfm"), &w, &h);
      if (i == 0) {
        W = w;
        H = h;
      }
      CHECK(w == W && h == H) << "disparity maps of one frame must share a size";
    }
    for (int i = 0; i < S; ++i) {  // loadResizedImages<Vec4f>(..., disps[0].size(), INTER_AREA)
      int w, h;
      std::vector<float> c = io::loadColorF32x4(io::imagePath(FLAGS_color, rig.ids[i], frameName), &w, &h);
      if (w != W || h != H) {
        std::vector<float> r((size_t)W * H * 4);
        io::area::resize(c.data(), w, h, 4, r.data(), W, H);
        c.swap(r);
      }
      colors[i] = std::move(c);
    }
    const int edge = H;  // cubeHeight = colors[0].rows
    const size_t cube = (size_t)6 * edge * edge;
    std::vector<float> refC(cube * 4), refD(cube * 4), renC(cube * 4), renD(cube * 4), x(cube * 3), y(cube * 3),
        score(cube * 3);
    std::vector<uint8_t> mask(cube);
    double frameScore[3] = {0, 0, 0};
    for (int i = 0; i < S; ++i) {
      const std::string& camId = rig.ids[i];
      if (!cameras.empty() && std::find(cameras.begin(), cameras.end(), camId) == cameras.end()) continue;
      LOG(INFO) << "Processing " << frameName << " - " << camId << "...";
      const float center[3] = {(float)rig.cams[i].origin[0], (float)rig.cams[i].origin[1], (float)rig.cams[i].origin[2]};
      const float* d1[1] = {disps[i].data()};
      const float* c1[1] = {colors[i].data()};
      DERP_CALL(derp_rephoto_cubemap(FLAGS_gpu, &rig.cams[i], 1, d1, c1, W, H, center, edge, refC.data(), refD.data(),
                                     nullptr));
      std::vector<DerpCameraDesc> others;
      std::vector<const float*> od, oc;
      for (int j = 0; j < S; ++j) {  // removeOne(i, ...)
        if (j == i) continue;
        others.push_back(rig.cams[j]);
        od.push_back(disps[j].data());
        oc.push_back(colors[j].data());
      }
      DERP_CALL(derp_rephoto_cubemap(FLAGS_gpu, others.data(), (int)others.size(), od.data(), oc.data(), W, H, center, edge,
                                     renC.data(), renD.data(), nullptr));
      for (size_t p = 0; p < cube; ++p) {  // mask = 255 * (alpha > 0); removeAlpha
        mask[p] = refC[4 * p + 3] > 0 ? 255 : 0;
        for (int c = 0; c < 3; ++c) {
          x[3 * p + c] = refC[4 * p + c];
          y[3 * p + c] = renC[4 * p + c];
        }
      }
      double avg[3];
      DERP_CALL(derp_rephoto_score(FLAGS_gpu, x.data(), y.data(), mask.data(), edge, 6 * edge, method, FLAGS_stat_radius,
                                   score.data(), avg));
      LOG(INFO) << camId << " " << FLAGS_method << ": " << formatResults(avg);
      for (int c = 0; c < 3; ++c) frameScore[c] += avg[c];
      const std::vector<uint8_t> plot = rephoto_plot::stackResults(refC.data(), refD.data(), renC.data(), renD.data(),
                                                                   score.data(), mask.data(), edge, 6 * edge);
      io::writePng8(rephotoDir / camId / (frameName + ".png"), plot.data(), 5 * edge, 6 * edge, 3);
    }
    const int n = !cameras.empty() ? (int)cameras.size() : S;
    for (int c = 0; c < 3; ++c) frameScore[c] /= n;
    LOG(INFO) << frameName << " average " << FLAGS_method << ": " << formatResults(frameScore);
    for (int c = 0; c < 3; ++c) totalScore[c] += frameScore[c];
  }
  for (int c = 0; c < 3; ++c) totalScore[c] /= numFrames;
  LOG(INFO) << "TOTAL average " << FLAGS_method << ": " << formatResults(totalScore);
  return EXIT_SUCCESS;
}
