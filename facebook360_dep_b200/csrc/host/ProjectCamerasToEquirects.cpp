// ProjectCamerasToEquirects — drop-in for source/conversion/ProjectCamerasToEquirects.cpp.  Each camera's colour becomes
// an equirect around the rig origin, assuming every pixel sees the scene at --depth.  The reference renders it through
// GL (CanopyScene::equirect); here the canopy rasteriser of libderp_b200.so (derp_canopy_render) renders the same scene:
// one camera, a constant disparity 1 / depth, no eye offset, no alpha blending.  See INTEGRATION.md for what differs.
#include "../../../include/derp_canopy.h"
#include "io.h"
#include "smr_host.h"
#include "sweep_host.h"

const std::string kUsage = R"(
  - Reads cameras and projects them to equirect at a given depth.

  - Example:
    ./ProjectCamerasToEquirects \
    --color=/path/to/video/color \
    --rig=/path/to/rigs/rig_calibrated.json \
    --first=000000 \
    --last=000000 \
    --output=/path/to/output
)";

DEFINE_string(cameras, "", "comma-separated cameras to render (empty for all)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_double(depth, 1000, "depth to project at (m)");
DEFINE_int32(eqr_width, 1024, "equirect width (pixels)");
DEFINE_string(file_type, "png", "Supports any image type allowed in OpenCV");
DEFINE_string(first, "000000", "first frame to process (lexical)");
DEFINE_string(last, "000000", "last frame to process (lexical)");
DEFINE_string(output, "", "output directory (required)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_rig, "");
  const io::Rig full = io::loadRig(FLAGS_rig);
  io::Rig rig;
  for (int i : io::filterDestinations(full, FLAGS_cameras)) {
    rig.cams.push_back(full.cams[i]);
    rig.ids.push_back(full.ids[i]);
  }

  // verifyInputs
  CHECK_NE(FLAGS_color, "");
  CHECK_NE(FLAGS_first, "");
  CHECK_NE(FLAGS_last, "");
  CHECK_NE(FLAGS_output, "");
  CHECK_GT(FLAGS_depth, 0);
  CHECK_GE(FLAGS_eqr_width, 0);
  CHECK_EQ(FLAGS_eqr_width % 2, 0) << "equirect width must be a multiple of 2";
  CHECK_GT(rig.cams.size(), 0);
  // the reference's imwrite throws on the empty image of --eqr_width 0
  CHECK_GT(FLAGS_eqr_width, 0) << "--eqr_width 0 renders an empty equirect";
  CHECK(FLAGS_file_type == "png") << "unsupported --file_type " << FLAGS_file_type << ": this build writes png";
  const int first = std::stoi(FLAGS_first), last = std::stoi(FLAGS_last);
  CHECK_LE(first, last);
  io::verifyImagePaths(FLAGS_color, rig, first, last, "");

  const int S = (int)rig.cams.size();
  const int height = FLAGS_eqr_width / 2.0f;
  const float position[3] = {0, 0, 0};
  const double t0 = sweep_host::nowMs();
  double decodeMs = 0, deviceMs = 0;
  std::atomic<double> encodeMs{0};
  {
    sweep_host::Writer writer((int)std::max(1u, std::thread::hardware_concurrency()));
    for (int iFrame = first; iFrame <= last; ++iFrame) {
      const std::string frameName = io::zeroPad(iFrame);
      LOG(INFO) << "Frame " << frameName << ": Loading colors...";
      double t = sweep_host::nowMs();
      std::vector<std::vector<float>> colors(S);
      std::vector<int> cw(S), ch(S);
      for (int i = 0; i < S; ++i)
        colors[i] = io::loadColorF32x4(io::imagePath(FLAGS_color, rig.ids[i], frameName), &cw[i], &ch[i]);
      decodeMs += sweep_host::nowMs() - t;

      for (int i = 0; i < S; ++i) {
        LOG(INFO) << "-- Frame " << frameName << ": Projecting " << rig.ids[i] << "...";
        // disparities.emplace_back(resolution.y(), resolution.x(), 1.0f / FLAGS_depth)
        const int dw = (int)rig.cams[i].resolution[0], dh = (int)rig.cams[i].resolution[1];
        const std::vector<float> disparity((size_t)dw * dh, float(1.0f / FLAGS_depth));
        const float* dp = disparity.data();
        const float* cp = colors[i].data();
        auto eqr = std::make_shared<std::vector<float>>((size_t)2 * height * height * 4);
        t = sweep_host::nowMs();
        DERP_CALL(derp_canopy_render(FLAGS_gpu, &rig.cams[i], 1, &dp, dw, dh, &cp, cw[i], ch[i], DERP_CANOPY_EQUIRECT,
                                     position, nullptr, 2 * height, height, 0.0f, 0, DERP_CANOPY_ON_SCREEN, eqr->data(),
                                     nullptr, nullptr));
        deviceMs += sweep_host::nowMs() - t;
        const fs::path file = fs::path(FLAGS_output) / rig.ids[i] / (frameName + "." + FLAGS_file_type);
        fs::create_directories(file.parent_path());
        writer.submit([eqr, height, file, &encodeMs] {
          const double te = sweep_host::nowMs();
          // convertImage<cv::Vec4w>: B, G, R and alpha at 16 bits, NaN -> 0
          const std::vector<uint16_t> v = smr::toPng16(eqr->data(), (size_t)2 * height * height, 4);
          io::writePng16(file, v.data(), 2 * height, height, 4);
          encodeMs = encodeMs + (sweep_host::nowMs() - te);
        });
      }
    }
  }
  LOG(INFO) << "Timing: decode " << decodeMs << " ms, device " << deviceMs << " ms, encode " << encodeMs.load()
            << " ms (summed over encoder threads), wall " << (sweep_host::nowMs() - t0) << " ms";
  return EXIT_SUCCESS;
}
