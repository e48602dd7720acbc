// ProjectEquirectsToCameras — drop-in for source/conversion/ProjectEquirectsToCameras.cpp.  Each camera's equirect mask
// (a region painted once in 360 degrees) becomes a mask in that camera, assuming every pixel sees the scene at --depth.
// The projection runs in libderp_b200.so (derp_project_equirect_masks, csrc/derp_sweepview.cuh) for the whole rig per
// frame; PNGs are encoded on host threads while the next frame runs.  See INTEGRATION.md for what differs from the
// reference.
#include "../../../include/derp_sweepview.h"
#include "io.h"
#include "sweep_host.h"

const std::string kUsage = R"(
  - Reads equirect masks and projects them to individual cameras assuming a given depth.

  - Example:
    ./ProjectEquirectsToCameras \
    --eqr_masks=/path/to/video/equirect_masks/ \
    --rig=/path/to/rigs/rig.json \
    --first=000000 \
    --last=000000 \
    --output=/path/to/output/
)";

DEFINE_string(cameras, "", "comma-separated cameras to render (empty for all)");
DEFINE_double(depth, 1000, "depth to project at (m)");
DEFINE_string(eqr_masks, "", "path to input equirect masks (required)");
DEFINE_string(file_type, "png", "Supports any image type allowed in OpenCV");
DEFINE_string(first, "000000", "first frame to process (lexical) (required)");
DEFINE_string(last, "000000", "last frame to process (lexical) (required)");
DEFINE_string(output, "", "output directory (required)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_int32(threads, -1, "number of threads (-1 = auto, 0 = none)");
DEFINE_int32(width, 0, "width of projected camera images (0 = size from rig file)");
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
  CHECK_NE(FLAGS_eqr_masks, "");
  CHECK_NE(FLAGS_first, "");
  CHECK_NE(FLAGS_last, "");
  CHECK_NE(FLAGS_output, "");
  CHECK_GT(FLAGS_depth, 0);
  CHECK_GE(FLAGS_width, 0);
  CHECK_EQ(FLAGS_width % 2, 0) << "equirect width must be a multiple of 2";
  CHECK_GT(rig.cams.size(), 0);
  CHECK(FLAGS_file_type == "png") << "unsupported --file_type " << FLAGS_file_type << ": this build writes png";
  const int first = std::stoi(FLAGS_first), last = std::stoi(FLAGS_last);
  CHECK_LE(first, last);
  io::verifyImagePaths(FLAGS_eqr_masks, rig, first, last, "");

  // rescaleCameras
  const int S = (int)rig.cams.size();
  std::vector<DerpCameraDesc> cams(rig.cams);
  for (int i = 0; i < S; ++i) {
    if (FLAGS_width > 0) cams[i] = sweep_host::rescaledToWidth(rig.cams[i], FLAGS_width);
    LOG(INFO) << rig.ids[i] << " output resolution: " << cams[i].resolution[0] << "x" << cams[i].resolution[1];
  }

  const double t0 = sweep_host::nowMs();
  double decodeMs = 0, deviceMs = 0;
  std::atomic<double> encodeMs{0};
  {
    const int threads = FLAGS_threads > 0 ? FLAGS_threads : FLAGS_threads == 0 ? 1 : (int)std::max(1u, std::thread::hardware_concurrency());
    sweep_host::Writer writer(threads);
    for (int iFrame = first; iFrame <= last; ++iFrame) {
      const std::string frameName = io::zeroPad(iFrame);
      LOG(INFO) << "Frame " << frameName << ": Loading equirect masks...";
      double t = sweep_host::nowMs();
      std::vector<std::vector<uint8_t>> masks(S);
      std::vector<int32_t> sizes(2 * S);
      std::vector<const uint8_t*> maskPtrs(S);
      for (int i = 0; i < S; ++i) {
        masks[i] = io::loadMask(io::imagePath(FLAGS_eqr_masks, rig.ids[i], frameName), &sizes[2 * i], &sizes[2 * i + 1]);
        maskPtrs[i] = masks[i].data();
      }
      decodeMs += sweep_host::nowMs() - t;

      std::vector<std::shared_ptr<std::vector<uint8_t>>> outs(S);
      std::vector<uint8_t*> outPtrs(S);
      for (int i = 0; i < S; ++i) {
        LOG(INFO) << "-- Frame " << frameName << ": Projecting to " << rig.ids[i] << "...";
        outs[i] = std::make_shared<std::vector<uint8_t>>((size_t)(int)cams[i].resolution[0] * (int)cams[i].resolution[1]);
        outPtrs[i] = outs[i]->data();
      }
      t = sweep_host::nowMs();
      DERP_CALL(derp_project_equirect_masks(FLAGS_gpu, cams.data(), S, FLAGS_depth, maskPtrs.data(), sizes.data(),
                                            outPtrs.data()));
      deviceMs += sweep_host::nowMs() - t;
      for (int i = 0; i < S; ++i) {
        const fs::path file = fs::path(FLAGS_output) / rig.ids[i] / (frameName + "." + FLAGS_file_type);
        fs::create_directories(file.parent_path());
        auto out = outs[i];
        const int w = (int)cams[i].resolution[0], h = (int)cams[i].resolution[1];
        writer.submit([out, w, h, file, &encodeMs] {
          const double te = sweep_host::nowMs();
          io::writePng8Gray(file, out->data(), w, h);  // imwrite(255.0f * camMask): 0 / 255 bytes
          encodeMs = encodeMs + (sweep_host::nowMs() - te);
        });
      }
    }
  }
  LOG(INFO) << "Timing: decode " << decodeMs << " ms, device " << deviceMs << " ms, encode " << encodeMs.load()
            << " ms (summed over encoder threads), wall " << (sweep_host::nowMs() - t0) << " ms";
  return EXIT_SUCCESS;
}
