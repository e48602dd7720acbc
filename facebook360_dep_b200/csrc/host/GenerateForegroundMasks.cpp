// GenerateForegroundMasks — drop-in for source/render/GenerateForegroundMasks.cpp on H100 (SURVEY.md §8(f) rank 3):
// the masks DerpCLI --use_foreground_masks consumes.  Same flags, directory contract and output files; the per-camera
// work (INTER_AREA downscale to --width, Gaussian blur, L2 colour difference against the background frame, threshold,
// morphological closing: BackgroundSubtractionUtil.h:20-59) runs in libderp_b200.so.
#include <thread>

#include "../../../include/derp_blur.h"
#include "io.h"

const std::string kUsage = R"(
   - Generates foreground masks for a series of frames assuming a fixed background. Various
   parameters can be tweaked to improve the mask accuracy.

   - Example:
     ./GenerateForegroundMasks \
     --first=000000 \
     --last=000000 \
     --rig=/path/to/rigs/rig.json \
     --color=/path/to/video/color \
     --background_color=/path/to/background/color \
     --foreground_masks=/path/to/video/output
 )";

DEFINE_string(background_color, "", "path to input background color images (required)");
DEFINE_string(background_frame, "000000", "background frame (lexical)");
DEFINE_int32(blur_radius, 1, "Gaussian blur radius (0 = no blur)");
DEFINE_string(cameras, "", "comma-separated cameras to render (empty for all)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_string(first, "", "first frame to process (lexical) (required)");
DEFINE_string(foreground_masks, "", "path to output foreground masks (required)");
DEFINE_string(last, "", "last frame to process (lexical) (required)");
DEFINE_int32(morph_closing_size, 4, "Morphological closing size (0 = no closing)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_int32(threads, -1, "number of threads (-1 = max allowed, 0 = no threading)");
DEFINE_double(threshold, 0.04, "foreground/background RGB L2-norm threshold [0..1]");
DEFINE_int32(width, 2048, "optional downscaled output width");
DEFINE_int32(gpu, 0, "first CUDA device to use");
DEFINE_int32(gpus, 1, "number of GPUs of this box to shard frames across");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

// loadImage<Vec3w> + cv_util::resizeImage(..., outputSize) (INTER_AREA; identity when the size already matches)
static std::vector<uint16_t> loadResized(const fs::path& p, int W, int H, int device) {
  int w, h;
  std::vector<uint16_t> img = io::loadColor16(p, &w, &h);
  if (w == W && h == H) return img;
  CHECK(w >= W && h >= H) << "image smaller than the output size: " << p.string();
  std::vector<uint16_t> out((size_t)W * H * 3);
  DERP_CALL(derp_downscale_area(device, img.data(), w, h, out.data(), W, H));
  return out;
}

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_color, "");
  CHECK_NE(FLAGS_rig, "");
  CHECK_NE(FLAGS_background_color, "");
  CHECK_NE(FLAGS_foreground_masks, "");
  CHECK_NE(FLAGS_first, "");
  CHECK_NE(FLAGS_last, "");
  CHECK_NE(FLAGS_background_frame, "");
  CHECK_GT(FLAGS_width, 0);
  CHECK_GE(FLAGS_blur_radius, 0);
  CHECK_LE(FLAGS_blur_radius, 64) << "--blur_radius above 64 is not supported";
  CHECK_GE(FLAGS_threshold, 0);
  CHECK_GE(FLAGS_morph_closing_size, 0);
  const io::Rig rig = io::loadRig(FLAGS_rig);
  const std::vector<int> cams = io::filterDestinations(rig, FLAGS_cameras);
  CHECK_GT(cams.size(), 0u);

  // output size from the first background image (GenerateForegroundMasks.cpp:84-88)
  int bw, bh;
  {
    const io::Image first = io::loadUnchanged(io::imagePath(FLAGS_background_color, rig.ids[cams[0]], FLAGS_background_frame));
    bw = first.w;
    bh = first.h;
  }
  const int W = std::min(bw, FLAGS_width);
  const int H = (int)std::lrint(W * bh / float(bw));
  std::vector<std::vector<uint16_t>> background(cams.size());
  // derp_foreground_mask blurs with the default radius (1: its 3 x 3 kernel) or not at all. Larger radii (the UI's slider
  // goes up to 20) blur each background once and each frame with derp_gaussian_blur, and the mask is told not to blur.
  const bool ownBlur = FLAGS_blur_radius > 1;
  const int maskBlur = ownBlur ? 0 : FLAGS_blur_radius;
  for (size_t i = 0; i < cams.size(); ++i) {
    background[i] = loadResized(io::imagePath(FLAGS_background_color, rig.ids[cams[i]], FLAGS_background_frame), W, H, FLAGS_gpu);
    if (ownBlur) DERP_CALL(derp_gaussian_blur(FLAGS_gpu, background[i].data(), W, H, FLAGS_blur_radius, background[i].data()));
  }
  for (int c : cams) fs::create_directories(fs::path(FLAGS_foreground_masks) / rig.ids[c]);

  const int firstFrame = std::stoi(FLAGS_first), numFrames = std::stoi(FLAGS_last) - firstFrame + 1;
  CHECK_GT(numFrames, 0);
  for (int c : cams)
    for (int f = 0; f < numFrames; ++f)
      CHECK(fs::is_regular_file(io::imagePath(FLAGS_color, rig.ids[c], io::zeroPad(firstFrame + f))))
          << "Missing file for camera " << rig.ids[c] << " frame " << io::zeroPad(firstFrame + f);
  const int G = std::max(1, std::min(FLAGS_gpus, numFrames));
  LOG(INFO) << "backend " << derp_backend() << ", " << G << " GPU(s), masks " << W << "x" << H;
  const int per = (numFrames + G - 1) / G;
  std::vector<std::thread> threads;
  for (int g = 0; g < G; ++g)
    threads.emplace_back([&, g] {
      const int device = FLAGS_gpu + g;
      for (int i = g * per; i < std::min(numFrames, (g + 1) * per); ++i) {
        const std::string frame = io::zeroPad(firstFrame + i);
        LOG(INFO) << "Processing frame " << frame << "...";
        for (size_t k = 0; k < cams.size(); ++k) {
          const std::string& id = rig.ids[cams[k]];
          std::vector<uint16_t> color = loadResized(io::imagePath(FLAGS_color, id, frame), W, H, device);
          if (ownBlur) DERP_CALL(derp_gaussian_blur(device, color.data(), W, H, FLAGS_blur_radius, color.data()));
          std::vector<uint8_t> mask((size_t)W * H);
          DERP_CALL(derp_foreground_mask(device, background[k].data(), color.data(), W, H, maskBlur,
                                         (float)FLAGS_threshold, FLAGS_morph_closing_size, mask.data()));
          size_t count = 0;
          for (uint8_t& m : mask) {
            count += m;
            m = m ? 255 : 0;  // imwrite(255.0f * mask): 8-bit PNG, 0 / 255
          }
          LOG(INFO) << "foreground amount: " << 100.0 * count / mask.size() << "%";
          io::writePng8(fs::path(FLAGS_foreground_masks) / id / (frame + ".png"), mask.data(), W, H, 1);
        }
      }
    });
  for (auto& t : threads) t.join();
  return EXIT_SUCCESS;
}
