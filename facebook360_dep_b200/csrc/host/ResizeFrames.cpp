// ResizeFrames — the render pipeline's "Resize" stage (scripts/render/resize.py, resize_frames) on H100: every camera of
// every frame resized to the ten pyramid widths DerpCLI reads (scripts/render/config.py:46), written to
// <dst_dir>/level_<L>/<camera>/<frame><ext>.  Each image is read once and uploaded once; its ten cv2.resize(INTER_AREA)
// [+ cv2.threshold] run in libderp_b200.so (derp_resize_area).  PNG decode and encode run on host threads meanwhile.
// Differences from resize.py, all deliberate: frames are every integer from int(--first) to int(--last), zero-padded to
// six digits, as the pipeline's workers pass them (resize.py's own main passes list indexes); a failed check exits
// non-zero (resize.py prints and exits 0); each camera's extension is that of its first visible file in sorted order
// (resize.py takes the first file os.walk lists, in directory order).
#include <atomic>
#include <thread>

#include "../../../include/derp_resize.h"
#include "io.h"

const std::string kUsage = R"(
   - Resizes full-size frames to the fixed pyramid level sizes depth estimation reads.

   - Example:
     ./ResizeFrames \
     --src_dir=/path/to/video/color \
     --dst_dir=/path/to/video/color_levels \
     --rig=/path/to/rigs/rig.json \
     --first=000000 \
     --last=000000
 )";

DEFINE_string(dst_dir, "", "Destination directory (required)");
DEFINE_string(first, "", "First frame to extract (default: the first frame of the first camera)");
DEFINE_string(last, "", "Last frame to extract (default: the last frame of the first camera)");
DEFINE_string(rig, "", "Camera rig json (to get list of cameras) (required)");
DEFINE_string(src_dir, "", "Directory containing camera images (required)");
DEFINE_int32(threshold, -1, "binary threshold applied after the resize (v > threshold ? 255 : 0); -1: none");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

// config.WIDTHS
static const int kWidths[] = {2048, 1024, 512, 256, 200, 128, 100, 80, 60, 50};
constexpr int kLevels = sizeof(kWidths) / sizeof(kWidths[0]);

// resize_camera's level height: round(ratio * width) with Python's round (half to even), then height += height % 2
static int levelHeight(double resW, double resH, int width) {
  const double ratio = resH / resW;
  int h = (int)std::nearbyint(ratio * width);
  return h + h % 2;
}

static std::vector<std::string> visibleDirsSorted(const fs::path& dir) {
  std::vector<std::string> r;
  for (const auto& e : fs::directory_iterator(dir))
    if (fs::is_directory(e) && !io::isHidden(e.path())) r.push_back(e.path().filename().string());
  std::sort(r.begin(), r.end());
  return r;
}

// One caller's device copy of a full-size image, grown as needed and freed when its thread ends
struct DeviceImage {
  void* p = nullptr;
  size_t bytes = 0;
  int device = 0;
  ~DeviceImage() {
    if (p) derp_device_free(device, p);
  }
  void* upload(int dev, const void* host, size_t n) {
    if (n > bytes || dev != device) {
      if (p) DERP_CALL(derp_device_free(device, p));
      p = nullptr;
      device = dev;
      DERP_CALL(derp_device_alloc(device, n, &p));
      bytes = n;
    }
    DERP_CALL(derp_device_copy(device, p, host, n));
    return p;
  }
};

// Host threads: each keeps a device copy of its current full-size image and the library's per-thread scratch, and all
// of them share one GPU, so their number is capped rather than following the core count
constexpr int kMaxThreads = 8;
template <class F>
static void parallelFor(int n, F&& fn) {
  const int T = std::min({(int)std::max(1u, std::thread::hardware_concurrency()), kMaxThreads, n});
  std::atomic<int> next(0);
  std::vector<std::thread> pool;
  for (int t = 0; t < T; ++t)
    pool.emplace_back([&] {
      for (int i = next++; i < n; i = next++) fn(i);
    });
  for (auto& th : pool) th.join();
}

// A frame's header alone, so that every file is checked before any image is resized: .png at 8 or 16 bits with 1, 3 or 4
// channels (a palette expands to 3), or a 1-channel .pfm ("Pf")
static void checkHeader(const fs::path& p) {
  std::ifstream f(p, std::ios::binary);
  CHECK(f.good()) << "cannot read " << p.string();
  if (p.extension() == ".pfm") {
    std::string magic;
    std::getline(f, magic);
    CHECK(magic == "Pf") << "only 1-channel (Pf) .pfm files are supported: " << p.string();
    return;
  }
  uint8_t b[26] = {};
  f.read(reinterpret_cast<char*>(b), sizeof(b));
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  CHECK(f.gcount() == (std::streamsize)sizeof(b) && std::memcmp(b, sig, 8) == 0 && std::memcmp(b + 12, "IHDR", 4) == 0)
      << "not a PNG file: " << p.string();
  const int depth = b[24], ctype = b[25];
  CHECK(depth == 8 || depth == 16) << "PNG bit depth " << depth << " is not supported: " << p.string();
  const int channels = ctype == 0 ? 1 : ctype == 2 || ctype == 3 ? 3 : ctype == 4 ? 2 : ctype == 6 ? 4 : 0;
  CHECK(channels == 1 || channels == 3 || channels == 4) << channels << "-channel images are not supported: " << p.string();
}

// resize.py reads and writes .pfm through imageio (FreeImage), which, like cv2.imread, hands out the rows in the order of
// the PFM specification: the file's last row first.  So it resizes a PFM that stores its top row first (DerpCLI's
// disparities, io::writePfm) upside down and flips the levels back as it writes them.  INTER_AREA is not symmetric under
// a vertical flip, so the app resizes the rows in that same order.
static void flipRows(void* data, int h, size_t rowBytes) {
  uint8_t* d = static_cast<uint8_t*>(data);
  for (int y = 0; y < h / 2; ++y) std::swap_ranges(d + y * rowBytes, d + (y + 1) * rowBytes, d + (h - 1 - y) * rowBytes);
}

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_src_dir, "");
  CHECK_NE(FLAGS_dst_dir, "");
  CHECK_NE(FLAGS_rig, "");
  CHECK_GE(FLAGS_threshold, -1) << "--threshold: -1 (none) or a value to threshold at";
  const io::Rig rig = io::loadRig(FLAGS_rig);

  // the checks of resize.py's main, before any work
  CHECK(fs::is_directory(FLAGS_src_dir)) << "No cameras found in " << FLAGS_src_dir;
  const std::vector<std::string> camerasDir = visibleDirsSorted(FLAGS_src_dir);
  CHECK_GT(camerasDir.size(), 0u) << "No cameras found in " << FLAGS_src_dir;
  std::vector<std::string> camerasRig = rig.ids;
  std::sort(camerasRig.begin(), camerasRig.end());
  if (camerasRig != camerasDir) {
    std::string a, b;
    for (const auto& s : camerasRig) a += " " + s;
    for (const auto& s : camerasDir) b += " " + s;
    LOG(FATAL) << "Cameras from rig differ from cameras in source directory:" << a << " vs" << b;
  }
  // the frames come from the first camera's directory; each camera's extension from its own first file (get_frame_path)
  const fs::path dirCamRef = fs::path(FLAGS_src_dir) / camerasDir[0];
  const std::vector<fs::path> files = io::visibleFilesSorted(dirCamRef);
  CHECK_GT(files.size(), 0u) << "No frames found in " << dirCamRef.string();
  const std::string first = FLAGS_first.empty() ? files.front().stem().string() : FLAGS_first;
  const std::string last = FLAGS_last.empty() ? files.back().stem().string() : FLAGS_last;
  const int firstFrame = std::stoi(first), lastFrame = std::stoi(last);
  CHECK_LE(firstFrame, lastFrame) << "--first after --last";
  std::vector<std::string> exts;
  for (const std::string& id : rig.ids) {
    const std::vector<fs::path> own = io::visibleFilesSorted(fs::path(FLAGS_src_dir) / id);
    CHECK_GT(own.size(), 0u) << "No frames found in " << (fs::path(FLAGS_src_dir) / id).string();
    exts.push_back(own[0].extension().string());
    CHECK(exts.back() == ".png" || exts.back() == ".pfm") << "only .png and .pfm frames are supported (got "
                                                          << own[0].string() << ")";
  }

  struct Job {
    int cam;
    std::string frame;
  };
  std::vector<Job> jobs;
  for (int f = firstFrame; f <= lastFrame; ++f)
    for (size_t c = 0; c < rig.ids.size(); ++c) {
      const fs::path p = fs::path(FLAGS_src_dir) / rig.ids[c] / (io::zeroPad(f) + exts[c]);
      CHECK(fs::is_regular_file(p)) << "Non-existent file for resize: " << p.string();
      checkHeader(p);
      jobs.push_back(Job{(int)c, io::zeroPad(f)});
    }
  LOG(INFO) << "backend " << derp_backend() << ", " << jobs.size() << " images, " << kLevels << " levels each";
  for (size_t c = 0; c < rig.ids.size(); ++c) {
    std::string sizes;
    for (int W : kWidths)
      sizes += " " + std::to_string(W) + "x" + std::to_string(levelHeight(rig.cams[c].resolution[0], rig.cams[c].resolution[1], W));
    LOG(INFO) << "levels of " << rig.ids[c] << ":" << sizes;
  }

  parallelFor((int)jobs.size(), [&](int j) {
    static thread_local DeviceImage dsrc;
    const std::string& id = rig.ids[jobs[j].cam];
    const std::string name = jobs[j].frame + exts[jobs[j].cam];
    io::Image img = io::loadUnchanged(fs::path(FLAGS_src_dir) / id / name);
    const size_t n = (size_t)img.w * img.h * img.channels;
    std::vector<uint8_t> u8;
    const void* host = img.bits == 32 ? (const void*)img.f.data() : (const void*)img.u.data();
    if (img.bits == 8) {  // io::Image keeps 8-bit samples in 16-bit words
      u8.assign(img.u.begin(), img.u.end());
      host = u8.data();
    }
    const size_t sampleBytes = img.bits / 8;
    if (img.bits == 32) flipRows(img.f.data(), img.h, (size_t)img.w * sizeof(float));
    const void* src = dsrc.upload(FLAGS_gpu, host, n * sampleBytes);
    const DerpCameraDesc& cam = rig.cams[jobs[j].cam];
    for (int level = 0; level < kLevels; ++level) {
      const int W = kWidths[level], H = levelHeight(cam.resolution[0], cam.resolution[1], W);
      std::vector<uint8_t> out((size_t)W * H * img.channels * sampleBytes);
      DERP_CALL(derp_resize_area(FLAGS_gpu, src, img.bits, img.channels, img.w, img.h, out.data(), W, H, FLAGS_threshold));
      const fs::path dir = fs::path(io::levelDir(FLAGS_dst_dir, level)) / id;
      fs::create_directories(dir);
      if (img.bits == 32) {
        flipRows(out.data(), H, (size_t)W * sizeof(float));
        io::writePfm(dir / name, reinterpret_cast<const float*>(out.data()), W, H);
      } else if (img.bits == 16)
        io::writePng16(dir / name, reinterpret_cast<const uint16_t*>(out.data()), W, H, img.channels);
      else
        io::writePng8(dir / name, out.data(), W, H, img.channels);
    }
  });
  return EXIT_SUCCESS;
}
