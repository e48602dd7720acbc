// DerpCLI — drop-in for facebook360_dep's source/depth_estimation/DerpCLI.cpp on H100.
// Same flags (names, types, defaults, help), same input/output directory tree, same rig JSON, same
// PFM/PNG outputs; the per-level work runs through libderp_b200.so (sm_90a CUDA kernels).
// Additions (surface extensions, defaults reproduce the reference): --num_depths (kNumDepths, Derp.h:33),
// --gpus / --gpu (frames are sharded across the GPUs of one box: frames are independent,
// DerpCLI.cpp:229-320).  There is no CPU fallback: without a CUDA device the process aborts.
#include <atomic>
#include <chrono>
#include <thread>

#include "exchange.h"
#include "io.h"

const std::string kUsageMessage = R"(
 - Runs depth estimation on a set of frames. We assume the inputs have already been resized into
 the appropriate pyramid level widths before execution. See scripts/render/config.py to see
 the assumed widths.

 - Example:
   ./DerpCLI \
   --input_root=/path/to/ \
   --output_root=/path/to/output \
   --rig=/path/to/rigs/rig.json \
   --first=000000 \
   --last=000000
 )";

DEFINE_string(background_disp, "", "path to background disparities");
DEFINE_string(background_frame, "000000", "background frame (lexical)");
DEFINE_string(cameras, "", "comma-separated destinations to render (empty for all)");
DEFINE_string(color, "", "path to input color images");
DEFINE_bool(do_bilateral_filter, true, "apply bilateral filter at each level");
DEFINE_bool(do_median_filter, true, "apply median filter to disparity at each level");
DEFINE_string(first, "000000", "first frame to process (lexical)");
DEFINE_string(foreground_masks, "", "path to foreground masks");
DEFINE_string(input_root, "", "path to input data (required)");
DEFINE_string(last, "000000", "last frame to process (lexical)");
DEFINE_int32(level_end, -1, "level to end at (-1 = finest)");
DEFINE_int32(level_start, -1, "level to start at (-1 = coarsest)");
DEFINE_double(max_depth_m, 1e4, "max depth (m)");
DEFINE_double(min_depth_m, .50, "min depth (m)");
DEFINE_int32(mismatches_start_level, -1, "(-1 = no mismatch handling)");
DEFINE_int32(num_levels, -1, "number of levels in the pyramid (-1 = uses highest level)");
DEFINE_string(output_formats, "", "saved formats, comma separated (exr, png, pfm supported)");
DEFINE_string(output_root, "", "path to output directory (required)");
DEFINE_bool(partial_coverage, false, "set to true if no 360 coverage");
DEFINE_int32(ping_pong_iterations, 1, "number of spatial propagation iterations");
DEFINE_int32(random_proposals, 2, "number of proposed random disparities before propagation");
DEFINE_int32(resolution, 2048, "Output resolution (width in pixels)");
DEFINE_string(rig, "", "path to camera rig .json");
DEFINE_bool(save_debug_images, false, "if true, save debugging output images");
DEFINE_int32(threads, -1, "number of threads (-1 = auto, 0 = none)");
DEFINE_bool(use_foreground_masks, false, "use pre-computed foreground masks");
DEFINE_double(var_high_thresh, 1e-3, "ignore variances higher than this threshold");
DEFINE_double(var_noise_floor, 4e-5, "noise variance floor on original, full-size images");
// extensions of this project
DEFINE_int32(num_depths, 150, "number of brute-force depth candidates (reference constant kNumDepths)");
DEFINE_int32(gpus, 1, "number of GPUs of this box to shard frames across");
DEFINE_int32(gpu, 0, "first CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

static void verifyInputs() {  // DerpCLI.cpp:69-118
  CHECK_NE(FLAGS_input_root, "");
  CHECK_NE(FLAGS_output_root, "");
  if (FLAGS_level_start >= 0 && FLAGS_level_end >= 0) CHECK_GE(FLAGS_level_start, FLAGS_level_end);
  if (FLAGS_rig.empty()) FLAGS_rig = FLAGS_input_root + "/rigs/rig_calibrated.json";
  if (FLAGS_color.empty()) FLAGS_color = FLAGS_input_root + "/" + io::kColorLevels;
  if (FLAGS_background_disp.empty()) FLAGS_background_disp = FLAGS_input_root + "/" + io::kBackgroundDispLevels;
  if (FLAGS_foreground_masks.empty()) FLAGS_foreground_masks = FLAGS_input_root + "/" + io::kForegroundMasksLevels;
  CHECK_GE(FLAGS_random_proposals, 0);
  CHECK_LE(FLAGS_first, FLAGS_last);
  CHECK_GE(FLAGS_num_depths, 2);
  CHECK(fs::is_directory(FLAGS_color)) << "No images in " << FLAGS_color;
  if (FLAGS_use_foreground_masks) {
    CHECK(fs::is_directory(FLAGS_background_disp))
        << "Asked to use background but no background disparities found in " << FLAGS_background_disp;
    CHECK(fs::is_directory(FLAGS_foreground_masks))
        << "Asked to use foreground masks but no foreground masks found in " << FLAGS_foreground_masks;
  }
  std::stringstream ss(FLAGS_output_formats);
  std::string fmt;
  while (std::getline(ss, fmt, ','))
    CHECK(fmt.empty() || fmt == "exr" || fmt == "png" || fmt == "pfm") << "Invalid output format specified: " << fmt;
}

// image size from the file header only
static bool imageSize(const fs::path& p, int* w, int* h) {
  std::ifstream f(p, std::ios::binary);
  if (!f.good()) return false;
  if (p.extension() == ".pfm") {
    std::string fmt;
    std::getline(f, fmt);
    f >> *w >> *h;
    return f.good();
  }
  uint8_t hdr[24];
  f.read(reinterpret_cast<char*>(hdr), 24);
  if (!f.good() || std::memcmp(hdr + 12, "IHDR", 4) != 0) return false;
  *w = (int)io::be32(hdr + 16);
  *h = (int)io::be32(hdr + 20);
  return true;
}

// getPyramidLevelSizes (Derp.cpp:72-99): first non-.tar file found under each level_<L> directory
static void getPyramidLevelSizes(std::map<int, std::pair<int, int>>& sizes, const fs::path& imageDir) {
  if (!fs::exists(imageDir)) return;
  for (const auto& entry : fs::directory_iterator(imageDir)) {
    const fs::path p = entry.path();
    if (!fs::is_directory(entry) || io::isHidden(p)) continue;
    const std::string name = p.filename().string();
    if (name.rfind("level_", 0) != 0) continue;
    std::vector<fs::path> files;
    for (const auto& e : fs::recursive_directory_iterator(p))
      if (fs::is_regular_file(e) && !io::isHidden(e.path()) && e.path().extension() != ".tar") files.push_back(e.path());
    if (files.empty()) continue;
    std::sort(files.begin(), files.end());
    int w = 0, h = 0;
    CHECK(imageSize(files[0], &w, &h)) << "cannot read image header: " << files[0].string();
    sizes[std::stoi(name.substr(6))] = {w, h};
  }
}

// verifyImagePaths (ImageUtil.cpp:62-94)
static void verifyImagePaths(const fs::path& dir, const io::Rig& rig, const std::vector<int>& cams,
                             const std::string& first, const std::string& last) {
  int a = 0, b = 0;
  try {
    a = std::stoi(first);
  } catch (...) {
    LOG(FATAL) << "Invalid frame name: " << first;
  }
  try {
    b = std::stoi(last);
  } catch (...) {
    LOG(FATAL) << "Invalid frame name: " << last;
  }
  CHECK_LE(a, b);
  CHECK_GT(cams.size(), 0u);
  const std::string ext = io::firstExtension(dir / rig.ids[cams[0]]);
  for (int c : cams)
    for (int f = a; f <= b; ++f) {
      const fs::path p = dir / rig.ids[c] / (io::zeroPad(f) + ext);
      CHECK(fs::is_regular_file(p)) << "Missing file: " << p.string();
    }
}

// --threads like ThreadPool.h:30-45 (-1 = all cores, 0 = inline): host-side image decoding and file writing only — the
// reference decodes a level's images with one task per camera (ImageUtil.h:65-94)
static int hostThreads() {
  return FLAGS_threads < 0 ? (int)std::max(1u, std::thread::hardware_concurrency()) : FLAGS_threads;
}
template <class F>
static void parallelFor(int n, F&& fn) {
  const int T = std::min(hostThreads(), n);
  if (T <= 1) {
    for (int i = 0; i < n; ++i) fn(i);
    return;
  }
  std::atomic<int> next(0);
  std::vector<std::thread> pool;
  for (int t = 0; t < T; ++t)
    pool.emplace_back([&] {
      for (int i = next++; i < n; i = next++) fn(i);
    });
  for (auto& th : pool) th.join();
}

struct Shared {
  io::Rig rig;
  std::vector<int> dst;  // indices into rig
  std::map<int, std::pair<int, int>> sizes;
  int numLevels = 0, levelStart = 0, levelEnd = 0, widthFull = 0, heightFull = 0, firstFrame = 0, numFrames = 0;
};

// one GPU's share of the work: a context and the destination cameras it owns
struct Worker {
  DerpCtx* ctx = nullptr;
  std::vector<int> dst;  // indices into rig
  std::vector<std::thread> writers;  // file output of finished levels, overlapped with the next level's GPU work
  void drain() {
    for (auto& t : writers) t.join();
    writers.clear();
  }
};

static void saveLevel(const Shared& shAll, Worker& wk, int level, const std::string& frameName, int W, int H) {
  DerpCtx* ctx = wk.ctx;
  Shared sh = shAll;
  sh.dst = wk.dst;
  // saveResults (Derp.cpp:922-938, PyramidLevel.h:487-529): pfm always; png/exr on request
  std::vector<std::string> formats = {"pfm"};
  std::stringstream ss(FLAGS_output_formats);
  std::string f;
  while (std::getline(ss, f, ','))
    if (!f.empty() && f != "pfm") formats.push_back(f);
  std::vector<float> disp((size_t)W * H), cost, conf;
  std::vector<uint8_t> mism, fov;
  if (FLAGS_save_debug_images) {
    cost.resize(disp.size());
    conf.resize(disp.size());
    mism.resize(disp.size());
    fov.resize(disp.size());
  }
  for (size_t d = 0; d < sh.dst.size(); ++d) {
    DERP_CALL(derp_get_disparity(ctx, (int)d, disp.data(), cost.empty() ? nullptr : cost.data(),
                                 conf.empty() ? nullptr : conf.data()));
    if (FLAGS_save_debug_images) {
      DERP_CALL(derp_get_mismatch_mask(ctx, (int)d, mism.data()));
      DERP_CALL(derp_get_fov_mask(ctx, (int)d, fov.data()));
    }
    // the buffers are copied into the writer: encoding + disk IO run while the GPU works on the next level
    wk.writers.emplace_back([=, &sh0 = shAll, dstIds = sh.dst]() {
    const Shared& sh = sh0;
    (void)dstIds;
    const std::string& id = sh.rig.ids[dstIds[d]];
    const fs::path stem = fs::path(io::levelDir(FLAGS_output_root + "/" + io::kDisparityLevels, level)) / id / frameName;
    for (const auto& ext : formats) io::saveDisparity(stem, ext, disp.data(), W, H);
    if (FLAGS_save_debug_images) {
      // saveDebugImages (PyramidLevel.h:418-461).  disparity_levels: convertTo<uint16_t> -> the same 16-bit PNG as the
      // png output format.  cost / confidence / mismatches: a CV_32F matrix times its plot scale handed to cv::imwrite,
      // which converts it to 8 bits (saturate_cast<uchar>(cvRound(v)), NaN -> 0) before encoding.
      io::saveDisparity(stem, "png", disp.data(), W, H);
      std::vector<uint8_t> g(disp.size());
      for (size_t i = 0; i < g.size(); ++i) g[i] = io::saturateU8(cost[i] * (255.0f / 100.0f));  // kScaleCostPlot
      io::writePng8(fs::path(io::levelDir(FLAGS_output_root + "/" + io::kCost, level)) / id / (frameName + ".png"), g.data(), W, H, 1);
      for (size_t i = 0; i < g.size(); ++i) g[i] = io::saturateU8(conf[i] * (255.0f * 100.0f));  // kScaleConfidencePlot
      io::writePng8(fs::path(io::levelDir(FLAGS_output_root + "/" + io::kConfidence, level)) / id / (frameName + ".png"), g.data(), W, H, 1);
      // overlayMismatchedDstDisparityMask (PyramidLevel.h:441-461): BGRA float, NaN outside the FOV, red where the
      // mismatch mask is set, (d, d, d, 1) elsewhere; times kScaleDisparityPlot = 255
      std::vector<uint8_t> bgra(disp.size() * 4);
      for (size_t i = 0; i < disp.size(); ++i) {
        float px[4];
        if (!fov[i]) {
          px[0] = NAN;  // cv::Mat_<cv::Vec4f>(size, NAN): Vec4f(NAN) sets channel 0 only
          px[1] = px[2] = px[3] = 0.f;
        } else if (mism[i]) {
          px[0] = 0.f;
          px[1] = 0.f;
          px[2] = 1.f;
          px[3] = 1.f;
        } else {
          px[0] = px[1] = px[2] = disp[i];
          px[3] = 1.f;
        }
        for (int k = 0; k < 4; ++k) bgra[i * 4 + k] = io::saturateU8(px[k] * 255.0f);
      }
      io::writePng8(fs::path(io::levelDir(FLAGS_output_root + "/" + io::kMismatches, level)) / id / (frameName + ".png"), bgra.data(), W, H, 4);
    }
    });
    if ((int)wk.writers.size() >= std::max(1, hostThreads())) wk.drain();  // bound the copies in flight
  }
}

// One (level, frame): DerpCLI.cpp:229-320
// `fromKept`: the coarser level of this frame was processed by this context just before and its disparities are still
// in device memory (derp_level_keep) — the PFM round trip of DerpCLI.cpp:287-288 is skipped (the files are still written).
static void processFrame(const Shared& shAll, Worker& wk, int level, int iFrame, Exchange* ex, bool fromKept) {
  DerpCtx* ctx = wk.ctx;
  Shared sh = shAll;
  sh.dst = wk.dst;
  const std::string frameName = io::zeroPad(iFrame + sh.firstFrame);
  const int W = sh.sizes.at(level).first, H = sh.sizes.at(level).second;
  const int S = (int)sh.rig.cams.size(), Sd = (int)sh.dst.size();
  DerpLevelParams lp{};
  lp.width = W;
  lp.height = H;
  lp.level = level;
  lp.num_levels = sh.numLevels;
  lp.full_width = sh.widthFull;
  lp.full_height = sh.heightFull;
  lp.var_noise_floor = (float)FLAGS_var_noise_floor;
  lp.var_high_thresh = (float)FLAGS_var_high_thresh;
  lp.use_foreground_masks = FLAGS_use_foreground_masks ? 1 : 0;
  DERP_CALL(derp_level_begin(ctx, &lp));

  const std::string colorDir = io::levelDir(FLAGS_color, level);
  std::vector<std::vector<uint16_t>> colors(S);
  std::vector<const uint16_t*> cptr(S);
  parallelFor(S, [&](int s) {
    int w, h;
    colors[s] = io::loadColor16(io::imagePath(colorDir, sh.rig.ids[s], frameName), &w, &h);
    CHECK(w == W && h == H) << "unexpected image size for " << sh.rig.ids[s] << " at level " << level;
    cptr[s] = colors[s].data();
  });
  DERP_CALL(derp_set_colors(ctx, cptr.data()));

  std::vector<std::vector<uint8_t>> masks, masksCoarse;
  if (FLAGS_use_foreground_masks) {
    const std::string maskDir = io::levelDir(FLAGS_foreground_masks, level);
    masks.resize(S);
    std::vector<const uint8_t*> mptr(S);
    for (int s = 0; s < S; ++s) {
      int w, h;
      masks[s] = io::loadMask(io::imagePath(maskDir, sh.rig.ids[s], frameName), &w, &h);
      CHECK(w == W && h == H) << "unexpected mask size";
      mptr[s] = masks[s].data();
    }
    DERP_CALL(derp_set_foreground_masks(ctx, mptr.data()));
    const std::string bgDir = io::levelDir(FLAGS_background_disp, level);
    std::vector<std::vector<float>> bgs(Sd);
    std::vector<const float*> bptr(Sd);
    for (int d = 0; d < Sd; ++d) {
      int w, h;
      bgs[d] = io::loadFloat(io::imagePath(bgDir, sh.rig.ids[sh.dst[d]], FLAGS_background_frame), &w, &h);
      CHECK(w == W && h == H) << "unexpected background disparity size";
      bptr[d] = bgs[d].data();
    }
    DERP_CALL(derp_set_background_disparity(ctx, bptr.data()));
  }

  if (level < sh.numLevels - 1) {  // DerpCLI.cpp:276-303: coarser disparity comes from disk
    const std::string coarseDir = io::levelDir(FLAGS_output_root + "/" + io::kDisparityLevels, level + 1);
    for (int d = 0; d < Sd; ++d) {
      const std::string& id = sh.rig.ids[sh.dst[d]];
      int cw = sh.sizes.at(level + 1).first, ch = sh.sizes.at(level + 1).second;
      std::vector<float> coarse;
      if (!fromKept) coarse = io::loadFloat(io::imagePath(coarseDir, id, frameName), &cw, &ch);
      std::vector<uint8_t> mc;
      const uint8_t* mfine = nullptr;
      if (FLAGS_use_foreground_masks) {
        int w, h;
        mc = io::loadMask(io::imagePath(io::levelDir(FLAGS_foreground_masks, level + 1), id, frameName), &w, &h);
        CHECK(w == cw && h == ch) << "coarse mask / disparity size mismatch";
        mfine = masks[sh.dst[d]].data();
      }
      if (fromKept)
        DERP_CALL(derp_upsample_from_kept(ctx, d, mc.empty() ? nullptr : mc.data(), mfine));
      else
        DERP_CALL(derp_upsample_from(ctx, d, coarse.data(), cw, ch, mc.empty() ? nullptr : mc.data(), mfine));
    }
  }

  DerpProcessOpts o{};
  o.num_depths = FLAGS_num_depths;
  o.min_depth_m = (float)FLAGS_min_depth_m;
  o.max_depth_m = (float)FLAGS_max_depth_m;
  o.partial_coverage = FLAGS_partial_coverage ? 1 : 0;
  o.random_proposals = FLAGS_random_proposals;
  o.ping_pong_iterations = FLAGS_ping_pong_iterations;
  o.mismatches_start_level = FLAGS_mismatches_start_level;
  o.do_bilateral_filter = FLAGS_do_bilateral_filter ? 1 : 0;
  o.do_median_filter = FLAGS_do_median_filter ? 1 : 0;
  LOG(INFO) << "Processing " << frameName << " level " << level;
  const bool mismatchLevel = !(level > FLAGS_mismatches_start_level || level == sh.numLevels - 1);  // Derp.cpp:726-728
  if (ex && mismatchLevel) {
    DERP_CALL(derp_level_estimate(ctx, &o));
    for (int d = 0; d < Sd; ++d) ex->planes[sh.dst[d]] = derp_disparity_device_ptr(ctx, d);
    ex->arriveAndWait();  // every plane estimated and published
    DERP_CALL(derp_gather_disparities(ctx, ex->planes.data()));
    ex->arriveAndWait();  // every GPU holds its copy: planes may change now
    DERP_CALL(derp_mismatches_gathered(ctx));
    DERP_CALL(derp_level_filter(ctx, &o));
  } else {
    DERP_CALL(derp_process_level(ctx, &o));
  }
  if (level > shAll.levelEnd) DERP_CALL(derp_level_keep(ctx));  // hand the level to the next finer one in device memory
  saveLevel(shAll, wk, level, frameName, W, H);
}

int main(int argc, char* argv[]) {
  flags::initDep(argc, argv, kUsageMessage);
  const auto t0 = std::chrono::steady_clock::now();
  verifyInputs();

  Shared sh;
  sh.rig = io::loadRig(FLAGS_rig);
  CHECK_GT(sh.rig.cams.size(), 0u) << "no source cameras!";
  // checked before any sharding, so it covers every --gpus layout
  CHECK_LE(sh.rig.cams.size(), 64u) << "this build handles rigs of up to 64 cameras (source-visibility masks are 64-bit); the "
                                       "reference has no such limit";
  sh.dst = io::filterDestinations(sh.rig, FLAGS_cameras);
  CHECK_GT(sh.dst.size(), 0u) << "no destination cameras!";

  getPyramidLevelSizes(sh.sizes, FLAGS_color);
  getPyramidLevelSizes(sh.sizes, FLAGS_output_root + "/" + io::kDisparityLevels);
  CHECK(!sh.sizes.empty()) << "no level_<n> directories under " << FLAGS_color;
  sh.numLevels = FLAGS_num_levels == -1 ? sh.sizes.rbegin()->first + 1 : FLAGS_num_levels;
  sh.levelStart = FLAGS_level_start >= 0 ? FLAGS_level_start : sh.numLevels - 1;
  // getLevelEnd (DerpCLI.cpp:158-177): first level whose width <= --resolution
  sh.levelEnd = 0;
  for (const auto& kv : sh.sizes)
    if (kv.second.first <= FLAGS_resolution) {
      sh.levelEnd = kv.first;
      break;
    }
  if (FLAGS_level_end >= 0)
    CHECK_GE(FLAGS_level_end, sh.levelEnd) << "Requested end level " << FLAGS_level_end
                                           << " is larger than requested resolution (" << FLAGS_resolution << ")";
  sh.levelEnd = std::max(sh.levelEnd, FLAGS_level_end);
  CHECK_LE(FLAGS_level_start, sh.numLevels);
  sh.firstFrame = std::stoi(FLAGS_first);
  sh.numFrames = std::stoi(FLAGS_last) - sh.firstFrame + 1;

  // verifyInputImagePaths (DerpCLI.cpp:136-156)
  std::vector<int> all(sh.rig.cams.size());
  for (size_t i = 0; i < all.size(); ++i) all[i] = (int)i;
  verifyImagePaths(io::levelDir(FLAGS_color, sh.levelStart), sh.rig, all, FLAGS_first, FLAGS_last);
  if (FLAGS_use_foreground_masks) {
    verifyImagePaths(io::levelDir(FLAGS_background_disp, sh.levelStart), sh.rig, sh.dst, FLAGS_background_frame,
                     FLAGS_background_frame);
    verifyImagePaths(io::levelDir(FLAGS_foreground_masks, sh.levelStart), sh.rig, sh.dst, FLAGS_first, FLAGS_last);
  }
  if (sh.levelStart < sh.numLevels - 1)
    verifyImagePaths(io::levelDir(FLAGS_output_root + "/" + io::kDisparityLevels, sh.levelStart + 1), sh.rig, sh.dst,
                     FLAGS_first, FLAGS_last);
  fs::create_directories(FLAGS_output_root);
  sh.widthFull = (int)sh.rig.cams[sh.dst[0]].resolution[0];
  sh.heightFull = (int)sh.rig.cams[sh.dst[0]].resolution[1];

  // One context per GPU (SURVEY.md 8(e)).  Enough frames: contiguous frame blocks per GPU, every context owns all
  // destinations.  Fewer frames than GPUs (e.g. one 24-camera 4096^2 frame on 8 GPUs): the DESTINATION cameras
  // are dealt round-robin to the GPUs instead and every GPU processes every frame for its destinations — all
  // stages except mismatch handling are independent per destination; that one stage exchanges the disparity
  // planes between the GPUs (struct Exchange).
  const int Gmax = std::max(1, FLAGS_gpus);
  const bool shardCameras = sh.numFrames < Gmax && (int)sh.dst.size() > 1;
  const int G = shardCameras ? std::min(Gmax, (int)sh.dst.size()) : std::max(1, std::min(Gmax, sh.numFrames));
  if (shardCameras && FLAGS_mismatches_start_level >= 0)
    CHECK_EQ(sh.dst.size(), sh.rig.cams.size()) << "Mismatches only valid when considering all cameras";  // Derp.cpp:689
  std::vector<Worker> workers(G);
  for (int g = 0; g < G; ++g) {
    if (shardCameras) {
      for (size_t i = g; i < sh.dst.size(); i += G) workers[g].dst.push_back(sh.dst[i]);
    } else {
      workers[g].dst = sh.dst;
    }
    std::vector<int32_t> d2s(workers[g].dst.begin(), workers[g].dst.end());
    DERP_CALL(derp_create(sh.rig.cams.data(), (int)sh.rig.cams.size(), d2s.data(), (int)d2s.size(), FLAGS_gpu + g,
                          &workers[g].ctx));
  }
  LOG(INFO) << "backend " << derp_backend() << ", " << G << " GPU(s), " << sh.numFrames << " frame(s), "
            << (shardCameras ? "destination cameras" : "frames") << " sharded, levels " << sh.levelStart << " -> "
            << sh.levelEnd;

  for (int level = sh.levelStart; level >= sh.levelEnd; --level) {
    CHECK(sh.sizes.count(level)) << "no images for level " << level;
    for (int d : sh.dst) {  // createLevelOutputDirs (DerpUtil.cpp:311-330)
      fs::create_directories(fs::path(FLAGS_output_root) / io::kDisparity / sh.rig.ids[d]);
      if (FLAGS_save_debug_images)
        for (const char* t : {io::kDisparityLevels, io::kCost, io::kConfidence, io::kMismatches})
          fs::create_directories(fs::path(io::levelDir(FLAGS_output_root + "/" + t, level)) / sh.rig.ids[d]);
    }
  }
  // The reference walks level-outer / frame-inner and re-reads the coarser level's PFMs (DerpCLI.cpp:220-320).  Frames
  // are independent, so each GPU worker walks ITS frames level by level instead and hands a finished level to the next
  // one in device memory; every file of the reference's run is still written, with the same bytes.
  {
    std::vector<std::thread> threads;
    const int per = (sh.numFrames + G - 1) / G;
    Exchange exchange(G, (int)sh.rig.cams.size());
    for (int g = 0; g < G; ++g)
      threads.emplace_back([&, g] {
        const int f0 = shardCameras ? 0 : g * per, f1 = shardCameras ? sh.numFrames : std::min(sh.numFrames, (g + 1) * per);
        for (int i = f0; i < f1; ++i)  // camera sharding: all GPUs walk the frames in step and meet on mismatch levels
          for (int level = sh.levelStart; level >= sh.levelEnd; --level)
            processFrame(sh, workers[g], level, i, (shardCameras && G > 1) ? &exchange : nullptr, level < sh.levelStart);
        workers[g].drain();
      });
    for (auto& w : threads) w.join();
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    LOG(INFO) << "-- Elapsed time: " << el << "s wall";
  }
  for (auto& w : workers) derp_destroy(w.ctx);
  const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  LOG(INFO) << "-- TOTAL: " << el << "s wall";
  return EXIT_SUCCESS;
}
