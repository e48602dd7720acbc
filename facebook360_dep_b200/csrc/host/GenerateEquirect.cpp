// GenerateEquirect — drop-in for source/render/GenerateEquirect.cpp.  At each of --num_depths depths, an equirect around
// the rig origin averages the nearest texel of every camera that sees each pixel's point (optionally cropped to the
// visible region and with the rig rotated so that --camera_id faces the centre).  The slices are computed in
// libderp_b200.so (derp_sweep_crop_bounds / derp_sweep_equirect, csrc/derp_sweepview.cuh); PNGs are encoded on host
// threads while the next slices run.  See INTEGRATION.md for what differs from the reference.
#include "../../../include/derp_sweepview.h"
#include "io.h"
#include "sweep_host.h"

const std::string kUsage = R"(
  - Generates an equirect from a set of color images at a uniformly spaced range of depths.

  - Example:
    ./GenerateEquirect \
    --color=/path/to/video/color \
    --output=/path/to/output \
    --rig=/path/to/rigs/rig.json \
    --frame=000000 \
    --depth_min=1.0 \
    --depth_max=1000.0 \
    --num_depths=50
  )";

DEFINE_bool(black_bg, false, "set the background to be optionally black (red by default)");
DEFINE_string(camera_id, "", "id of camera selected to be centered");
DEFINE_string(cameras, "", "cameras to render (comma-separated)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_bool(crop_equirect, false, "crop the equirect to only include visible images");
DEFINE_double(depth_max, 10.0, "max depth in m");
DEFINE_double(depth_min, 1.0, "min depth in m");
DEFINE_string(frame, "000000", "frame to process (lexical)");
DEFINE_uint64(height, 512, "equirect height in pixels");
DEFINE_uint64(num_depths, 50, "num depths");
DEFINE_string(output, "", "path to output directory (required)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_double(scale, 1, "image scale factor");
DEFINE_int32(threads, -1, "number of threads (-1 = max allowed, 0 = no threading)");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

constexpr int kSlicesPerCall = 8;

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_color, "");
  CHECK_NE(FLAGS_rig, "");
  CHECK_NE(FLAGS_output, "");
  if (FLAGS_height < 1 || FLAGS_height > 32768) LOG(FATAL) << "--height must be 1..32768 (got " << FLAGS_height << ")";
  if (FLAGS_num_depths < 1 || FLAGS_num_depths > 65535) LOG(FATAL) << "--num_depths must be 1..65535";

  const io::Rig full = io::loadRig(FLAGS_rig);
  io::Rig rig;
  for (int i : io::filterDestinations(full, FLAGS_cameras)) {
    rig.cams.push_back(full.cams[i]);
    rig.ids.push_back(full.ids[i]);
  }
  const int S = (int)rig.cams.size();
  int center = -1;
  if (!FLAGS_camera_id.empty()) {  // Camera::findCameraById
    for (int i = 0; i < S; ++i)
      if (rig.ids[i] == FLAGS_camera_id) center = i;
    if (center < 0) LOG(FATAL) << "Camera id " << FLAGS_camera_id << " not found";
  }

  LOG(INFO) << "Loading images...";
  double t0 = sweep_host::nowMs();
  std::vector<std::vector<float>> host(S);
  std::vector<int32_t> sizes(2 * S);
  for (int i = 0; i < S; ++i)
    host[i] = sweep_host::loadScaled(io::imagePath(FLAGS_color, rig.ids[i], FLAGS_frame), FLAGS_scale, &sizes[2 * i],
                                     &sizes[2 * i + 1]);
  const double decodeMs = sweep_host::nowMs() - t0;
  CHECK_GT(S, 0) << "no images loaded!";
  std::vector<DerpCameraDesc> cams(S);
  for (int i = 0; i < S; ++i) {
    cams[i] = sweep_host::rescaled(rig.cams[i], FLAGS_scale);
    // images(int(y), int(x)) is not clamped: a camera larger than its scaled image would read past the row
    if (cams[i].resolution[0] > sizes[2 * i] || cams[i].resolution[1] > sizes[2 * i + 1])
      LOG(FATAL) << "--scale " << FLAGS_scale << ": camera " << rig.ids[i] << " rescales to " << cams[i].resolution[0]
                 << " x " << cams[i].resolution[1] << ", larger than its scaled image " << sizes[2 * i] << " x "
                 << sizes[2 * i + 1];
  }
  std::vector<void*> dev(S);
  for (int i = 0; i < S; ++i) {
    DERP_CALL(derp_device_alloc(FLAGS_gpu, host[i].size() * sizeof(float), &dev[i]));
    DERP_CALL(derp_device_copy(FLAGS_gpu, dev[i], host[i].data(), host[i].size() * sizeof(float)));
    std::vector<float>().swap(host[i]);
  }

  const uint64_t height = FLAGS_height;
  const int n = (int)FLAGS_num_depths;
  const std::vector<float> depths = sweep_host::equirectDepths(FLAGS_num_depths, FLAGS_depth_min, FLAGS_depth_max);
  std::vector<std::string> names;
  for (float d : depths) names.push_back(sweep_host::equirectFile(d));
  const std::vector<bool> keep = sweep_host::lastOfEachName(names);
  const fs::path equirectDir = fs::path(FLAGS_output) / "equirect";
  fs::create_directories(equirectDir);

  std::vector<double> bounds;
  std::vector<uint64_t> widths(n, 2 * height);
  double deviceMs = 0;
  if (FLAGS_crop_equirect) {
    bounds.resize(4 * (size_t)n);
    const double t = sweep_host::nowMs();
    DERP_CALL(derp_sweep_crop_bounds(FLAGS_gpu, cams.data(), S, center, height, depths.data(), n, bounds.data()));
    deviceMs += sweep_host::nowMs() - t;
    for (int k = 0; k < n; ++k)
      if (derp_sweep_crop_width(height, &bounds[4 * k], &widths[k]) != 0)
        LOG(FATAL) << "depth " << depths[k] << " m: " << derp_last_error();
  }

  std::vector<const float*> images(S);
  for (int i = 0; i < S; ++i) images[i] = static_cast<const float*>(dev[i]);
  std::atomic<double> encodeMs{0};
  {
    const int threads = FLAGS_threads > 0 ? FLAGS_threads : FLAGS_threads == 0 ? 1 : (int)std::max(1u, std::thread::hardware_concurrency());
    sweep_host::Writer writer(threads);
    for (int k0 = 0; k0 < n; k0 += kSlicesPerCall) {
      const int k1 = std::min(n, k0 + kSlicesPerCall);
      std::vector<std::shared_ptr<std::vector<float>>> outs;
      std::vector<float*> ptrs;
      for (int k = k0; k < k1; ++k) {
        LOG(INFO) << "Depth " << (k + 1) << " of " << n << "...";
        outs.push_back(std::make_shared<std::vector<float>>((size_t)widths[k] * height * 4));
        ptrs.push_back(outs.back()->data());
      }
      const double t = sweep_host::nowMs();
      DERP_CALL(derp_sweep_equirect(FLAGS_gpu, cams.data(), S, center, images.data(), sizes.data(), height, &depths[k0],
                                    k1 - k0, FLAGS_crop_equirect ? &bounds[4 * k0] : nullptr, FLAGS_black_bg ? 1 : 0,
                                    ptrs.data()));
      deviceMs += sweep_host::nowMs() - t;
      for (int k = k0; k < k1; ++k) {
        if (!keep[k]) continue;
        auto out = outs[k - k0];
        const int W = (int)widths[k];
        const fs::path file = equirectDir / names[k];
        writer.submit([out, W, height, file, &encodeMs] {
          const double te = sweep_host::nowMs();
          const std::vector<uint8_t> png = sweep_host::toPng8(out->data(), (size_t)W * height);
          io::writePng8(file, png.data(), W, (int)height, 4);
          encodeMs = encodeMs + (sweep_host::nowMs() - te);
        });
      }
    }
  }
  for (void* p : dev) derp_device_free(FLAGS_gpu, p);
  LOG(INFO) << "Timing: decode " << decodeMs << " ms, device " << deviceMs << " ms, encode " << encodeMs.load()
            << " ms (summed over encoder threads), wall " << (sweep_host::nowMs() - t0) << " ms";
  return EXIT_SUCCESS;
}
