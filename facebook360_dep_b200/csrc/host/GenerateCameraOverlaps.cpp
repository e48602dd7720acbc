// GenerateCameraOverlaps — drop-in for source/render/GenerateCameraOverlaps.cpp.  For each destination camera and each
// of --num_depths disparities (the brute-force sweep's probeDisparity table), every pixel is projected to that depth and
// coloured with the mean bilinear colour of every camera that sees the point.  The slices are computed in libderp_b200.so
// (derp_sweep_overlaps, csrc/derp_sweepview.cuh); PNGs are encoded on host threads while the next slices run.  See
// INTEGRATION.md for what differs from the reference (no depth label, refusals where the reference is undefined).
#include "../../../include/derp_sweepview.h"
#include "io.h"
#include "sweep_host.h"

const std::string kUsage = R"(
   - Generates a series of images of the rig cameras projected into destination cameras over
   a series of fixed depths.

   - Example:
     ./GenerateCameraOverlaps \
     --frame=000000 \
     --output=/path/to/output \
     --rig=/path/to/rigs/rig.json \
     --color=/path/to/video/color
 )";

DEFINE_string(cameras, "", "cameras to render (comma-separated)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_string(frame, "000000", "frame to process (lexical)");
DEFINE_uint64(max_depth_m, 10, "max depth in cm");
DEFINE_uint64(min_depth_m, 1, "min depth in cm");
DEFINE_uint64(num_depths, 50, "num depths");
DEFINE_string(output, "", "path to output directory (required)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_double(scale, 0.5, "image scale factor");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                 \
  do {                                                                  \
    const int rc_ = (expr);                                             \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

constexpr int kSlicesPerCall = 8;  // host buffer per call: 8 slices of one destination

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_color, "");
  CHECK_NE(FLAGS_rig, "");
  CHECK_NE(FLAGS_output, "");
  // probeDisparity divides 0 by 0 for one slice, and int(NaN) would name its file
  if (FLAGS_num_depths < 2) LOG(FATAL) << "--num_depths must be at least 2 (got " << FLAGS_num_depths << ")";
  if (FLAGS_num_depths > 100000) LOG(FATAL) << "--num_depths must be at most 100000";

  const io::Rig rig = io::loadRig(FLAGS_rig);
  const int S = (int)rig.cams.size();
  std::vector<DerpCameraDesc> cams(S);
  for (int i = 0; i < S; ++i) cams[i] = sweep_host::rescaled(rig.cams[i], FLAGS_scale);
  const std::vector<int> dsts = io::filterDestinations(rig, FLAGS_cameras);
  CHECK_GT(dsts.size(), 0u) << "no destinations!";

  LOG(INFO) << "Loading images...";
  double t0 = sweep_host::nowMs();
  std::vector<void*> dev(S);
  std::vector<int32_t> sizes(2 * S);
  for (int i = 0; i < S; ++i) {
    int w, h;
    const std::vector<float> img =
        sweep_host::loadScaled(io::imagePath(FLAGS_color, rig.ids[i], FLAGS_frame), FLAGS_scale, &w, &h);
    sizes[2 * i] = w;
    sizes[2 * i + 1] = h;
    DERP_CALL(derp_device_alloc(FLAGS_gpu, img.size() * sizeof(float), &dev[i]));
    DERP_CALL(derp_device_copy(FLAGS_gpu, dev[i], img.data(), img.size() * sizeof(float)));
  }
  const double decodeMs = sweep_host::nowMs() - t0;

  const fs::path overlapsDir = fs::path(FLAGS_output) / "overlaps";
  for (int d : dsts) fs::create_directories(overlapsDir / rig.ids[d]);
  const int n = (int)FLAGS_num_depths;
  const std::vector<float> disps = sweep_host::overlapDisparities(FLAGS_num_depths, FLAGS_min_depth_m, FLAGS_max_depth_m);
  std::vector<std::string> names;
  for (float d : disps) names.push_back(sweep_host::overlapFile(d));
  const std::vector<bool> keep = sweep_host::lastOfEachName(names);

  std::vector<const float*> images(S);
  for (int i = 0; i < S; ++i) images[i] = static_cast<const float*>(dev[i]);
  std::atomic<double> encodeMs{0};
  double deviceMs = 0;
  {
    sweep_host::Writer writer(std::max(1u, std::thread::hardware_concurrency()));
    for (int k0 = 0; k0 < n; k0 += kSlicesPerCall) {
      const int k1 = std::min(n, k0 + kSlicesPerCall);
      for (int k = k0; k < k1; ++k) LOG(INFO) << "Depth " << (k + 1) << " of " << n << "...";
      for (int d : dsts) {
        const int W = (int)cams[d].resolution[0], H = (int)cams[d].resolution[1];
        const size_t plane = (size_t)W * H;
        auto out = std::make_shared<std::vector<float>>(plane * 4 * (k1 - k0));
        const double t = sweep_host::nowMs();
        DERP_CALL(derp_sweep_overlaps(FLAGS_gpu, cams.data(), S, images.data(), sizes.data(), d, &disps[k0], k1 - k0,
                                      out->data()));
        deviceMs += sweep_host::nowMs() - t;
        for (int k = k0; k < k1; ++k) {
          if (!keep[k]) continue;
          const fs::path file = overlapsDir / rig.ids[d] / names[k];
          writer.submit([out, k, k0, plane, W, H, file, &encodeMs] {
            const double te = sweep_host::nowMs();
            const std::vector<uint8_t> png = sweep_host::toPng8(out->data() + (size_t)(k - k0) * plane * 4, plane);
            io::writePng8(file, png.data(), W, H, 4);
            encodeMs = encodeMs + (sweep_host::nowMs() - te);
          });
        }
      }
    }
  }
  for (void* p : dev) derp_device_free(FLAGS_gpu, p);
  LOG(INFO) << "Timing: decode " << decodeMs << " ms, device " << deviceMs << " ms, encode " << encodeMs.load()
            << " ms (summed over encoder threads), wall " << (sweep_host::nowMs() - t0) << " ms";
  return EXIT_SUCCESS;
}
