// Host steps shared by GenerateCameraOverlaps and GenerateEquirect: the scaled colour loader, the slice tables, the
// file names and the 8-bit conversion of the written slices, each in the reference's arithmetic.
#pragma once

#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "area_resize.h"
#include "io.h"

namespace sweep_host {

// image_util::loadScaledImages<Vec4f> (ImageUtil.h:126-141, CvUtil.h:151-154): loadImage<Vec4f>, then INTER_AREA to
// round(w * scale) x round(h * scale); an image of that size already is returned unchanged.
inline std::vector<float> loadScaled(const fs::path& path, double scale, int* w, int* h) {
  int sw, sh;
  std::vector<float> img = io::loadColorF32x4(path, &sw, &sh);
  const int dw = (int)std::round(sw * scale), dh = (int)std::round(sh * scale);
  CHECK(dw > 0 && dh > 0) << "--scale " << scale << " leaves " << path.string() << " with no pixels";
  *w = dw;
  *h = dh;
  if (dw == sw && dh == sh) return img;
  std::vector<float> out((size_t)dw * dh * 4);
  io::area::resize(img.data(), sw, sh, 4, out.data(), dw, dh);
  return out;
}

// GenerateCameraOverlaps' slices: float(probeDisparity(d, n, 1.0f / min_depth_m, 1.0f / max_depth_m))
// (GenerateCameraOverlaps.cpp:100-103, ImageUtil.cpp:100-107); the uint64 flags divide in fp32
inline std::vector<float> overlapDisparities(uint64_t n, uint64_t minDepth, uint64_t maxDepth) {
  const float minDisparity = 1.0f / minDepth, maxDisparity = 1.0f / maxDepth;
  std::vector<float> out;
  for (int d = 0; d < (int)n; ++d) {
    const double fraction = double(d) / double(int(n) - 1);
    out.push_back((float)(fraction * (double)minDisparity + (1 - fraction) * (double)maxDisparity));
  }
  return out;
}

// "<cam>/<NNNNN>_cm.png" with int(depthCm), depthCm = (1.0f / disparity) * 100 in fp32
inline std::string overlapFile(float disparity) {
  const float depth = 1.0f / disparity;
  const float depthCm = depth * 100;
  char b[64];
  std::snprintf(b, sizeof b, "%05d_cm.png", int(depthCm));
  return b;
}

// GenerateEquirect's depths in slice order i = n - 1 .. 0 (GenerateEquirect.cpp:264-272)
inline std::vector<float> equirectDepths(uint64_t n, double depthMin, double depthMax) {
  const float dispMin = 1.0f / depthMax, dispMax = 1.0f / depthMin;
  std::vector<float> out;
  for (int i = int(n) - 1; i >= 0; --i) {
    const float fraction = float(i) / float(n - 1);
    const float disp = n == 1 ? dispMin : fraction * dispMin + (1 - fraction) * dispMax;
    out.push_back(1.0f / disp);
  }
  return out;
}

// "<NNNNN>_cm.png" with int(depth * 100) in fp64 (saveImage takes a double, GenerateEquirect.cpp:58-76)
inline std::string equirectFile(float depth) {
  const double d = depth;
  char b[64];
  std::snprintf(b, sizeof b, "%05d_cm.png", int(d * 100));
  return b;
}

// imwrite(filename, 255.0f * image) of a float B, G, R, A image: the fp32 product, then convertTo(CV_8U) (round half
// to even, saturate; NaN and +-inf become 0 through cvRound's INT_MIN)
inline std::vector<uint8_t> toPng8(const float* bgra, size_t n) {
  std::vector<uint8_t> out(n * 4);
  for (size_t i = 0; i < n * 4; ++i) out[i] = io::saturateU8(255.0f * bgra[i]);
  return out;
}

// The camera after Camera::rescale({w, h}) (Camera.cpp:217-223): principal and focal times newResolution / resolution
// per axis
inline DerpCameraDesc rescaledTo(const DerpCameraDesc& in, double w, double h) {
  DerpCameraDesc d = in;
  const double nr[2] = {w, h};
  for (int i = 0; i < 2; ++i) {
    const double p = in.has_principal ? in.principal[i] : in.resolution[i] / 2;
    d.principal[i] = p * (nr[i] / in.resolution[i]);
    d.focal[i] = in.focal[i] * (nr[i] / in.resolution[i]);
    d.resolution[i] = nr[i];
  }
  d.has_principal = 1;
  return d;
}

// ProjectEquirectsToCameras' rescaleCameras at --width > 0: height = ceil(width * res.y / float(res.x)), rounded up to
// even, then Camera::rescale({width, height})
inline DerpCameraDesc rescaledToWidth(const DerpCameraDesc& c, int width) {
  int height = std::ceil(width * c.resolution[1] / float(c.resolution[0]));
  height += height % 2;  // force even number of rows
  return rescaledTo(c, width, height);
}

// The camera as the apps hold it after Camera::rescale(resolution * scale)
inline DerpCameraDesc rescaled(const DerpCameraDesc& in, double scale) {
  return rescaledTo(in, in.resolution[0] * scale, in.resolution[1] * scale);
}

// For slices written in index order: keep[k] is false when a later slice has the same file name (it would overwrite k)
inline std::vector<bool> lastOfEachName(const std::vector<std::string>& names) {
  std::vector<bool> keep(names.size(), true);
  for (size_t k = 0; k < names.size(); ++k)
    for (size_t j = k + 1; j < names.size(); ++j)
      if (names[j] == names[k]) keep[k] = false;
  return keep;
}

// PNG encoding on host threads, overlapped with the next slices' kernels.  Each job owns one file (see lastOfEachName).
class Writer {
 public:
  explicit Writer(int threads) {
    for (int i = 0; i < threads; ++i) pool_.emplace_back([this] { run(); });
  }
  ~Writer() { join(); }
  void submit(std::function<void()> job) {
    std::unique_lock<std::mutex> l(m_);
    full_.wait(l, [this] { return q_.size() < 2 * pool_.size(); });
    q_.push_back(std::move(job));
    cv_.notify_one();
  }
  void join() {
    {
      std::lock_guard<std::mutex> l(m_);
      done_ = true;
    }
    cv_.notify_all();
    for (auto& t : pool_)
      if (t.joinable()) t.join();
    pool_.clear();
  }

 private:
  void run() {
    for (;;) {
      std::function<void()> job;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [this] { return done_ || !q_.empty(); });
        if (q_.empty()) return;
        job = std::move(q_.front());
        q_.pop_front();
        full_.notify_one();
      }
      job();
    }
  }
  std::vector<std::thread> pool_;
  std::deque<std::function<void()>> q_;
  std::mutex m_;
  std::condition_variable cv_, full_;
  bool done_ = false;
};

inline double nowMs() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace sweep_host
