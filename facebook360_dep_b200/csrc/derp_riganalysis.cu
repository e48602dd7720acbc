// include/derp_riganalysis.h: RigAnalyzer's coverage counts on sm_90a (per-point code and proof in
// derp_riganalysis.cuh), the host resolution of the points the device leaves undecided, and the host instantiation of
// the per-point code for the CPU tests.
#include <cstring>
#include <thread>

#include "derp_host.cuh"
#include "derp_riganalysis.cuh"
#include "../../include/derp_riganalysis.h"

using namespace derp;
using namespace derp::rig;

namespace {

struct RigScratch {
  DevBuf<DevCamera> cams;
  DevBuf<double> tabs;
  DevBuf<unsigned long long> hist;
  UndecidedList<unsigned long long> undecided;  // pixel index, or distance << 32 | sample for the histogram
  DevBuf<int32_t> counts, resolvedCounts;
  DevBuf<float> timing, resolvedTiming;
};
thread_local RigScratch g_rigA;
thread_local unsigned long long g_rigHostPoints = 0;  // points the last call resolved on the host
constexpr int kThreads = 256;

// main's coverage loop: thread (j, k) counts the cameras that see distances[k] * samples[j] into hist[k][count]; one
// atomic per distinct count in the warp
__global__ void __launch_bounds__(kThreads) coverageKernel(const DevCamera* __restrict__ cams, int n,
                                                           const double* __restrict__ samples, int numSamples,
                                                           const double* __restrict__ distances,
                                                           unsigned long long* __restrict__ hist,
                                                           UndecidedView<unsigned long long> undecided) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
  if (j >= numSamples) return;
  const double d = distances[k];
  const int c = provenCount<false>(cams, n, d * samples[3 * j], d * samples[3 * j + 1], d * samples[3 * j + 2], nullptr);
  if (c < 0) undecided.append((unsigned long long)k << 32 | (unsigned)j);
  const unsigned peers = __match_any_sync(__activemask(), c);
  if (c >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1)
    atomicAdd(&hist[(size_t)k * (n + 1) + c], (unsigned long long)__popc(peers));
}

// saveEquirect's pixel (x, y): (cos(lat) cos(lon), cos(lat) sin(lon), sin(lat)) * distance from the host's tables
// tabs = {cosLat[H], sinLat[H], cosLon[W], sinLon[W]}; undecided pixels are written -1 / 0 and listed
__global__ void __launch_bounds__(kThreads) equirectKernel(const DevCamera* __restrict__ cams, int n, int W, int H,
                                                           const double* __restrict__ tabs, double distance,
                                                           int32_t* __restrict__ counts, float* __restrict__ timing,
                                                           UndecidedView<unsigned long long> undecided) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const double cl = tabs[y], sl = tabs[H + y], co = tabs[2 * H + x], so = tabs[2 * H + W + x];
  const double px = cl * co * distance, py = cl * so * distance, pz = sl * distance;
  const size_t at = (size_t)y * W + x;
  float m = 1.0f;
  const int c = timing ? provenCount<true>(cams, n, px, py, pz, &m) : provenCount<false>(cams, n, px, py, pz, nullptr);
  if (c < 0) undecided.append(at);
  counts[at] = c;
  if (timing) timing[at] = m;
}

// saveCamera's pixel (x, y) of camera `cam`: 0 outside its image circle (edge2 from the host), else the cameras that
// see the interval of cam.rig({x + .5, y + .5}, distance)
__global__ void __launch_bounds__(kThreads) cameraKernel(const DevCamera* __restrict__ cams, int n, int cam,
                                                         double edge2, int W, int H, double distance,
                                                         int32_t* __restrict__ counts,
                                                         UndecidedView<unsigned long long> undecided) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const size_t at = (size_t)y * W + x;
  const DevCamera& c = cams[cam];
  if (!c.defaultFov) {
    const double sx = (x + 0.5 - c.principal[0]) / c.focal[0], sy = (y + 0.5 - c.principal[1]) / c.focal[1];
    if (sx * sx + sy * sy >= edge2) {
      counts[at] = 0;
      return;
    }
  }
  Iv w[3];
  rigPointIv(c, x, y, distance, w);
  int total = 0;
  for (int i = 0; i < n; ++i) {
    Iv py;
    const int s = seesIv(cams[i], w, &py);
    if (s == kUndecided) {
      total = -1;
      undecided.append(at);
      break;
    }
    total += s;
  }
  counts[at] = total;
}

// saveCrossSection's point (x + .5 - .5 dim, y + .5 - .5 dim, 0), exact
__global__ void __launch_bounds__(kThreads) crossSectionKernel(const DevCamera* __restrict__ cams, int n, int dim,
                                                               int32_t* __restrict__ counts,
                                                               UndecidedView<unsigned long long> undecided) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dim) return;
  const size_t at = (size_t)y * dim + x;
  const int c = provenCount<false>(cams, n, x + 0.5 - 0.5 * dim, y + 0.5 - 0.5 * dim, 0.0, nullptr);
  if (c < 0) undecided.append(at);
  counts[at] = c;
}

// Writes the host's values of the listed pixels
__global__ void resolveKernel(const unsigned long long* __restrict__ list, const int32_t* __restrict__ c,
                              const float* __restrict__ t, int num, int32_t* counts, float* timing) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= num) return;
  counts[list[k]] = c[k];
  if (timing) timing[list[k]] = t[k];
}

// Cameras as the caller holds them, with rotation9's rotation when given
int rigCameras(const char* who, const DerpCameraDesc* cams, const double* rotation9, int n, std::vector<DevCamera>& out) {
  if (!cams || n < 1) return fail(DERP_EINVAL, std::string(who) + ": at least one camera is required");
  out.resize(n);
  for (int i = 0; i < n; ++i) {
    if (!host::makeCamera(cams[i], &out[i])) return fail(DERP_EINVAL, std::string(who) + ": invalid camera " + std::to_string(i));
    if (rotation9)
      for (int k = 0; k < 9; ++k) out[i].rot[k] = rotation9[9 * i + k];
  }
  return DERP_OK;
}

int checkGrid(const char* who, long long w, long long h) {
  if (w < 1 || h < 1 || h > 65535 || w * h >= (1ll << 31))
    return fail(DERP_EINVAL, std::string(who) + ": the grid must have 1..65535 rows and fewer than 2^31 points");
  return DERP_OK;
}

// The equirect's sample tables {cosLat[H], sinLat[H], cosLon[W], sinLon[W]} (RigAnalyzer.cpp:393-397)
std::vector<double> equirectTables(int W, int H) {
  std::vector<double> t(2 * (size_t)H + 2 * (size_t)W);
  for (int y = 0; y < H; ++y) {
    const double lat = M_PI / 2 - (y + 0.5) / H * M_PI;
    t[y] = cos(lat);
    t[H + y] = sin(lat);
  }
  for (int x = 0; x < W; ++x) {
    const double lon = -M_PI + (x + 0.5) / W * 2 * M_PI;
    t[2 * H + x] = cos(lon);
    t[2 * H + W + x] = sin(lon);
  }
  return t;
}

// Writes the host's values c (and t) of the listed pixels into the device planes
int resolvePixels(const std::vector<unsigned long long>& list, const std::vector<int32_t>& c,
                  const std::vector<float>* t, int32_t* counts, float* timing) {
  if (list.empty()) return DERP_OK;
  RigScratch& g = g_rigA;
  if (int rc = upload(g.resolvedCounts, c.data(), c.size())) return rc;
  if (t)
    if (int rc = upload(g.resolvedTiming, t->data(), t->size())) return rc;
  resolveKernel<<<grid1(list.size()), 256>>>(g.undecided.items.p, g.resolvedCounts.p,
                                             t ? g.resolvedTiming.p : nullptr, (int)list.size(), counts, timing);
  CU(cudaGetLastError());
  return DERP_OK;
}

int uploadCams(const std::vector<DevCamera>& c) { return upload(g_rigA.cams, c.data(), c.size()); }

// ---- test probes: the proofs' device functions on caller-given inputs ------------------------------------------------
// The device's math function `fn` (derp_test_math) and its interval as the proofs widen it
__global__ void mathProbeKernel(int fn, const double* a, const double* b, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double v;
  Iv w;
  switch (fn) {
    case DERP_MATH_SIN: w = widenD(v = sin(a[i]), kSinUlps, 0); break;
    case DERP_MATH_COS: w = widenD(v = cos(a[i]), kSinUlps, 0); break;
    case DERP_MATH_ATAN: w = widenD(v = atan(a[i]), kAtanUlps, 0); break;
    case DERP_MATH_ASIN: w = widenD(v = asin(a[i]), kAtanUlps, 0); break;
    case DERP_MATH_ATAN2: w = widenD(v = atan2(a[i], b[i]), kAtan2Ulps, 0); break;
    case DERP_MATH_ACOSF: {
      const float f = acosf((float)a[i]);
      w = widenF(f, kAcosfUlps);
      v = f;
      break;
    }
    case DERP_MATH_ATAN2F: {
      const float f = atan2f((float)a[i], (float)b[i]);
      w = widenF(f, kAtan2fUlps);
      v = f;
      break;
    }
    default: w = Iv{v = atan2Pos(a[i], b[i]), v}; break;
  }
  out[3 * i] = v;
  out[3 * i + 1] = w.lo;
  out[3 * i + 2] = w.hi;
}

// Every float x in [first, first + count) (bit patterns) against the host's acosf(x) and acos(double(x)) (ref): the
// greatest device and host errors in ulps of ref (x 2^20), the greatest distance in float steps between the two, and
// the number of host values outside widenF of the device's
__global__ void acosfCheckKernel(uint32_t first, uint32_t count, const float* __restrict__ host,
                                 const double* __restrict__ ref, unsigned* stats) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned devErr = 0, hostErr = 0, steps = 0, outside = 0;
  if (i < count) {
    const float x = __uint_as_float(first + i), d = acosf(x), h = host[i];
    const double r = ref[i];
    int e;
    frexp(r, &e);
    const double ulp = ldexp(1.0, max(e - 24, -149));
    devErr = (unsigned)fmin(fabs(d - r) / ulp * 0x1p20, 4294967295.0);
    hostErr = (unsigned)fmin(fabs(h - r) / ulp * 0x1p20, 4294967295.0);
    const int bd = __float_as_int(d), bh = __float_as_int(h);  // acos >= 0: bit patterns order the values
    steps = (unsigned)abs(bd - bh);
    const Iv w = widenF(d, kAcosfUlps);
    outside = !(w.lo <= h && h <= w.hi);
  }
  const unsigned m = __activemask();
  devErr = __reduce_max_sync(m, devErr);
  hostErr = __reduce_max_sync(m, hostErr);
  steps = __reduce_max_sync(m, steps);
  outside = __reduce_add_sync(m, outside);
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&stats[0], devErr);
    atomicMax(&stats[1], hostErr);
    atomicMax(&stats[2], steps);
    atomicAdd(&stats[3], outside);
  }
}

__global__ void rigPointIvKernel(DevCamera c, const int32_t* pix, int n, double depth, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Iv w[3];
  rigPointIv(c, pix[2 * i], pix[2 * i + 1], depth, w);
  for (int k = 0; k < 3; ++k) {
    out[7 * i + 2 * k] = w[k].lo;
    out[7 * i + 2 * k + 1] = w[k].hi;
  }
  const double sx = (pix[2 * i] + 0.5 - c.principal[0]) / c.focal[0];
  const double sy = (pix[2 * i + 1] + 0.5 - c.principal[1]) / c.focal[1];
  out[7 * i + 6] = undistort(c, sqrt(sx * sx + sy * sy));
}

__global__ void seesIvKernel(DevCamera c, const double* box, int n, int32_t* decision, double* py) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Iv w[3] = {{box[6 * i], box[6 * i + 1]}, {box[6 * i + 2], box[6 * i + 3]}, {box[6 * i + 4], box[6 * i + 5]}};
  Iv y{NAN, NAN};
  decision[i] = seesIv(c, w, &y);
  py[2 * i] = y.lo;
  py[2 * i + 1] = y.hi;
}

__global__ void seesKernel(DevCamera c, const double* pts, int n, double* pix, uint8_t* seen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double x = NAN, y = NAN;
  seen[i] = sees(c, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], &x, &y);
  pix[2 * i] = x;
  pix[2 * i + 1] = y;
}

__global__ void provenCountKernel(const DevCamera* cams, int num, const double* pts, int n, int32_t* counts,
                                  float* timing) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float m = NAN;
  counts[i] = provenCount<true>(cams, num, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], &m);
  timing[i] = m;
}

int probeCamera(const DerpCameraDesc* d, DevCamera* c) {
  if (!d || !host::makeCamera(*d, c)) return fail(DERP_EINVAL, "invalid camera");
  return DERP_OK;
}

// Copies n elements of a device buffer to the caller's host array
template <typename T>
int download(T* dst, const DevBuf<T>& src, size_t n) {
  CU(cudaGetLastError());
  CU(cudaMemcpy(dst, src.p, n * sizeof(T), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

}  // namespace

extern "C" {

int derp_rig_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                      const double* samples, int num_samples, const double* distances, int num_distances,
                      uint64_t* hist) {
  static const char* who = "derp_rig_coverage";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (!samples || !distances || !hist || num_samples < 1 || num_distances < 1 || num_distances > 65535)
    return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  CU(cudaSetDevice(device));
  RigScratch& g = g_rigA;
  if (int rc = uploadCams(c)) return rc;
  if (int rc = upload(g.tabs, samples, 3 * (size_t)num_samples)) return rc;
  DevBuf<double> dist;
  if (int rc = upload(dist, distances, num_distances)) return rc;
  const size_t nh = (size_t)num_distances * (num_cams + 1);
  CU(g.hist.ensure(nh));
  CU(cudaMemset(g.hist.p, 0, nh * sizeof(unsigned long long)));
  std::vector<unsigned long long> list;
  const dim3 grid(grid1(num_samples, kThreads), num_distances);
  auto run = [&](UndecidedView<unsigned long long> undecided) {
    CU(cudaMemset(g.hist.p, 0, nh * sizeof(unsigned long long)));
    coverageKernel<<<grid, kThreads>>>(g.cams.p, num_cams, g.tabs.p, num_samples, dist.p, g.hist.p, undecided);
    return DERP_OK;
  };
  if (int rc = g.undecided.collect(run, list)) return rc;
  g_rigHostPoints = list.size();
  std::vector<unsigned long long> h(nh);
  CU(cudaMemcpy(h.data(), g.hist.p, nh * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  for (unsigned long long e : list) {
    const int k = (int)(e >> 32), j = (int)(unsigned)e;
    const double d = distances[k];
    ++h[(size_t)k * (num_cams + 1) + countSees(c.data(), num_cams, d * samples[3 * j], d * samples[3 * j + 1],
                                               d * samples[3 * j + 2])];
  }
  CU(cudaMemcpy(hist, h.data(), nh * sizeof(uint64_t), cudaMemcpyDefault));
  return DERP_OK;
}

int derp_rig_equirect_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int width,
                               int height, double distance, int32_t* counts, float* min_timing) {
  static const char* who = "derp_rig_equirect_coverage";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (int rc = checkGrid(who, width, height)) return rc;
  if (!counts) return fail(DERP_EINVAL, std::string(who) + ": counts is required");
  CU(cudaSetDevice(device));
  RigScratch& g = g_rigA;
  if (int rc = uploadCams(c)) return rc;
  const std::vector<double> tabs = equirectTables(width, height);
  if (int rc = upload(g.tabs, tabs.data(), tabs.size())) return rc;
  const size_t np = (size_t)width * height;
  int32_t* dc = counts;
  float* dt = min_timing;
  if (int rc = outBuffer(dc, np, g.counts)) return rc;
  if (dt)
    if (int rc = outBuffer(dt, np, g.timing)) return rc;
  std::vector<unsigned long long> list;
  const dim3 grid(grid1(width, kThreads), height);
  auto run = [&](UndecidedView<unsigned long long> undecided) {
    equirectKernel<<<grid, kThreads>>>(g.cams.p, num_cams, width, height, g.tabs.p, distance, dc, dt, undecided);
    return DERP_OK;
  };
  if (int rc = g.undecided.collect(run, list)) return rc;
  g_rigHostPoints = list.size();
  std::vector<int32_t> rc(list.size());
  std::vector<float> rt(list.size()), scratch(num_cams);
  for (size_t k = 0; k < list.size(); ++k) {
    const int x = (int)(list[k] % width), y = (int)(list[k] / width);
    const double cl = tabs[y], sl = tabs[height + y], co = tabs[2 * height + x], so = tabs[2 * height + width + x];
    double m;
    rc[k] = countTiming(c.data(), num_cams, cl * co * distance, cl * so * distance, sl * distance, scratch.data(), &m);
    rt[k] = (float)m;
  }
  if (int e = resolvePixels(list, rc, dt ? &rt : nullptr, dc, dt)) return e;
  if (int e = stageOut(counts, dc, np)) return e;
  if (dt)
    if (int e = stageOut(min_timing, dt, np)) return e;
  return DERP_OK;
}

int derp_rig_camera_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int cam,
                             double distance, int32_t* counts) {
  static const char* who = "derp_rig_camera_coverage";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (cam < 0 || cam >= num_cams || !counts) return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  const int W = (int)c[cam].res[0], H = (int)c[cam].res[1];  // kDimX = int(resolution.x())
  if (int rc = checkGrid(who, W, H)) return rc;
  const double edge2 = c[cam].defaultFov ? 0 : imageCircleEdge2(c[cam]);
  CU(cudaSetDevice(device));
  RigScratch& g = g_rigA;
  if (int rc = uploadCams(c)) return rc;
  const size_t np = (size_t)W * H;
  int32_t* dc = counts;
  if (int rc = outBuffer(dc, np, g.counts)) return rc;
  std::vector<unsigned long long> list;
  const dim3 grid(grid1(W, kThreads), H);
  auto run = [&](UndecidedView<unsigned long long> undecided) {
    cameraKernel<<<grid, kThreads>>>(g.cams.p, num_cams, cam, edge2, W, H, distance, dc, undecided);
    return DERP_OK;
  };
  if (int rc = g.undecided.collect(run, list)) return rc;
  g_rigHostPoints = list.size();
  std::vector<int32_t> rc(list.size());
  for (size_t k = 0; k < list.size(); ++k)
    rc[k] = countCameraPixel(c.data(), num_cams, cam, edge2, (int)(list[k] % W), (int)(list[k] / W), distance);
  if (int e = resolvePixels(list, rc, nullptr, dc, nullptr)) return e;
  return stageOut(counts, dc, np);
}

int derp_rig_cross_section(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int dim,
                           int32_t* counts) {
  static const char* who = "derp_rig_cross_section";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (int rc = checkGrid(who, dim, dim)) return rc;
  if (!counts) return fail(DERP_EINVAL, std::string(who) + ": counts is required");
  CU(cudaSetDevice(device));
  RigScratch& g = g_rigA;
  if (int rc = uploadCams(c)) return rc;
  const size_t np = (size_t)dim * dim;
  int32_t* dc = counts;
  if (int rc = outBuffer(dc, np, g.counts)) return rc;
  std::vector<unsigned long long> list;
  const dim3 grid(grid1(dim, kThreads), dim);
  auto run = [&](UndecidedView<unsigned long long> undecided) {
    crossSectionKernel<<<grid, kThreads>>>(g.cams.p, num_cams, dim, dc, undecided);
    return DERP_OK;
  };
  if (int rc = g.undecided.collect(run, list)) return rc;
  g_rigHostPoints = list.size();
  std::vector<int32_t> rc(list.size());
  for (size_t k = 0; k < list.size(); ++k)
    rc[k] = countSees(c.data(), num_cams, (int)(list[k] % dim) + 0.5 - 0.5 * dim, (int)(list[k] / dim) + 0.5 - 0.5 * dim,
                      0.0);
  if (int e = resolvePixels(list, rc, nullptr, dc, nullptr)) return e;
  return stageOut(counts, dc, np);
}

uint64_t derp_rig_analysis_last_host_points(void) { return g_rigHostPoints; }

int derp_test_rig_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                                const double* samples, int num_samples, const double* distances, int num_distances,
                                uint64_t* hist) {
  std::vector<DevCamera> c;
  if (int rc = rigCameras("derp_test_rig_coverage_host", cams, rotation9, num_cams, c)) return rc;
  if (!samples || !distances || !hist || num_samples < 1 || num_distances < 1) return fail(DERP_EINVAL, "bad arguments");
  std::fill(hist, hist + (size_t)num_distances * (num_cams + 1), 0);
  for (int k = 0; k < num_distances; ++k)
    for (int j = 0; j < num_samples; ++j) {
      const double d = distances[k];
      ++hist[(size_t)k * (num_cams + 1) +
             countSees(c.data(), num_cams, d * samples[3 * j], d * samples[3 * j + 1], d * samples[3 * j + 2])];
    }
  return DERP_OK;
}

int derp_test_rig_equirect_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int width,
                                         int height, double distance, int32_t* counts, float* min_timing) {
  static const char* who = "derp_test_rig_equirect_coverage_host";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (int rc = checkGrid(who, width, height)) return rc;
  if (!counts) return fail(DERP_EINVAL, std::string(who) + ": counts is required");
  const std::vector<double> t = equirectTables(width, height);
  std::vector<float> scratch(num_cams);
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      const double cl = t[y], sl = t[height + y], co = t[2 * height + x], so = t[2 * height + width + x];
      double m;
      const size_t at = (size_t)y * width + x;
      counts[at] = countTiming(c.data(), num_cams, cl * co * distance, cl * so * distance, sl * distance,
                               scratch.data(), &m);
      if (min_timing) min_timing[at] = (float)m;
    }
  return DERP_OK;
}

int derp_test_rig_camera_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int cam,
                                       double distance, int32_t* counts) {
  static const char* who = "derp_test_rig_camera_coverage_host";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (cam < 0 || cam >= num_cams || !counts) return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  const int W = (int)c[cam].res[0], H = (int)c[cam].res[1];
  if (int rc = checkGrid(who, W, H)) return rc;
  const double edge2 = c[cam].defaultFov ? 0 : imageCircleEdge2(c[cam]);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) counts[(size_t)y * W + x] = countCameraPixel(c.data(), num_cams, cam, edge2, x, y, distance);
  return DERP_OK;
}

int derp_test_rig_cross_section_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int dim,
                                     int32_t* counts) {
  static const char* who = "derp_test_rig_cross_section_host";
  std::vector<DevCamera> c;
  if (int rc = rigCameras(who, cams, rotation9, num_cams, c)) return rc;
  if (int rc = checkGrid(who, dim, dim)) return rc;
  if (!counts) return fail(DERP_EINVAL, std::string(who) + ": counts is required");
  for (int y = 0; y < dim; ++y)
    for (int x = 0; x < dim; ++x)
      counts[(size_t)y * dim + x] = countSees(c.data(), num_cams, x + 0.5 - 0.5 * dim, y + 0.5 - 0.5 * dim, 0.0);
  return DERP_OK;
}

int derp_test_math(int device, int fn, const double* a, const double* b, int n, double* out) {
  const bool two = fn == DERP_MATH_ATAN2 || fn == DERP_MATH_ATAN2F || fn == DERP_MATH_ATAN2POS;
  if (fn < DERP_MATH_SIN || fn > DERP_MATH_ATAN2POS || !a || (two && !b) || n < 1 || !out)
    return fail(DERP_EINVAL, "derp_test_math: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<double> da, db, dout;
  if (int rc = upload(da, a, n)) return rc;
  if (two)
    if (int rc = upload(db, b, n)) return rc;
  CU(dout.ensure(3 * (size_t)n));
  mathProbeKernel<<<grid1(n), 256>>>(fn, da.p, db.p, n, dout.p);
  return download(out, dout, 3 * (size_t)n);
}

int derp_test_acosf_exhaustive(int device, uint32_t* stats) {
  if (!stats) return fail(DERP_EINVAL, "derp_test_acosf_exhaustive: bad arguments");
  CU(cudaSetDevice(device));
  constexpr uint32_t kChunk = 1u << 25;
  DevBuf<float> dh;
  DevBuf<double> dr;
  DevBuf<unsigned> ds;
  CU(dh.ensure(kChunk));
  CU(dr.ensure(kChunk));
  CU(ds.ensure(4));
  CU(cudaMemset(ds.p, 0, 4 * sizeof(unsigned)));
  std::vector<float> h(kChunk);
  std::vector<double> r(kChunk);
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  for (const uint32_t sign : {0u, 0x80000000u})  // [+0, 1] and [-0, -1]: bit patterns up to 1.0f's
    for (uint32_t first = 0; first <= 0x3f800000u; first += kChunk) {
      const uint32_t count = std::min<uint32_t>(kChunk, 0x3f800001u - first);
      std::vector<std::thread> pool;
      for (unsigned t = 0; t < nt; ++t)
        pool.emplace_back([&, t] {
          for (uint32_t i = t; i < count; i += nt) {
            const uint32_t bits = (sign | first) + i;
            float x;
            memcpy(&x, &bits, 4);
            h[i] = acosf(x);
            r[i] = acos((double)x);
          }
        });
      for (auto& p : pool) p.join();
      CU(cudaMemcpy(dh.p, h.data(), count * sizeof(float), cudaMemcpyHostToDevice));
      CU(cudaMemcpy(dr.p, r.data(), count * sizeof(double), cudaMemcpyHostToDevice));
      acosfCheckKernel<<<grid1(count), 256>>>(sign | first, count, dh.p, dr.p, ds.p);
    }
  return download(stats, ds, 4);
}

int derp_test_rig_point_iv(int device, const DerpCameraDesc* cam, const int32_t* pix, int n, double depth, double* out) {
  DevCamera c;
  if (int rc = probeCamera(cam, &c)) return rc;
  if (!pix || n < 1 || !out) return fail(DERP_EINVAL, "derp_test_rig_point_iv: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<int32_t> dp;
  DevBuf<double> dout;
  if (int rc = upload(dp, pix, 2 * (size_t)n)) return rc;
  CU(dout.ensure(7 * (size_t)n));
  rigPointIvKernel<<<grid1(n), 256>>>(c, dp.p, n, depth, dout.p);
  return download(out, dout, 7 * (size_t)n);
}

int derp_test_sees_iv(int device, const DerpCameraDesc* cam, const double* boxes, int n, int32_t* decision,
                      double* py) {
  DevCamera c;
  if (int rc = probeCamera(cam, &c)) return rc;
  if (!boxes || n < 1 || !decision || !py) return fail(DERP_EINVAL, "derp_test_sees_iv: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<double> db, dy;
  DevBuf<int32_t> dd;
  if (int rc = upload(db, boxes, 6 * (size_t)n)) return rc;
  CU(dd.ensure(n));
  CU(dy.ensure(2 * (size_t)n));
  seesIvKernel<<<grid1(n), 256>>>(c, db.p, n, dd.p, dy.p);
  if (int rc = download(decision, dd, n)) return rc;
  return download(py, dy, 2 * (size_t)n);
}

int derp_test_sees_device(int device, const DerpCameraDesc* cam, const double* pts, int n, double* pix, uint8_t* seen) {
  DevCamera c;
  if (int rc = probeCamera(cam, &c)) return rc;
  if (!pts || n < 1 || !pix || !seen) return fail(DERP_EINVAL, "derp_test_sees_device: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<double> dp, dx;
  DevBuf<uint8_t> ds;
  if (int rc = upload(dp, pts, 3 * (size_t)n)) return rc;
  CU(dx.ensure(2 * (size_t)n));
  CU(ds.ensure(n));
  seesKernel<<<grid1(n), 256>>>(c, dp.p, n, dx.p, ds.p);
  if (int rc = download(pix, dx, 2 * (size_t)n)) return rc;
  return download(seen, ds, n);
}

int derp_test_proven_count(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                           const double* pts, int n, int32_t* counts, float* timing) {
  std::vector<DevCamera> c;
  if (int rc = rigCameras("derp_test_proven_count", cams, rotation9, num_cams, c)) return rc;
  if (!pts || n < 1 || !counts || !timing) return fail(DERP_EINVAL, "derp_test_proven_count: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<DevCamera> dc;
  DevBuf<double> dp;
  DevBuf<int32_t> dn;
  DevBuf<float> dt;
  if (int rc = upload(dc, c.data(), c.size())) return rc;
  if (int rc = upload(dp, pts, 3 * (size_t)n)) return rc;
  CU(dn.ensure(n));
  CU(dt.ensure(n));
  provenCountKernel<<<grid1(n), 256>>>(dc.p, num_cams, dp.p, n, dn.p, dt.p);
  if (int rc = download(counts, dn, n)) return rc;
  return download(timing, dt, n);
}

int derp_test_count_timing_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, const double* pts,
                                int n, int32_t* counts, float* timing) {
  std::vector<DevCamera> c;
  if (int rc = rigCameras("derp_test_count_timing_host", cams, rotation9, num_cams, c)) return rc;
  if (!pts || n < 1 || !counts || !timing) return fail(DERP_EINVAL, "derp_test_count_timing_host: bad arguments");
  std::vector<float> scratch(num_cams);
  for (int i = 0; i < n; ++i) {
    double m;
    counts[i] = countTiming(c.data(), num_cams, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], scratch.data(), &m);
    timing[i] = (float)m;
  }
  return DERP_OK;
}

}  // extern "C"
