// include/derp_sweepview.h: the rig's constant-depth sweep slices on sm_90a (derp_sweepview.cuh), and the host
// instantiation of their per-pixel code for the CPU tests.
#include "derp_host.cuh"
#include "derp_sweepview.cuh"
#include "../../include/derp_sweepview.h"

using namespace derp;

namespace {
using derp::sweep::SrcImage;

struct SweepScratch {
  DevBuf<DevCamera> cams;
  DevBuf<SrcImage> imgs;
  DevBuf<float4> upload, out;
  DevBuf<double> tabs;
  DevBuf<float> depths;
  DevBuf<int> widths, box;
  DevBuf<float4*> outs;
  DevBuf<unsigned long long> hits;
};
thread_local SweepScratch g_sweep;
thread_local unsigned long long g_sweepHits = 0;  // contributing (sample, camera) pairs of the last call

// Cameras as the apps hold them (already rescaled), optionally centred on camera `center`
int sweepCameras(const char* who, const DerpCameraDesc* cams, int n, int center, std::vector<DevCamera>& out) {
  const std::string name(who);
  if (!cams || n < 1 || n > derp::sweep::kMaxCams)
    return fail(DERP_EINVAL, name + ": between 1 and " + std::to_string(derp::sweep::kMaxCams) + " cameras");
  std::vector<DerpCameraDesc> d(cams, cams + n);
  if (center >= n) return fail(DERP_EINVAL, name + ": center index out of range");
  if (center >= 0 && !derp::sweep::host::centerRig(d.data(), n, center))
    return fail(DERP_EINVAL, name + ": centerRig produced an invalid rotation");
  out.resize(n);
  for (int i = 0; i < n; ++i)
    if (!host::makeCamera(d[i], &out[i])) return fail(DERP_EINVAL, name + ": invalid camera " + std::to_string(i));
  return DERP_OK;
}

int checkImages(const char* who, const float* const* images, const int32_t* sizes, int n) {
  if (!images || !sizes) return fail(DERP_EINVAL, std::string(who) + ": images and sizes are required");
  for (int i = 0; i < n; ++i)
    if (!images[i] || sizes[2 * i] < 1 || sizes[2 * i + 1] < 1 || (long long)sizes[2 * i] * sizes[2 * i + 1] >= (1ll << 30))
      return fail(DERP_EINVAL, std::string(who) + ": bad image " + std::to_string(i));
  return DERP_OK;
}

// The equirect reads images[c](int(py), int(px)) unclamped: every camera's resolution must fit its image
int checkFit(const char* who, const std::vector<DevCamera>& c, const int32_t* sizes) {
  for (size_t i = 0; i < c.size(); ++i)
    if (c[i].res[0] > sizes[2 * i] || c[i].res[1] > sizes[2 * i + 1])
      return fail(DERP_EINVAL, std::string(who) + ": camera " + std::to_string(i) + "'s resolution " +
                                   std::to_string(c[i].res[0]) + " x " + std::to_string(c[i].res[1]) +
                                   " exceeds its image " + std::to_string(sizes[2 * i]) + " x " +
                                   std::to_string(sizes[2 * i + 1]));
  return DERP_OK;
}

// Device copies of the rig and its images: device-resident images are used in place (16-byte aligned float4)
int stageSweepRig(const std::vector<DevCamera>& cams, const float* const* images, const int32_t* sizes) {
  SweepScratch& s = g_sweep;
  const int n = (int)cams.size();
  CU(s.cams.ensure(n));
  CU(cudaMemcpy(s.cams.p, cams.data(), n * sizeof(DevCamera), cudaMemcpyHostToDevice));
  if (!images) return DERP_OK;
  std::vector<SrcImage> im(n);
  std::vector<size_t> hostAt(n, SIZE_MAX);
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    if (!inPlace(images[i], 16)) {
      hostAt[i] = total;
      total += (size_t)sizes[2 * i] * sizes[2 * i + 1];
    }
    im[i] = SrcImage{reinterpret_cast<const float4*>(images[i]), sizes[2 * i], sizes[2 * i + 1]};
  }
  if (total) {
    CU(s.upload.ensure(total));
    for (int i = 0; i < n; ++i) {
      if (hostAt[i] == SIZE_MAX) continue;
      const size_t px = (size_t)sizes[2 * i] * sizes[2 * i + 1];
      CU(cudaMemcpy(s.upload.p + hostAt[i], images[i], px * sizeof(float4), cudaMemcpyDefault));
      im[i].p = s.upload.p + hostAt[i];
    }
  }
  CU(s.imgs.ensure(n));
  CU(cudaMemcpy(s.imgs.p, im.data(), n * sizeof(SrcImage), cudaMemcpyHostToDevice));
  return DERP_OK;
}

size_t sweepSmem(int n) { return (size_t)n * (sizeof(DevCamera) + sizeof(SrcImage)); }

// Host tables of one equirect slice set: full (bounds == NULL, one shared table) or cropped (one table per slice)
struct EquirectPlan {
  std::vector<double> cosT, sinT, sinP, cosP;
  std::vector<int> widths;
  int tStride = 0, pStride = 0, maxW = 0;
};
int planEquirect(const char* who, uint64_t height, int num, const double* bounds, EquirectPlan& p) {
  if (height < 1 || height > (1u << 15)) return fail(DERP_EINVAL, std::string(who) + ": height must be 1..32768");
  const double width = (double)(2 * height);
  if (!bounds) {
    std::vector<double> xs(2 * height), ys(height);
    for (uint64_t i = 0; i < 2 * height; ++i) xs[i] = (double)i;
    for (uint64_t i = 0; i < height; ++i) ys[i] = (double)i;
    p.cosT.resize(xs.size()); p.sinT.resize(xs.size()); p.sinP.resize(height); p.cosP.resize(height);
    derp::sweep::host::thetaTable(xs.data(), (int)xs.size(), width, p.cosT.data(), p.sinT.data());
    derp::sweep::host::phiTable(ys.data(), (int)height, (double)height, p.sinP.data(), p.cosP.data());
    p.widths.assign(num, (int)(2 * height));
    p.maxW = (int)(2 * height);
    return DERP_OK;
  }
  std::vector<uint64_t> ws(num);
  for (int k = 0; k < num; ++k) {
    if (!derp::sweep::host::cropWidth(height, bounds + 4 * k, &ws[k]))
      return fail(DERP_EINVAL, std::string(who) + ": slice " + std::to_string(k) +
                                   ": the crop box is empty or has zero width or height (nothing visible)");
    p.maxW = std::max<int>(p.maxW, (int)ws[k]);
  }
  p.tStride = p.maxW;
  p.pStride = (int)height;
  p.cosT.assign((size_t)num * p.maxW, 0); p.sinT.assign((size_t)num * p.maxW, 0);
  p.sinP.assign((size_t)num * height, 0); p.cosP.assign((size_t)num * height, 0);
  for (int k = 0; k < num; ++k) {
    std::vector<double> xs, ys;
    derp::sweep::host::cropSamples(height, ws[k], bounds + 4 * k, xs, ys);
    derp::sweep::host::thetaTable(xs.data(), (int)ws[k], width, &p.cosT[(size_t)k * p.maxW], &p.sinT[(size_t)k * p.maxW]);
    derp::sweep::host::phiTable(ys.data(), (int)height, (double)height, &p.sinP[(size_t)k * height],
                                &p.cosP[(size_t)k * height]);
    p.widths.push_back((int)ws[k]);
  }
  return DERP_OK;
}

// Device copy of an EquirectPlan; `outs` (device pointers) are filled by the caller
int uploadPlan(const EquirectPlan& p, const float* depths, int num, derp::sweep::EquirectSlices& s) {
  SweepScratch& g = g_sweep;
  const size_t nt = p.cosT.size(), np = p.sinP.size();
  CU(g.tabs.ensure(2 * nt + 2 * np));
  CU(cudaMemcpy(g.tabs.p, p.cosT.data(), nt * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + nt, p.sinT.data(), nt * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + 2 * nt, p.sinP.data(), np * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + 2 * nt + np, p.cosP.data(), np * 8, cudaMemcpyHostToDevice));
  CU(g.depths.ensure(num));
  CU(cudaMemcpy(g.depths.p, depths, num * sizeof(float), cudaMemcpyDefault));
  CU(g.widths.ensure(num));
  CU(cudaMemcpy(g.widths.p, p.widths.data(), num * sizeof(int), cudaMemcpyHostToDevice));
  s.cosT = g.tabs.p;
  s.sinT = g.tabs.p + nt;
  s.sinP = g.tabs.p + 2 * nt;
  s.cosP = g.tabs.p + 2 * nt + np;
  s.depths = g.depths.p;
  s.widths = g.widths.p;
  s.tStride = p.tStride;
  s.pStride = p.pStride;
  s.height = (int)(p.sinP.size() / (p.pStride ? (size_t)num : 1));
  s.numSlices = num;
  return DERP_OK;
}

}  // namespace

extern "C" {

int derp_sweep_overlaps(int device, const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                        const int32_t* image_sizes, int dst, const float* disparities, int num_slices, float* out) {
  static const char* who = "derp_sweep_overlaps";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, -1, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (dst < 0 || dst >= num_cams || !disparities || num_slices < 1 || !out)
    return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  const int W = (int)c[dst].res[0], H = (int)c[dst].res[1];  // Image colorDst(resolution.y(), resolution.x())
  if (W < 1 || H < 1) return fail(DERP_EINVAL, std::string(who) + ": the destination has no pixels");
  if ((long long)W * H * num_slices >= (1ll << 31)) return fail(DERP_EINVAL, std::string(who) + ": output too large");
  CU(cudaSetDevice(device));
  if (int rc = stageSweepRig(c, images_bgra, image_sizes)) return rc;
  SweepScratch& s = g_sweep;
  const size_t plane = (size_t)W * H;
  float4* dOut = reinterpret_cast<float4*>(out);  // float4 stores: 16-byte aligned
  if (int rc = outBuffer(dOut, plane * num_slices, s.out, 16)) return rc;
  CU(s.depths.ensure(num_slices));
  CU(cudaMemcpy(s.depths.p, disparities, num_slices * sizeof(float), cudaMemcpyDefault));
  CU(s.hits.ensure(1));
  CU(cudaMemset(s.hits.p, 0, sizeof(unsigned long long)));
  const int chunk = derp::sweep::kOverlapSlicesPerThread;
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((W + block.x - 1) / block.x, (H + block.y - 1) / block.y, (num_slices + chunk - 1) / chunk);
  derp::sweep::overlapsKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, s.imgs.p, num_cams, dst, W, H, s.depths.p,
                                                                     num_slices, chunk, dOut, s.hits.p);
  CU(cudaGetLastError());
  if (int rc = stageOut(reinterpret_cast<float4*>(out), dOut, plane * num_slices)) return rc;
  CU(cudaMemcpy(&g_sweepHits, s.hits.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_sweep_crop_bounds(int device, const DerpCameraDesc* cams, int num_cams, int center, uint64_t height,
                           const float* depths, int num_depths, double* bounds) {
  static const char* who = "derp_sweep_crop_bounds";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (!depths || num_depths < 1 || num_depths > 65535 || !bounds)
    return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, nullptr, p)) return rc;
  CU(cudaSetDevice(device));
  if (int rc = stageSweepRig(c, nullptr, nullptr)) return rc;
  derp::sweep::EquirectSlices sl{};
  if (int rc = uploadPlan(p, depths, num_depths, sl)) return rc;
  SweepScratch& s = g_sweep;
  std::vector<int> box(4 * num_depths);
  for (int k = 0; k < num_depths; ++k) {
    box[4 * k] = (int)(2 * height);  // minX = width, maxX = 0, minY = height, maxY = 0
    box[4 * k + 1] = 0;
    box[4 * k + 2] = (int)height;
    box[4 * k + 3] = 0;
  }
  CU(s.box.ensure(box.size()));
  CU(cudaMemcpy(s.box.p, box.data(), box.size() * sizeof(int), cudaMemcpyHostToDevice));
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((p.maxW + block.x - 1) / block.x, ((int)height + block.y - 1) / block.y, num_depths);
  derp::sweep::cropBoundsKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, num_cams, sl, s.box.p);
  CU(cudaGetLastError());
  CU(cudaMemcpy(box.data(), s.box.p, box.size() * sizeof(int), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < box.size(); ++i) bounds[i] = (double)box[i];
  return DERP_OK;
}

int derp_sweep_crop_width(uint64_t height, const double* bounds, uint64_t* width) {
  if (!bounds || !width) return fail(DERP_EINVAL, "derp_sweep_crop_width: bad arguments");
  if (!derp::sweep::host::cropWidth(height, bounds, width))
    return fail(DERP_EINVAL, "derp_sweep_crop_width: the crop box is empty or has zero width or height (nothing visible)");
  return DERP_OK;
}

int derp_sweep_equirect(int device, const DerpCameraDesc* cams, int num_cams, int center, const float* const* images_bgra,
                        const int32_t* image_sizes, uint64_t height, const float* depths, int num_depths,
                        const double* bounds, int black_bg, float* const* out) {
  static const char* who = "derp_sweep_equirect";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (int rc = checkFit(who, c, image_sizes)) return rc;
  if (!depths || num_depths < 1 || num_depths > 65535 || !out) return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  for (int k = 0; k < num_depths; ++k)
    if (!out[k]) return fail(DERP_EINVAL, std::string(who) + ": NULL output");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, bounds, p)) return rc;
  CU(cudaSetDevice(device));
  if (int rc = stageSweepRig(c, images_bgra, image_sizes)) return rc;
  derp::sweep::EquirectSlices sl{};
  if (int rc = uploadPlan(p, depths, num_depths, sl)) return rc;
  SweepScratch& s = g_sweep;
  // device-resident outputs are written in place; the others are staged in one scratch buffer and copied back
  std::vector<float4*> outs(num_depths);
  std::vector<size_t> at(num_depths, SIZE_MAX);
  size_t total = 0;
  for (int k = 0; k < num_depths; ++k) {
    if (inPlace(out[k], 16)) continue;
    at[k] = total;
    total += (size_t)p.widths[k] * height;
  }
  if (total) CU(s.out.ensure(total));
  for (int k = 0; k < num_depths; ++k)
    outs[k] = at[k] == SIZE_MAX ? reinterpret_cast<float4*>(out[k]) : s.out.p + at[k];
  CU(s.outs.ensure(num_depths));
  CU(cudaMemcpy(s.outs.p, outs.data(), num_depths * sizeof(float4*), cudaMemcpyHostToDevice));
  sl.outs = s.outs.p;
  CU(s.hits.ensure(1));
  CU(cudaMemset(s.hits.p, 0, sizeof(unsigned long long)));
  const float4 bg = black_bg ? make_float4(0.f, 0.f, 0.f, 1.f) : make_float4(0.f, 0.f, 1.f, 1.f);
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((p.maxW + block.x - 1) / block.x, ((int)height + block.y - 1) / block.y, num_depths);
  derp::sweep::equirectKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, s.imgs.p, num_cams, sl, bg, s.hits.p);
  CU(cudaGetLastError());
  for (int k = 0; k < num_depths; ++k)
    if (int rc = stageOut(reinterpret_cast<float4*>(out[k]), outs[k], (size_t)p.widths[k] * height)) return rc;
  CU(cudaMemcpy(&g_sweepHits, s.hits.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_sweep_center_rig(const DerpCameraDesc* cams, int num_cams, int center, DerpCameraDesc* out, double* rotation9) {
  if (!cams || num_cams < 1 || center < 0 || center >= num_cams || !out)
    return fail(DERP_EINVAL, "derp_sweep_center_rig: bad arguments");
  std::vector<DerpCameraDesc> d(cams, cams + num_cams);
  if (!derp::sweep::host::centerRig(d.data(), num_cams, center))
    return fail(DERP_EINVAL, "derp_sweep_center_rig: invalid camera rotation");
  for (int i = 0; i < num_cams; ++i) {
    out[i] = d[i];
    if (rotation9) {
      DevCamera c;
      if (!host::makeCamera(d[i], &c)) return fail(DERP_EINVAL, "derp_sweep_center_rig: invalid camera");
      for (int k = 0; k < 9; ++k) rotation9[9 * i + k] = c.rot[k];
    }
  }
  return DERP_OK;
}

uint64_t derp_sweep_last_hits(void) { return g_sweepHits; }

int derp_test_sweep_overlaps_host(const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                                  const int32_t* image_sizes, int dst, const float* disparities, int num_slices,
                                  float* out) {
  static const char* who = "derp_test_sweep_overlaps_host";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, -1, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (dst < 0 || dst >= num_cams || !disparities || num_slices < 1 || !out) return fail(DERP_EINVAL, "bad arguments");
  std::vector<SrcImage> im(num_cams);
  for (int i = 0; i < num_cams; ++i)
    im[i] = SrcImage{reinterpret_cast<const float4*>(images_bgra[i]), image_sizes[2 * i], image_sizes[2 * i + 1]};
  const int W = (int)c[dst].res[0], H = (int)c[dst].res[1];
  float4* o = reinterpret_cast<float4*>(out);
  int hits = 0;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const double px = x + 0.5, py = y + 0.5;
      const bool outside = outsideImageCircle(c[dst], px, py);
      double dir[3];
      if (!outside) pixelRay(c[dst], px, py, dir);
      for (int k = 0; k < num_slices; ++k)
        o[(size_t)k * W * H + (size_t)y * W + x] =
            outside ? make_float4(0.f, 0.f, 0.f, 0.f)
                    : derp::sweep::overlapPixel(c.data(), im.data(), num_cams, c[dst].pos, dir, disparities[k], &hits);
    }
  return DERP_OK;
}

int derp_test_sweep_equirect_host(const DerpCameraDesc* cams, int num_cams, int center,
                                  const float* const* images_bgra, const int32_t* image_sizes, uint64_t height,
                                  const float* depths, int num_depths, const double* bounds, int black_bg,
                                  float* const* out) {
  static const char* who = "derp_test_sweep_equirect_host";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (int rc = checkFit(who, c, image_sizes)) return rc;
  if (!depths || num_depths < 1 || !out) return fail(DERP_EINVAL, "bad arguments");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, bounds, p)) return rc;
  std::vector<SrcImage> im(num_cams);
  for (int i = 0; i < num_cams; ++i)
    im[i] = SrcImage{reinterpret_cast<const float4*>(images_bgra[i]), image_sizes[2 * i], image_sizes[2 * i + 1]};
  const float4 bg = black_bg ? make_float4(0.f, 0.f, 0.f, 1.f) : make_float4(0.f, 0.f, 1.f, 1.f);
  int hits = 0;
  for (int k = 0; k < num_depths; ++k) {
    const double depth = (double)depths[k];
    const int W = p.widths[k];
    for (uint64_t y = 0; y < height; ++y)
      for (int x = 0; x < W; ++x) {
        const double r = depth * p.sinP[(size_t)k * p.pStride + y];
        reinterpret_cast<float4*>(out[k])[y * W + x] = derp::sweep::equirectPixel(
            c.data(), im.data(), num_cams, r * p.cosT[(size_t)k * p.tStride + x], r * p.sinT[(size_t)k * p.tStride + x],
            depth * p.cosP[(size_t)k * p.pStride + y], bg, &hits);
      }
  }
  return DERP_OK;
}

}  // extern "C"
