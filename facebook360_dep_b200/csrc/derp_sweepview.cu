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
  // derp_project_equirect_masks
  DevBuf<uint8_t> maskUpload, maskOut;
  DevBuf<derp::sweep::EqrMask> masks;
  DevBuf<uint8_t*> maskOuts;
  UndecidedList<unsigned long long> undecided;  // camera << 32 | pixel
  DevBuf<long long> resolved;
};
thread_local SweepScratch g_sweep;
thread_local unsigned long long g_sweepHits = 0;  // contributing (sample, camera) pairs of the last call
thread_local unsigned long long g_projectHostPixels = 0;  // pixels the last derp_project_equirect_masks left to the host

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
  if (int rc = upload(s.cams, cams.data(), n)) return rc;
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
  return upload(s.imgs, im.data(), n);
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
  if (int rc = upload(g.widths, p.widths.data(), num)) return rc;
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

// Arguments of derp_project_equirect_masks and its host twin; W / H receive each camera's output size
int checkProject(const char* who, const DerpCameraDesc* cams, int n, double depth, const uint8_t* const* masks,
                 const int32_t* sizes, uint8_t* const* out, std::vector<DevCamera>& c, std::vector<int>& W,
                 std::vector<int>& H) {
  if (int rc = sweepCameras(who, cams, n, -1, c)) return rc;
  if (!(depth > 0) || !std::isfinite(depth)) return fail(DERP_EINVAL, std::string(who) + ": depth must be > 0 and finite");
  if (!masks || !sizes || !out) return fail(DERP_EINVAL, std::string(who) + ": masks, sizes and outputs are required");
  W.resize(n);
  H.resize(n);
  for (int i = 0; i < n; ++i) {
    if (!masks[i] || !out[i] || sizes[2 * i] < 1 || sizes[2 * i + 1] < 1 ||
        (long long)sizes[2 * i] * sizes[2 * i + 1] >= (1ll << 31))
      return fail(DERP_EINVAL, std::string(who) + ": bad mask or output " + std::to_string(i));
    W[i] = (int)c[i].res[0];  // cv::Mat_<bool>(resolution.y(), resolution.x())
    H[i] = (int)c[i].res[1];
    if (W[i] < 1 || H[i] < 1 || (long long)W[i] * H[i] >= (1ll << 31))
      return fail(DERP_EINVAL, std::string(who) + ": camera " + std::to_string(i) + " has no pixels or too many");
  }
  return DERP_OK;
}

// The host's decision at pixel (x, y) of camera c: the mask index, or -1 (the same DERP_HD code with the C library)
long long projectPixelHost(const DevCamera& c, int x, int y, double depth, int mw, int mh) {
  double w[3];
  derp::rigPoint(c, x, y, depth, w);
  return derp::sweep::eqrIndex(w[0], w[1], w[2], mw, mh);
}

// Test probe: eqrIndexProven of the boxes box[6 i .. 6 i + 5] (x lo, x hi, y lo, y hi, z lo, z hi)
__global__ void eqrIndexProvenKernel(const double* box, int n, int W, int H, long long* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Iv w[3] = {{box[6 * i], box[6 * i + 1]}, {box[6 * i + 2], box[6 * i + 3]}, {box[6 * i + 4], box[6 * i + 5]}};
  out[i] = derp::sweep::eqrIndexProven(w, W, H);
}

}  // namespace

extern "C" {

int derp_project_equirect_masks(int device, const DerpCameraDesc* cams, int num_cams, double depth,
                                const uint8_t* const* eqr_masks, const int32_t* mask_sizes, uint8_t* const* out) {
  static const char* who = "derp_project_equirect_masks";
  using derp::sweep::EqrMask;
  std::vector<DevCamera> c;
  std::vector<int> W, H;
  if (int rc = checkProject(who, cams, num_cams, depth, eqr_masks, mask_sizes, out, c, W, H)) return rc;
  CU(cudaSetDevice(device));
  SweepScratch& s = g_sweep;
  if (int rc = upload(s.cams, c.data(), num_cams)) return rc;
  // masks: device-resident ones in place, the others uploaded into one scratch buffer
  std::vector<EqrMask> m(num_cams);
  std::vector<size_t> maskAt(num_cams, SIZE_MAX), outAt(num_cams, SIZE_MAX);
  size_t maskTotal = 0, outTotal = 0;
  int maxW = 0, maxH = 0;
  for (int i = 0; i < num_cams; ++i) {
    m[i] = EqrMask{eqr_masks[i], mask_sizes[2 * i], mask_sizes[2 * i + 1]};
    if (!inPlace(eqr_masks[i], 1)) {
      maskAt[i] = maskTotal;
      maskTotal += (size_t)m[i].w * m[i].h;
    }
    if (!inPlace(out[i], 1)) {
      outAt[i] = outTotal;
      outTotal += (size_t)W[i] * H[i];
    }
    maxW = std::max(maxW, W[i]);
    maxH = std::max(maxH, H[i]);
  }
  if (maskTotal) CU(s.maskUpload.ensure(maskTotal));
  if (outTotal) CU(s.maskOut.ensure(outTotal));
  std::vector<uint8_t*> outs(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    if (maskAt[i] != SIZE_MAX) {
      CU(cudaMemcpy(s.maskUpload.p + maskAt[i], eqr_masks[i], (size_t)m[i].w * m[i].h, cudaMemcpyDefault));
      m[i].p = s.maskUpload.p + maskAt[i];
    }
    outs[i] = outAt[i] == SIZE_MAX ? out[i] : s.maskOut.p + outAt[i];
  }
  if (int rc = upload(s.masks, m.data(), num_cams)) return rc;
  if (int rc = upload(s.maskOuts, outs.data(), num_cams)) return rc;
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((maxW + block.x - 1) / block.x, (maxH + block.y - 1) / block.y, num_cams);
  std::vector<unsigned long long> list;
  auto launch = [&](UndecidedView<unsigned long long> undecided) {
    derp::sweep::projectMasksKernel<<<grid, block>>>(s.cams.p, s.masks.p, depth, s.maskOuts.p, undecided);
    return DERP_OK;
  };
  if (int rc = s.undecided.collect(launch, list)) return rc;
  const size_t count = list.size();
  if (count) {
    std::vector<long long> at(count);
    for (size_t k = 0; k < count; ++k) {
      const int i = (int)(list[k] >> 32);
      const unsigned pixel = (unsigned)list[k];
      at[k] = projectPixelHost(c[i], (int)(pixel % W[i]), (int)(pixel / W[i]), depth, m[i].w, m[i].h);
    }
    if (int rc = upload(s.resolved, at.data(), count)) return rc;
    derp::sweep::resolveMasksKernel<<<grid1(count), 256>>>(s.masks.p, s.maskOuts.p, s.undecided.items.p, s.resolved.p,
                                                           (int)count);
    CU(cudaGetLastError());
  }
  for (int i = 0; i < num_cams; ++i)
    if (int rc = stageOut(out[i], outs[i], (size_t)W[i] * H[i])) return rc;
  g_projectHostPixels = count;
  return DERP_OK;
}

uint64_t derp_project_last_host_pixels(void) { return g_projectHostPixels; }

int derp_test_project_equirect_masks_host(const DerpCameraDesc* cams, int num_cams, double depth,
                                          const uint8_t* const* eqr_masks, const int32_t* mask_sizes,
                                          uint8_t* const* out) {
  std::vector<DevCamera> c;
  std::vector<int> W, H;
  if (int rc = checkProject("derp_test_project_equirect_masks_host", cams, num_cams, depth, eqr_masks, mask_sizes, out,
                            c, W, H))
    return rc;
  for (int i = 0; i < num_cams; ++i)
    for (int y = 0; y < H[i]; ++y)
      for (int x = 0; x < W[i]; ++x) {
        const long long at = projectPixelHost(c[i], x, y, depth, mask_sizes[2 * i], mask_sizes[2 * i + 1]);
        out[i][(size_t)y * W[i] + x] = at >= 0 && eqr_masks[i][at] ? 255 : 0;
      }
  return DERP_OK;
}

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
  if (int rc = upload(s.box, box.data(), box.size())) return rc;
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
  if (int rc = upload(s.outs, outs.data(), num_depths)) return rc;
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

int derp_test_eqr_index_proven(int device, const double* boxes, int n, int width, int height, int64_t* out) {
  if (!boxes || n < 1 || width < 1 || height < 1 || !out)
    return fail(DERP_EINVAL, "derp_test_eqr_index_proven: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<double> db;
  DevBuf<long long> dout;
  if (int rc = upload(db, boxes, 6 * (size_t)n)) return rc;
  CU(dout.ensure(n));
  eqrIndexProvenKernel<<<grid1(n), 256>>>(db.p, n, width, height, dout.p);
  CU(cudaGetLastError());
  CU(cudaMemcpy(out, dout.p, n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_test_eqr_index_host(const double* pts, int n, int width, int height, int64_t* out) {
  if (!pts || n < 1 || width < 1 || height < 1 || !out) return fail(DERP_EINVAL, "derp_test_eqr_index_host: bad arguments");
  for (int i = 0; i < n; ++i) out[i] = derp::sweep::eqrIndex(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], width, height);
  return DERP_OK;
}

}  // extern "C"
