// Constant-depth sweep slices of GenerateCameraOverlaps and GenerateEquirect (include/derp_sweepview.h).
//
// One kernel serves both apps: each thread owns one target pixel and walks a chunk of slices.  The per-pixel bodies are
// DERP_HD, so derp_test_sweep_*_host runs the same code on the host.  Arithmetic follows the reference's operation
// order (-fmad=false, no contraction):
//   - overlaps (GenerateCameraOverlaps.cpp:54-83): the destination pixel's ray is computed once (pixelRay) and reused
//     for every slice, world = position + dir * double(1.0f / disparity) (Camera::rig = ParametrizedLine::pointAt);
//     every camera in rig order that sees the point adds getPixelBilinear (fp32, clamp to edge) to an fp32 sum; the
//     result is the fp32 product (1.0f / count) * sum, NaN where count is 0 (inf * 0).
//   - equirect (GenerateEquirect.cpp:79-131): point = ((depth * sin phi) * cos theta, (depth * sin phi) * sin theta,
//     depth * cos phi) in fp64 from host tables of sin / cos (the host's C library, so the points are the reference's
//     bits); the texel is images[c](int(py), int(px)); the mean is float(double(sum) * (1. / n)) per channel
//     (OpenCV's Vec / int), the background (0, 0, 1, 1) or (0, 0, 0, 1) when no camera sees the point.
//   - crop bounds (GenerateEquirect.cpp:139-156): per depth, the min / max column and row of the equirect pixels that
//     any camera sees, reduced with integer atomics.
// The source projection is derp::sees; on the device its FTHETA atan2 is the polynomial of derp_camera.cuh, so FTHETA
// rigs can differ from the reference where a pixel coordinate lands within an ulp of a texel or sensor edge.
#pragma once

#include <cstdint>

#include "derp_camera.cuh"
#include "derp_host.cuh"
#include "derp_interval.cuh"

namespace derp {
namespace sweep {

struct SrcImage {  // 16 bytes: one per camera, staged in shared memory next to the cameras
  const float4* p;
  int w, h;
};

constexpr int kMaxCams = 64;
constexpr int kSweepThreadsX = 32, kSweepThreadsY = 8;
constexpr int kOverlapSlicesPerThread = 16;

DERP_HD int clampI(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

DERP_HD void addScaled(float4& acc, float w, const float4& p) {
  acc.x = acc.x + w * p.x;
  acc.y = acc.y + w * p.y;
  acc.z = acc.z + w * p.z;
  acc.w = acc.w + w * p.w;
}

// cv_util::getPixelBilinear on a float BGRA image (CvUtil.h:84-120): integer pixel corners, clamp to edge
DERP_HD float4 bilinear4(const SrcImage& im, float x, float y) {
  const float xf = roundf(x), yf = roundf(y);
  const int xi = (int)xf, yi = (int)yf;
  const int x0 = clampI(xi - 1, im.w - 1), x1 = clampI(xi, im.w - 1);
  const int y0 = clampI(yi - 1, im.h - 1), y1 = clampI(yi, im.h - 1);
  const float xw = x - xf + 0.5f, yw = y - yf + 0.5f;
  const float w00 = (1 - xw) * (1 - yw), w01 = xw * (1 - yw), w10 = (1 - xw) * yw, w11 = xw * yw;
  const float4 p00 = im.p[(size_t)y0 * im.w + x0], p01 = im.p[(size_t)y0 * im.w + x1];
  const float4 p10 = im.p[(size_t)y1 * im.w + x0], p11 = im.p[(size_t)y1 * im.w + x1];
  float4 r = make_float4(w00 * p00.x, w00 * p00.y, w00 * p00.z, w00 * p00.w);
  addScaled(r, w01, p01);
  addScaled(r, w10, p10);
  addScaled(r, w11, p11);
  return r;
}

// One slice of projectSrcsToDst at a pixel inside the destination's image circle; org / dir: the pixel's ray
DERP_HD float4 overlapPixel(const DevCamera* cams, const SrcImage* imgs, int n, const double* org, const double* dir,
                            float disparity, int* hits) {
  const double depth = (double)(1.0f / disparity);
  const double wx = org[0] + dir[0] * depth, wy = org[1] + dir[1] * depth, wz = org[2] + dir[2] * depth;
  int count = 0;
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < n; ++s) {
    double px, py;
    if (sees(cams[s], wx, wy, wz, &px, &py)) {
      const float4 v = bilinear4(imgs[s], (float)px, (float)py);
      sum.x = sum.x + v.x;
      sum.y = sum.y + v.y;
      sum.z = sum.z + v.z;
      sum.w = sum.w + v.w;
      ++count;
    }
  }
  *hits += count;
  const float k = 1.0f / (float)count;
  return make_float4(k * sum.x, k * sum.y, k * sum.z, k * sum.w);
}

// getPixelColor (GenerateEquirect.cpp:79-100) at a rig point
DERP_HD float4 equirectPixel(const DevCamera* cams, const SrcImage* imgs, int n, double px, double py, double pz,
                             float4 background, int* hits) {
  int count = 0;
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < n; ++c) {
    double u, v;
    if (sees(cams[c], px, py, pz, &u, &v)) {
      const float4 t = imgs[c].p[(size_t)(int)v * imgs[c].w + (int)u];
      sum.x = sum.x + t.x;
      sum.y = sum.y + t.y;
      sum.z = sum.z + t.z;
      sum.w = sum.w + t.w;
      ++count;
    }
  }
  *hits += count;
  if (count == 0) return background;
  const double s = 1. / count;
  return make_float4((float)((double)sum.x * s), (float)((double)sum.y * s), (float)((double)sum.z * s),
                     (float)((double)sum.w * s));
}

DERP_HD bool anySees(const DevCamera* cams, int n, double px, double py, double pz) {
  for (int c = 0; c < n; ++c) {
    double u, v;
    if (sees(cams[c], px, py, pz, &u, &v)) return true;
  }
  return false;
}

// Equirect slice geometry: slice k samples column x at (cosT, sinT)[k * tStride + x] and row y at
// (sinP, cosP)[k * pStride + y]; widths[k] columns, written to outs[k].
struct EquirectSlices {
  const double* cosT;
  const double* sinT;
  const double* sinP;
  const double* cosP;
  const float* depths;
  const int* widths;
  float4* const* outs;
  int tStride, pStride, height, numSlices;
};

#if defined(__CUDACC__)
__device__ __forceinline__ void stageRig(const DevCamera* gCams, const SrcImage* gImgs, int n, DevCamera* sCams,
                                         SrcImage* sImgs) {
  const int t = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  const float4* src = reinterpret_cast<const float4*>(gCams);
  float4* dst = reinterpret_cast<float4*>(sCams);
  const int words = n * (int)(sizeof(DevCamera) / sizeof(float4));
  for (int i = t; i < words; i += nt) dst[i] = src[i];
  if (gImgs)
    for (int i = t; i < n; i += nt) sImgs[i] = gImgs[i];
  __syncthreads();
}

// GenerateCameraOverlaps: one thread per destination pixel, slices [z * chunk, min((z + 1) * chunk, num))
__global__ void __launch_bounds__(kSweepThreadsX * kSweepThreadsY) overlapsKernel(
    const DevCamera* __restrict__ gCams, const SrcImage* __restrict__ gImgs, int n, int dst, int W, int H,
    const float* __restrict__ disparities, int numSlices, int chunk, float4* __restrict__ out,
    unsigned long long* __restrict__ hitCount) {
  extern __shared__ float4 smem[];
  DevCamera* sCams = reinterpret_cast<DevCamera*>(smem);
  SrcImage* sImgs = reinterpret_cast<SrcImage*>(sCams + n);
  stageRig(gCams, gImgs, n, sCams, sImgs);
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const int k0 = blockIdx.z * chunk, k1 = min(numSlices, k0 + chunk);
  const DevCamera& cd = sCams[dst];
  const double px = x + 0.5, py = y + 0.5;
  const size_t plane = (size_t)W * H, at = (size_t)y * W + x;
  if (outsideImageCircle(cd, px, py)) {
    for (int k = k0; k < k1; ++k) out[k * plane + at] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  double dir[3];
  pixelRay(cd, px, py, dir);
  int hits = 0;
  for (int k = k0; k < k1; ++k) out[k * plane + at] = overlapPixel(sCams, sImgs, n, cd.pos, dir, disparities[k], &hits);
  if (hitCount) atomicAdd(hitCount, (unsigned long long)hits);
}

// GenerateEquirect: one thread per equirect pixel of slice blockIdx.z
__global__ void __launch_bounds__(kSweepThreadsX * kSweepThreadsY) equirectKernel(
    const DevCamera* __restrict__ gCams, const SrcImage* __restrict__ gImgs, int n, EquirectSlices s, float4 background,
    unsigned long long* __restrict__ hitCount) {
  extern __shared__ float4 smem[];
  DevCamera* sCams = reinterpret_cast<DevCamera*>(smem);
  SrcImage* sImgs = reinterpret_cast<SrcImage*>(sCams + n);
  stageRig(gCams, gImgs, n, sCams, sImgs);
  const int k = blockIdx.z;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int W = s.widths[k];
  if (x >= W || y >= s.height) return;
  const double depth = (double)s.depths[k];
  const double ct = s.cosT[(size_t)k * s.tStride + x], st = s.sinT[(size_t)k * s.tStride + x];
  const double sp = s.sinP[(size_t)k * s.pStride + y], cp = s.cosP[(size_t)k * s.pStride + y];
  const double r = depth * sp;
  int hits = 0;
  s.outs[k][(size_t)y * W + x] = equirectPixel(sCams, sImgs, n, r * ct, r * st, depth * cp, background, &hits);
  if (hitCount) atomicAdd(hitCount, (unsigned long long)hits);
}

// createCroppedEquirect's bounding box: box[4 k ..] = {minX, maxX, minY, maxY} of the visible pixels of slice k
__global__ void __launch_bounds__(kSweepThreadsX * kSweepThreadsY) cropBoundsKernel(
    const DevCamera* __restrict__ gCams, int n, EquirectSlices s, int* __restrict__ box) {
  extern __shared__ float4 smem[];
  DevCamera* sCams = reinterpret_cast<DevCamera*>(smem);
  SrcImage* sImgs = reinterpret_cast<SrcImage*>(sCams + n);
  stageRig(gCams, nullptr, n, sCams, sImgs);
  const int k = blockIdx.z;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= s.widths[k] || y >= s.height) return;
  const double depth = (double)s.depths[k];
  const double r = depth * s.sinP[y];
  if (anySees(sCams, n, r * s.cosT[x], r * s.sinT[x], depth * s.cosP[y])) {
    atomicMin(&box[4 * k + 0], x);
    atomicMax(&box[4 * k + 1], x);
    atomicMin(&box[4 * k + 2], y);
    atomicMax(&box[4 * k + 3], y);
  }
}
#endif

// ---- ProjectEquirectsToCameras (derp_project_equirect_masks) ------------------------------------------------
// Per camera pixel (ProjectEquirectsToCameras.cpp:104-118): world = cam.rig({x + .5, y + .5}, depth) in fp64, then
// worldToEquirect (ImageUtil.cpp:127-140) against the camera's W x H mask, the range test and mask(int(v H), int(u W)).
// The reference's ImageUtil.cpp calls acos / atan2 with float arguments and resolves them to the float overloads
// (acosf / atan2f; tests/test_eqr_project.py pins this against the compiled reference object).
struct EqrMask {  // 16 bytes: one per camera
  const uint8_t* p;
  int w, h;
};

// The mask index int(v H) * W + int(u W) that the reference reads at rig point w, or -1 where it reads nothing: out of
// range, or a NaN coordinate (z > 1 near a pole: the reference indexes the mask with int(NaN) there).
DERP_HD long long eqrIndex(double wx, double wy, double wz, int W, int H) {
  const float depth = (float)sqrt((wx * wx + wy * wy) + wz * wz);
  const float x = (float)(wx / depth), y = (float)(wy / depth), z = (float)(wz / depth);
  const float phi = acosf(z);
  float theta = atan2f(y, x);
  if (theta > 0) theta = (float)(theta - 2 * M_PI);
  const float v = (float)(phi / M_PI);
  const float u = (float)(-theta / (2.0f * M_PI));
  const float px = u * (float)W, py = v * (float)H;
  if (!(px >= 0 && py >= 0 && px < W && py < H)) return -1;
  return (long long)(int)py * W + (int)px;
}

#if defined(__CUDACC__)
// ---- the device's proof of a pixel: the interval chain and bounds of derp_interval.cuh ----
// p < 0 -> -1, p >= n -> n, else int(p): monotone in p, so equal codes at both ends fix the whole interval
__device__ __forceinline__ int rangeCode(float p, int n) { return p < 0 ? -1 : p >= n ? n : (int)p; }

// eqrIndex on the interval w: the index (>= 0) or -1 when proven, -2 when the interval does not decide
__device__ __forceinline__ long long eqrIndexProven(const Iv* w, int W, int H) {
  constexpr long long kUndecided = -2;
  const Iv n = ivAdd(ivAdd(ivSqr(w[0]), ivSqr(w[1])), ivSqr(w[2]));
  const Iv depth = ivFloat(Iv{__dsqrt_rd(n.lo), __dsqrt_ru(n.hi)});
  if (!(depth.lo > 0)) return kUndecided;
  const Iv x = ivFloat(ivDiv(w[0], depth)), y = ivFloat(ivDiv(w[1], depth)), z = ivFloat(ivDiv(w[2], depth));
  if (z.lo > 1 || z.hi < -1) return -1;                     // acos is NaN at every point: the pixel stays 0
  if (!(z.hi <= 1 && z.lo >= -1)) return kUndecided;        // NaN at some points only
  const Iv phi = Iv{widenF(acosf((float)z.hi), kAcosfUlps).lo, widenF(acosf((float)z.lo), kAcosfUlps).hi};
  // atan2 over the box x * y: off the origin and the branch cut (x < 0, y = 0) its extremes are at the corners
  if (x.lo <= 0 && x.hi >= 0 && y.lo <= 0 && y.hi >= 0) return kUndecided;
  // The cut: where y's interval holds 0 with x < 0.  A y that crosses 0 is also refused by the theta test below (the
  // corners' atan2f have opposite signs); this test covers the ends that are zeros, whose sign the interval does not
  // track while the host's atan2f(+-0, x < 0) = +-pi does
  if (x.lo < 0 && y.lo <= 0 && y.hi >= 0) return kUndecided;
  double tlo = INFINITY, thi = -INFINITY;
  for (int k = 0; k < 4; ++k) {
    const Iv t = widenF(atan2f((float)((k & 1) ? y.hi : y.lo), (float)((k & 2) ? x.hi : x.lo)), kAtan2fUlps);
    tlo = fmin(tlo, t.lo);
    thi = fmax(thi, t.hi);
  }
  Iv theta = ivFloat(Iv{tlo, thi});  // the host's theta is a float inside the widened range
  if (theta.lo > 0) {
    theta = ivFloat(Iv{__dadd_rd(theta.lo, -kTwoPi), __dadd_ru(theta.hi, -kTwoPi)});
  } else if (theta.hi > 0) {
    return kUndecided;
  }
  const Iv v = ivFloat(ivDivPos(ivFloat(phi), M_PI));
  const Iv u = ivFloat(ivDivPos(Iv{-theta.hi, -theta.lo}, kTwoPi));
  const float fW = (float)W, fH = (float)H;
  const float pxl = __fmul_rd((float)u.lo, fW), pxh = __fmul_ru((float)u.hi, fW);
  const float pyl = __fmul_rd((float)v.lo, fH), pyh = __fmul_ru((float)v.hi, fH);
  if (!(pxl <= pxh) || !(pyl <= pyh)) return kUndecided;  // NaN
  const int xl = rangeCode(pxl, W), xh = rangeCode(pxh, W), yl = rangeCode(pyl, H), yh = rangeCode(pyh, H);
  if ((xl == xh && (xl < 0 || xl >= W)) || (yl == yh && (yl < 0 || yl >= H))) return -1;  // skipped either way
  if (xl != xh || yl != yh) return kUndecided;
  return (long long)yl * W + xl;
}

// One thread per pixel of camera blockIdx.z: out = 255 where the proven mask texel is set, 0 where it is not or where
// the reference skips the pixel; undecided pixels are written 1 and listed (camera << 32 | pixel) for the host
__global__ void __launch_bounds__(kSweepThreadsX * kSweepThreadsY) projectMasksKernel(
    const DevCamera* __restrict__ gCams, const EqrMask* __restrict__ masks, double depth, uint8_t* const* outs,
    UndecidedView<unsigned long long> undecided) {
  __shared__ DevCamera cam;
  const int i = blockIdx.z;
  if (threadIdx.x == 0 && threadIdx.y == 0) cam = gCams[i];
  __syncthreads();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int W = (int)cam.res[0], H = (int)cam.res[1];
  if (x >= W || y >= H) return;
  const EqrMask m = masks[i];
  Iv w[3];
  rigPointIv(cam, x, y, depth, w);
  const long long at = eqrIndexProven(w, m.w, m.h);
  uint8_t v = 0;
  if (at >= 0) {
    v = m.p[at] ? 255 : 0;
  } else if (at == -2) {
    v = 1;
    undecided.append((unsigned long long)i << 32 | (unsigned)(y * W + x));
  }
  outs[i][(size_t)y * W + x] = v;
}

// Writes the host's decisions: at[k] is the mask index of undecided pixel list[k], or -1
__global__ void resolveMasksKernel(const EqrMask* __restrict__ masks, uint8_t* const* outs,
                                   const unsigned long long* __restrict__ list, const long long* __restrict__ at,
                                   int num) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= num) return;
  const int i = (int)(list[k] >> 32);
  const unsigned pixel = (unsigned)list[k];
  outs[i][pixel] = at[k] >= 0 && masks[i].p[at[k]] ? 255 : 0;
}
#endif

// ---- host side ----------------------------------------------------------------------------------------------
namespace host {

// theta / phi of getEquirectPoint (GenerateEquirect.cpp:102-115) for sample coordinates xs / ys of a width x height
// equirect, with the host's sin / cos
inline void thetaTable(const double* xs, int count, double width, double* cosT, double* sinT) {
  for (int i = 0; i < count; ++i) {
    const double theta = -1 * ((xs[i] + 0.5) / width * 2 * M_PI);
    cosT[i] = cos(theta);
    sinT[i] = sin(theta);
  }
}
inline void phiTable(const double* ys, int count, double height, double* sinP, double* cosP) {
  for (int i = 0; i < count; ++i) {
    const double phi = (ys[i] + 0.5) / height * M_PI;
    sinP[i] = sin(phi);
    cosP[i] = cos(phi);
  }
}

// createCroppedEquirect's output width and sample positions (GenerateEquirect.cpp:158-169)
inline bool cropWidth(uint64_t height, const double* b, uint64_t* width) {
  const double minX = b[0], maxX = b[1], minY = b[2], maxY = b[3];
  if (!(maxX > minX) || !(maxY > minY)) return false;
  const double w = height / (maxY - minY) * (maxX - minX);
  if (!(w >= 1) || w >= 1e9) return false;
  *width = (uint64_t)w;
  return true;
}
inline void cropSamples(uint64_t height, uint64_t newWidth, const double* b, std::vector<double>& xs,
                        std::vector<double>& ys) {
  const double minX = b[0], maxX = b[1], minY = b[2], maxY = b[3];
  xs.resize(newWidth);
  ys.resize(height);
  for (uint64_t i = 0; i < newWidth; ++i) xs[i] = (double)i * (maxX - minX) / newWidth + minX;
  for (uint64_t i = 0; i < height; ++i) ys[i] = (double)i * (maxY - minY) / height + minY;
}

// ---- centerRig (GenerateEquirect.cpp:177-231) with transformRig (source/rig/RigTransform.h) -------------------------
// Eigen's geometry in the order written out in oracle/sweepshim/geometry_extra.h: AngleAxis -> quaternion, the
// quaternion product z * y * x, toRotationMatrix, [s I | s t] * [R | 0], and Transform * v = L v + t.
using derp::host::Quat;
using derp::host::quatOf;
using derp::host::quatMul;
using derp::host::quatToRotation;
using derp::host::mulMV;
struct Affine {
  double L[9];
  double t[3];
};
// generateTransform(rotation, translation, UniformScaling(1), false) = (scale * Translation) * Affine3d(z * y * x)
inline Affine generateTransform(const double* rot, const double* trans) {
  double R[9];
  quatToRotation(quatMul(quatMul(quatOf(rot[2], 2), quatOf(rot[1], 1)), quatOf(rot[0], 0)), R);
  const double s = 1;
  double S[9];
  for (int i = 0; i < 9; ++i) S[i] = (i % 4 == 0) ? s : 0.0;
  Affine a;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      a.L[3 * i + j] = (S[3 * i] * R[j] + S[3 * i + 1] * R[3 + j]) + S[3 * i + 2] * R[6 + j];
  const double zero[3] = {0, 0, 0};
  double lt[3];
  mulMV(S, zero, lt);
  for (int i = 0; i < 3; ++i) a.t[i] = lt[i] + trans[i] * s;
  return a;
}
inline void apply(const Affine& a, const double* v, double* out) {
  double lv[3];
  mulMV(a.L, v, lv);
  for (int i = 0; i < 3; ++i) out[i] = lv[i] + a.t[i];
}
inline double rotationAngle(const double* v1, const double* v2, int sign) {
  const double dot = (v1[0] * v2[0] + v1[1] * v2[1]) + v1[2] * v2[2];
  const double n1 = sqrt((v1[0] * v1[0] + v1[1] * v1[1]) + v1[2] * v1[2]);
  const double n2 = sqrt((v2[0] * v2[0] + v2[1] * v2[1]) + v2[2] * v2[2]);
  const double magnitude = n1 * n2;
  return magnitude == 0 ? 0 : sign * acos(dot / magnitude);
}
// transformRig(rig, rotation, 0, 1): every camera's forward / up / right (rows of its current rotation) and origin
inline bool transformRig(DerpCameraDesc* cams, int n, const double* rotation) {
  const double zero[3] = {0, 0, 0};
  const Affine rot = generateTransform(rotation, zero), xform = generateTransform(rotation, zero);
  for (int i = 0; i < n; ++i) {
    DevCamera c;
    if (!derp::host::makeCamera(cams[i], &c)) return false;
    const double fwd[3] = {-c.rot[6], -c.rot[7], -c.rot[8]}, up[3] = {c.rot[3], c.rot[4], c.rot[5]},
                 right[3] = {c.rot[0], c.rot[1], c.rot[2]};
    apply(rot, fwd, cams[i].forward);
    apply(rot, up, cams[i].up);
    apply(rot, right, cams[i].right);
    double pos[3];
    apply(xform, cams[i].origin, pos);
    for (int k = 0; k < 3; ++k) cams[i].origin[k] = pos[k];
  }
  return true;
}
inline bool centerRig(DerpCameraDesc* cams, int n, int sel) {
  const double centerOfEquirect[3] = {-1, 0, 0}, upwards[3] = {0, 0, 1};
  DevCamera c;
  if (!derp::host::makeCamera(cams[sel], &c)) return false;
  const double proj1[3] = {-c.rot[6], -c.rot[7], 0};
  const double phi = rotationAngle(centerOfEquirect, proj1, -c.rot[7] > 0 ? 1 : -1);
  const double r1[3] = {0, 0, phi};
  if (!transformRig(cams, n, r1) || !derp::host::makeCamera(cams[sel], &c)) return false;
  const double proj2[3] = {-c.rot[6], 0, -c.rot[8]};
  const double psi = rotationAngle(centerOfEquirect, proj2, -c.rot[8] > 0 ? -1 : 1);
  const double r2[3] = {0, psi, 0};
  if (!transformRig(cams, n, r2) || !derp::host::makeCamera(cams[sel], &c)) return false;
  const double proj3[3] = {0, c.rot[4], c.rot[5]};
  const double theta = rotationAngle(upwards, proj3, c.rot[4] > 0 ? 1 : -1);
  const double r3[3] = {theta, 0, 0};
  return transformRig(cams, n, r3);
}

}  // namespace host
}  // namespace sweep
}  // namespace derp
