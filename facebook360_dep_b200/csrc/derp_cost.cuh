// Device-side matching cost of the depth path: computeCost (Derp.cpp:104-226) with computeSSD
// (DerpUtil.cpp:126-162) and cv_util::getPixelBilinear (CvUtil.h:78-120) fused into one function.
//
// Arithmetic contract (bit-exactness with the reference CPU path):
//   * fp64 projection in the reference's operation order, -fmad=false;
//   * fp32 bilinear weights ((1-xw)*(1-yw))*p00 + (xw*(1-yw))*p01 + ((1-xw)*yw)*p10 + (xw*yw)*p11,
//     summed left to right, then truncated to integer (bilerp<ushort> returns ushort);
//   * SSD accumulation order dx outer / dy inner / channel 0..2, cv::Matx::dot order;
//   * robust camera mean in libstdc++'s nth_element order (derp_select.cuh).
//
// HBM layout: the source colour images are W*H texels of 4 x u16 (B,G,R,0) = 8 B; the per-destination
// pair tables the cost reads (projColor, projBias) hold the same integer values pre-converted to
// float4 (B,G,R,0) = one aligned 128-bit load per texel and no u16->f32 conversion in the inner loop
// (the sweep is instruction-issue bound, not bandwidth bound); warp tables are
// W*H x float2.
#pragma once

#include <cfloat>
#include <cstdint>

#include "derp_camera.cuh"
#include "derp_select.cuh"

namespace derp {

// Rig size limit: evalCost's visibility mask is one machine word, 32 bits (uint32_t) for rigs of up to kNarrowMaxCams
// cameras and 64 bits (uint64_t) above; every kernel that evaluates costs is instantiated for both (costKernels in
// derp_b200.cu picks one per rig).
constexpr int kMaxCams = 64;
constexpr int kNarrowMaxCams = 32;
constexpr float kMinVarF = 1.0f / 12.0f / 65025.0f;  // DerpUtil.h:32

// One (frame, level, destination) as the cost function sees it.
struct CostView {
  int W, H, S, self;
  const float4* projColor;  // [S][H][W] texels (self slot = the destination's own colour)
  const float4* projBias;   // [S][H][W]
  // The same two tables as 4 x u16 (B,G,R,R of the texel below) = 8 B per texel, for the compacted fine-level
  // kernels: their gathers are scattered (list entries of one warp span several image rows) and L1-tag bound, and
  // half-size texels halve the cache lines a request touches; the conversion costs 4 instructions per texel.
  const uint2* projColor16;
  const uint2* projBias16;
  const unsigned* selTab;  // robustSumTable's permutation table (derp_select.cuh)
  const float2* projWarp;   // [S][H][W]  src px -> dst px at infinity (self slot unused)
  const float* variance;    // destination's own variance [H][W]
  const DevCamera* cams;    // [S] normalised cameras (global memory; staged to smem by kernels)
  // 1.0f and 2^23 passed as kernel parameters: they reach the two-lane arithmetic as constant-bank /
  // uniform-register operands, and because ptxas cannot see their values it can neither fold
  // fma(p, one, q) back into an add nor contract it with the multiply that produced p (see f32x2 notes).
  float one, b23;
};

// The per-destination block every cost kernel's arguments begin with (DerpCtx::dstArgs builds it on the host).
struct DstArgs {
  CostView v;
  const uint8_t* fov;
  const uint8_t* fg;  // nullable (all-pass)
  const float* bg;    // nullable unless foreground masks are used
};

__device__ __forceinline__ int clampIdx(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

// u16 -> float without the conversion pipe: 0x4B000000 | u is the float 2^23 + u exactly.
__device__ __forceinline__ float u16lo(uint32_t w) {
  return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7610)) - 8388608.0f;
}
__device__ __forceinline__ float u16hi(uint32_t w) {
  return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7632)) - 8388608.0f;
}
// (ushort)v for 0 <= v < 2^23, returned as the float 2^23 + trunc(v): adding 2^23 with
// round-toward-zero drops the fraction.  The cost only ever uses DIFFERENCES of such truncated values
// and integer texels, so everything on the dst side is biased by 2^23 as well (exact: all values are
// integers below 2^24) and the second FADD is never needed.
constexpr float kBias23 = 8388608.0f;
__device__ __forceinline__ float truncBiased(float v) { return __fadd_rz(v, kBias23); }

struct Texel {
  float b, g, r;
};
__device__ __forceinline__ Texel unpack(uint2 t) { return Texel{u16lo(t.x), u16hi(t.x), u16lo(t.y)}; }

// bilerp (CvUtil.h:83-86) for one channel, float result
__device__ __forceinline__ float bilerp1(float p00, float p01, float p10, float p11, float w00, float w01,
                                         float w10, float w11) {
  return w00 * p00 + w01 * p01 + w10 * p10 + w11 * p11;  // left-to-right, no FMA (-fmad=false)
}

__device__ __forceinline__ Texel texelOf(float4 t) { return Texel{t.x, t.y, t.z}; }

// One table texel as float4 (B, G, R, R-below), from either table format.  u16 -> f32 is exact.
__device__ __forceinline__ float4 ldTexel(const float4* p) { return __ldg(p); }
__device__ __forceinline__ float4 ldTexel(const uint2* p) {
  const uint2 t = __ldg(p);
  return make_float4((float)(t.x & 0xffffu), (float)(t.x >> 16), (float)(t.y & 0xffffu), (float)(t.y >> 16));
}
template <class TX>
struct TablesOf;
template <>
struct TablesOf<float4> {
  static __device__ __forceinline__ const float4* color(const CostView& v) { return v.projColor; }
  static __device__ __forceinline__ const float4* bias(const CostView& v) { return v.projBias; }
};
template <>
struct TablesOf<uint2> {
  static __device__ __forceinline__ const uint2* color(const CostView& v) { return v.projColor16; }
  static __device__ __forceinline__ const uint2* bias(const CostView& v) { return v.projBias16; }
};

// getPixelBilinear on a Vec3w image: per-channel truncated result (CvUtil.h:90-120), biased by 2^23.
// Generic path: per-tap clamp-to-edge.
template <class TX>
__device__ __forceinline__ Texel sampleTexelTruncBiased(const TX* __restrict__ img, int W, int H, float x, float y) {
  const float xf = roundf(x), yf = roundf(y);
  const int xi = (int)xf, yi = (int)yf;
  const int x0 = clampIdx(xi - 1, W - 1), x1 = clampIdx(xi, W - 1);
  const int y0 = clampIdx(yi - 1, H - 1), y1 = clampIdx(yi, H - 1);
  const float xw = x - xf + 0.5f, yw = y - yf + 0.5f;
  const float w00 = (1 - xw) * (1 - yw), w01 = xw * (1 - yw), w10 = (1 - xw) * yw, w11 = xw * yw;
  const Texel p00 = texelOf(ldTexel(img + (size_t)y0 * W + x0));
  const Texel p01 = texelOf(ldTexel(img + (size_t)y0 * W + x1));
  const Texel p10 = texelOf(ldTexel(img + (size_t)y1 * W + x0));
  const Texel p11 = texelOf(ldTexel(img + (size_t)y1 * W + x1));
  Texel o;
  o.b = truncBiased(bilerp1(p00.b, p01.b, p10.b, p11.b, w00, w01, w10, w11));
  o.g = truncBiased(bilerp1(p00.g, p01.g, p10.g, p11.g, w00, w01, w10, w11));
  o.r = truncBiased(bilerp1(p00.r, p01.r, p10.r, p11.r, w00, w01, w10, w11));
  return o;
}

// getPixelBilinear on a Vec2f image (float result, no truncation)
__device__ __forceinline__ float2 sampleWarp(const float2* __restrict__ img, int W, int H, float x, float y) {
  const float xf = roundf(x), yf = roundf(y);
  const int xi = (int)xf, yi = (int)yf;
  const int x0 = clampIdx(xi - 1, W - 1), x1 = clampIdx(xi, W - 1);
  const int y0 = clampIdx(yi - 1, H - 1), y1 = clampIdx(yi, H - 1);
  const float xw = x - xf + 0.5f, yw = y - yf + 0.5f;
  const float w00 = (1 - xw) * (1 - yw), w01 = xw * (1 - yw), w10 = (1 - xw) * yw, w11 = xw * yw;
  const float2 p00 = __ldg(img + (size_t)y0 * W + x0);
  const float2 p01 = __ldg(img + (size_t)y0 * W + x1);
  const float2 p10 = __ldg(img + (size_t)y1 * W + x0);
  const float2 p11 = __ldg(img + (size_t)y1 * W + x1);
  float2 o;
  o.x = bilerp1(p00.x, p01.x, p10.x, p11.x, w00, w01, w10, w11);
  o.y = bilerp1(p00.y, p01.y, p10.y, p11.y, w00, w01, w10, w11);
  return o;
}

// getPixelBilinear on a float image
__device__ __forceinline__ float sampleF32(const float* __restrict__ img, int W, int H, float x, float y) {
  const float xf = roundf(x), yf = roundf(y);
  const int xi = (int)xf, yi = (int)yf;
  const int x0 = clampIdx(xi - 1, W - 1), x1 = clampIdx(xi, W - 1);
  const int y0 = clampIdx(yi - 1, H - 1), y1 = clampIdx(yi, H - 1);
  const float xw = x - xf + 0.5f, yw = y - yf + 0.5f;
  const float w00 = (1 - xw) * (1 - yw), w01 = xw * (1 - yw), w10 = (1 - xw) * yw, w11 = xw * yw;
  return bilerp1(img[(size_t)y0 * W + x0], img[(size_t)y0 * W + x1], img[(size_t)y1 * W + x0],
                 img[(size_t)y1 * W + x1], w00, w01, w10, w11);
}

// ---- two-lane fp32 arithmetic -------------------------------------------------------------------------------
// The sweep is instruction-issue bound and ~40 % of its instructions are the fp32 mul/add of the
// truncated-bilinear SSD, which pairs channels (B, G) and the R samples of two rows as two lanes.  Hopper has no
// packed fp32 instruction, so each two-lane helper issues two scalar IEEE fp32 operations with explicit rounding
// (__fmul_rn / __fadd_rn / __fsub_rn / __fadd_rz / __fmaf_rn, which the compiler never contracts or re-associates):
// the results are bit-identical to the scalar reference arithmetic.  An add whose operand is a product is written as
// fma(p, one, q) with an opaque one (CostView::one): RN(p*1+q) == RN(p+q) exactly, and an FMA cannot absorb a second
// multiply.  The lane pairs still reach the arithmetic through 64-bit shared-memory loads of the float2 tile planes.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ float lo2(f32x2 v) { return v.x; }
__device__ __forceinline__ float hi2(f32x2 v) { return v.y; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 addrz2(f32x2 a, f32x2 b) { return make_float2(__fadd_rz(a.x, b.x), __fadd_rz(a.y, b.y)); }
__device__ __forceinline__ f32x2 addp2(f32x2 p, f32x2 q, f32x2 one2) {  // p + q where p and/or q are products
  return make_float2(__fmaf_rn(p.x, one2.x, q.x), __fmaf_rn(p.y, one2.y, q.y));
}
__device__ __forceinline__ float addp(float p, float q, float one) { return __fmaf_rn(p, one, q); }

// bilerp of CvUtil.h:83-86 on two lanes: ((w00*p00 + w01*p01) + w10*p10) + w11*p11, per-lane RN after every op
__device__ __forceinline__ f32x2 bilerp2(f32x2 p00, f32x2 p01, f32x2 p10, f32x2 p11, f32x2 w00, f32x2 w01, f32x2 w10,
                                         f32x2 w11, f32x2 one2) {
  f32x2 s = addp2(mul2(p01, w01), mul2(p00, w00), one2);
  s = addp2(mul2(p10, w10), s, one2);
  return addp2(mul2(p11, w11), s, one2);
}

// ---- destination patch tile in shared memory ----------------------------------------------------------
// The 3x3 dst colour patches of a CTA's 32x8 pixels overlap: one (32+2)x(8+2) tile of the destination's
// own colour (+2^23, see truncBiased) serves all of them and keeps 27 values per thread out of registers.
// Two float2 planes so that the two-lane arithmetic gets its operands with 64-bit shared loads:
//   bg[row][col] = (B, G),   rr[row][col] = (R(row), R(row+1))   (vertical pair: see the R channel below)
constexpr int kTileW = 32 + 2;
constexpr int kSweepMaxRows = 20;  // tallest CTA the sweep is launched with (32 x 20 threads => 96 registers, 20 warps/SM)
constexpr int kMaxTileH = kSweepMaxRows + 2;
constexpr int kTileFloats = 2 * kMaxTileH * kTileW * 2;

// `addend`: 2^23 for the exact cost (see truncBiased), 0.5 for the lower-bound pass (midpoint of the truncation interval).
__device__ __forceinline__ void loadDstTile(float* tile, const CostView& v, int x0, int y0, float addend = kBias23) {
  const float4* col = v.projColor + (size_t)v.self * v.W * v.H;
  float2* bg = reinterpret_cast<float2*>(tile);
  const int tileH = blockDim.y + 2;
  float2* rr = bg + tileH * kTileW;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  for (int i = tid; i < kTileW * tileH; i += nt) {
    const int ty = i / kTileW, tx = i - ty * kTileW;
    const int gx = clampIdx(x0 + tx - 1, v.W - 1), gy = clampIdx(y0 + ty - 1, v.H - 1);
    const int gy1 = clampIdx(y0 + ty, v.H - 1);
    const float4 t = __ldg(col + (size_t)gy * v.W + gx);
    const float4 t1 = __ldg(col + (size_t)gy1 * v.W + gx);
    bg[i] = make_float2(t.x + addend, t.y + addend);
    rr[i] = make_float2(t.z + addend, t1.z + addend);
  }
  __syncthreads();
}

// Candidate-independent state of one destination pixel.
struct PixelState {
  const float2* bg;    // &bg[threadIdx.y][threadIdx.x]: patch(dx,dy) = bg[(dy+1)*kTileW + dx+1]
  const float2* rr;    // same indexing, (R(dy), R(dy+1))
  float dBias[3];      // projColorBias(dst,self)(y,x) + 2^23
  float conf;          // max(variance(y,x), kMinVar)
  double dir[3];       // ray direction of the pixel in rig space
  float2* sel;         // this thread's (ssdB, ssdU) slots in shared memory: entry i at sel[i * selStride]
  int selStride;       // = threads per CTA
};

// The per-source (biased, unbiased) SSD pairs of one cost evaluation live in shared memory, [slot][thread]: S - 1
// slots per thread, sized at launch (16 cameras, 640-thread sweep CTA: 75 KB).  kSelSlots = how many of them the
// table-driven selection covers.
constexpr int kSelSlots = 8;
struct SmemPairs {
  float2* p;
  int stride;
  __device__ __forceinline__ PairVal get(int i) const {
    const float2 t = p[i * stride];
    return PairVal{t.x, t.y};
  }
  __device__ __forceinline__ void set(int i, PairVal v) const { p[i * stride] = make_float2(v.a, v.b); }
};

__device__ __forceinline__ void loadPixelState(const CostView& v, const DevCamera& camDst, const float* tile, int x,
                                               int y, PixelState& ps, float addend = kBias23) {
  ps.bg = reinterpret_cast<const float2*>(tile) + threadIdx.y * kTileW + threadIdx.x;
  ps.rr = ps.bg + (blockDim.y + 2) * kTileW;
  ps.selStride = blockDim.x * blockDim.y;
  ps.sel = reinterpret_cast<float2*>(const_cast<float*>(tile) + kTileFloats) + threadIdx.y * blockDim.x + threadIdx.x;
  const float4 tb = __ldg(v.projBias + (size_t)v.self * v.W * v.H + (size_t)y * v.W + x);
  ps.dBias[0] = tb.x + addend;
  ps.dBias[1] = tb.y + addend;
  ps.dBias[2] = tb.z + addend;
  ps.conf = fmaxf(__ldg(v.variance + (size_t)y * v.W + x), kMinVarF);
  // dstToWorldPoint (DerpUtil.cpp:38-52): normalised pixel centre, ray through it
  const double px = (x + 0.5) / v.W, py = (y + 0.5) / v.H;
  pixelRay(camDst, px, py, ps.dir);
}

// Compacted kernels (one thread per ACTIVE pixel, pixels of a CTA are not a rectangle): every thread keeps its
// own 3x3 patch in shared memory, laid out [row][col][thread] so that a warp reads consecutive words.
constexpr int kPatchThreads = 256;
// Resident CTAs per SM the compacted kernels are compiled for (register cap).  2 => 128 registers, 16 warps/SM: these
// kernels are L1-bound (scattered 4x4 gathers), so spill traffic costs more than the lost warps.
constexpr int kPatchMinCtas = 2;
constexpr int kPatchRP = 3 * kPatchThreads, kPatchCP = kPatchThreads;
constexpr int kPatchFloats = 2 * 9 * kPatchThreads * 2;
// pingPongKernel has its own CTA shape: 128 threads x 5 CTAs per SM (96 registers, 20 warps/SM), while proposalKernel
// keeps 256 x 2 (it spills more at 96 registers).
constexpr int kPingThreads = 128;
constexpr int kPingMinCtas = 5;

template <int T>
__device__ __forceinline__ void loadPixelStateCompact(const CostView& v, const DevCamera& camDst, float* patches, int x,
                                                      int y, PixelState& ps) {
  const int tid = threadIdx.x;
  float2* bg = reinterpret_cast<float2*>(patches) + tid;
  float2* rr = bg + 9 * T;
  const uint2* col = v.projColor16 + (size_t)v.self * v.W * v.H;  // u16 -> f32 is exact
  float rz[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {  // rows y-1 .. y+1 (interior pixel: always in bounds)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4 t = ldTexel(col + (size_t)(y - 1 + r) * v.W + (x - 1 + c));
      bg[r * (3 * T) + c * T] = make_float2(t.x + kBias23, t.y + kBias23);
      // rr[r] = (R(row r), R(row r+1)); the fast path reads rr[0] (both lanes) and rr[2].x, the slow path rr[r].x
      if (r >= 1) rr[(r - 1) * (3 * T) + c * T] = make_float2(rz[c] + kBias23, t.z + kBias23);
      if (r == 2) rr[2 * (3 * T) + c * T] = make_float2(t.z + kBias23, 0.f);
      rz[c] = t.z;
    }
  }
  ps.bg = bg;
  ps.rr = rr;
  ps.selStride = T;
  ps.sel = reinterpret_cast<float2*>(patches + 2 * 9 * T * 2) + tid;
  const float4 tb = ldTexel(v.projBias16 + (size_t)v.self * v.W * v.H + (size_t)y * v.W + x);
  ps.dBias[0] = tb.x + kBias23;
  ps.dBias[1] = tb.y + kBias23;
  ps.dBias[2] = tb.z + kBias23;
  ps.conf = fmaxf(__ldg(v.variance + (size_t)y * v.W + x), kMinVarF);
  const double px = (x + 0.5) / v.W, py = (y + 0.5) / v.H;
  pixelRay(camDst, px, py, ps.dir);
}

// The same for the refine pass of the filtered sweep: list entries of the DENSE level, so patches and bias come from the
// float4 tables the sweep already built.
__device__ __forceinline__ void loadPixelStateCompactF32(const CostView& v, const DevCamera& camDst, float* patches, int x,
                                                         int y, PixelState& ps) {
  const int tid = threadIdx.x;
  float2* bg = reinterpret_cast<float2*>(patches) + tid;
  float2* rr = bg + 9 * kPatchThreads;
  const float4* col = v.projColor + (size_t)v.self * v.W * v.H;
  float rz[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4 t = __ldg(col + (size_t)(y - 1 + r) * v.W + (x - 1 + c));
      bg[r * kPatchRP + c * kPatchCP] = make_float2(t.x + kBias23, t.y + kBias23);
      if (r >= 1) rr[(r - 1) * kPatchRP + c * kPatchCP] = make_float2(rz[c] + kBias23, t.z + kBias23);
      if (r == 2) rr[2 * kPatchRP + c * kPatchCP] = make_float2(t.z + kBias23, 0.f);
      rz[c] = t.z;
    }
  }
  ps.bg = bg;
  ps.rr = rr;
  ps.selStride = kPatchThreads;
  ps.sel = reinterpret_cast<float2*>(patches + kPatchFloats) + tid;
  const float4 tb = __ldg(v.projBias + (size_t)v.self * v.W * v.H + (size_t)y * v.W + x);
  ps.dBias[0] = tb.x + kBias23;
  ps.dBias[1] = tb.y + kBias23;
  ps.dBias[2] = tb.z + kBias23;
  ps.conf = fmaxf(__ldg(v.variance + (size_t)y * v.W + x), kMinVarF);
  const double px = (x + 0.5) / v.W, py = (y + 0.5) / v.H;
  pixelRay(camDst, px, py, ps.dir);
}

// isOutsideFov (Camera.h:154-164) for a world point; true = the cone test passes (camera may see it)
__device__ __forceinline__ bool insideCone(const DevCamera& c, double wx, double wy, double wz) {
  if (c.cosFov == -1) return true;
  const double vx = wx - c.pos[0], vy = wy - c.pos[1], vz = wz - c.pos[2];
  const double camz = c.rot[6] * vx + c.rot[7] * vy + c.rot[8] * vz;
  if (c.cosFov == 0) return !(camz >= 0);  // !isBehind
  const double dot = -camz;
  const double n2 = vx * vx + vy * vy + vz * vz;
  return !(dot * fabs(dot) <= c.cosFov * fabs(c.cosFov) * n2);
}

// pixel() + isOutsideSensor + de-normalisation + narrowing (Camera.h:121-128,180-190, DerpUtil.cpp:56-73,
// Derp.cpp:175) for a point that already passed the cone test.  Straight-line code (no early exit) so that
// the scheduler can interleave it with the fp32 SSD of the previous source.
struct SrcPoint {
  float x, y;
  bool ok;
};
__device__ __forceinline__ SrcPoint projectToSource(const DevCamera& c, double wx, double wy, double wz, int W, int H) {
  const double vx = wx - c.pos[0], vy = wy - c.pos[1], vz = wz - c.pos[2];
  const double camx = c.rot[0] * vx + c.rot[1] * vy + c.rot[2] * vz;
  const double camy = c.rot[3] * vx + c.rot[4] * vy + c.rot[5] * vz;
  const double camz = c.rot[6] * vx + c.rot[7] * vy + c.rot[8] * vz;
  double sx, sy;
  cameraToSensor(c, camx, camy, camz, &sx, &sy);
  double px = c.focal[0] * sx + c.principal[0];
  double py = c.focal[1] * sy + c.principal[1];
  SrcPoint o;
  o.ok = !(0 > px || px >= c.res[0] || 0 > py || py >= c.res[1]);
  px *= W;  // worldToSrcPoint: de-normalise (cameras are normalised, DerpUtil.cpp:67-71)
  py *= H;
  o.x = (float)px;
  o.y = (float)py;
  return o;
}

// Generic (border / inconsistent-rounding / invalid) path of one source: returns false if the source
// contributes no SSD (warp entry NaN).  Kept out of line: it runs for a few pixels per image.
template <class TX>
__device__ __noinline__ bool ssdSlowPath(const TX* __restrict__ srcColor, const TX* __restrict__ srcBiasImg,
                                         int W, int H, const float2* bg, const float2* rr, int rowPitch, int colPitch,
                                         float dBias0, float dBias1, float dBias2, float xDstSrc, float yDstSrc,
                                         float* ssdB, float* ssdU) {
  if (isnan(xDstSrc) || isnan(yDstSrc)) return false;
  const Texel sbias = sampleTexelTruncBiased(srcBiasImg, W, H, xDstSrc, yDstSrc);
  const float bias0 = dBias0 - sbias.b, bias1 = dBias1 - sbias.g, bias2 = dBias2 - sbias.r;
  float sB = 0.0f, sU = 0.0f;
  for (int dx = -1; dx <= 1; ++dx)
    for (int dy = -1; dy <= 1; ++dy) {
      const Texel cs = sampleTexelTruncBiased(srcColor, W, H, xDstSrc + (float)dx, yDstSrc + (float)dy);
      const float2 pbg = bg[(dy + 1) * rowPitch + (dx + 1) * colPitch];
      const float pr = rr[(dy + 1) * rowPitch + (dx + 1) * colPitch].x;
      const float d0 = pbg.x - cs.b, d1 = pbg.y - cs.g, d2 = pr - cs.r;
      const float u0 = d0 - bias0, u1 = d1 - bias1, u2 = d2 - bias2;
      sB += d0 * d0 + d1 * d1 + d2 * d2;
      sU += u0 * u0 + u1 * u1 + u2 * u2;
    }
  const float scaleFactor = 1.0f / (65535.0f * 65535.0f);
  *ssdB = sB * scaleFactor;
  *ssdU = sU * scaleFactor;
  return true;
}

// roundf(p) for both lanes of p when 0 <= p < 2^22, returned biased by 2^23 (so the integer index is a
// plain integer subtract of the bit patterns): floor(RZ(p + .5)) == floor(p + .5) == roundf(p) for p >= 0.
__device__ __forceinline__ f32x2 roundBiased2(f32x2 p, f32x2 half2, f32x2 b23) { return addrz2(addrz2(p, half2), b23); }


// ---- lower-bound pass of the filtered sweep (derp_refine.cuh) ------------------------------------------------------
// Per sample and channel the reference computes t = (ushort) fl32(bilerp) (CvUtil.h:83-120).  The cheap path computes
// a = fma-based separable bilerp of the SAME four texels with the SAME fp32 weights.  Bounds (texels in [0, 65535],
// weights in [0, 1], u = 2^-24):
//   |fl32(bilerp) - V| <= 0.0273   (V = the real-valued bilerp: three roundings per weight, one per product, three adds)
//   |a - V|            <= 0.0234   (three fused lerps on exact integer differences)
//   t in (fl32(bilerp) - 1, fl32(bilerp)]
// so with the midpoint m = a - 0.5:  |t - m| <= 0.5 + 0.0507, and after the two fp32 subtractions that form the
// difference against the destination texel (+0.5) and the bias: |e_d| <= 0.56 per term, |e_bias| <= 0.56.
// Over the 27 terms of one source: ||d|| >= ||d'|| - ||e_d||, ||e_d|| <= 0.56 sqrt(27) < 2.91 (reverse triangle
// inequality in l2), and for the bias-compensated differences ||e_u|| <= 2 * 2.91.  (kErrB and kErrU are the constants of
// the full-patch sums; tests/test_lower_bound_model.py checks the per-term claims and both aggregates.)
constexpr float kErrB = 2.91f;
constexpr float kErrU = 5.82f;
// The pass bounds only the bias-compensated sum, and from the six samples of the rows dy = 0 and dy = +1 alone: their 18
// terms are a subset of the 27 non-negative terms of the exact sum, so their exact sum bounds it from below, and the
// l2 error of those 18 terms is ||e_u|| <= 2 * 0.56 sqrt(18) < 4.76 (tests/test_lower_bound_row_model.py).  The
// relative errors (fp32 sums, sqrt.approx) are covered by the final factor 1 - 2^-16 (KeptBound).
constexpr float kErrURows = 4.76f;

__device__ __forceinline__ float sqrtApprox(float x) {  // MUFU.SQRT, relative error < 2^-22: covered by the slack of kErr*
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
// a + w (b - a), both lanes
__device__ __forceinline__ f32x2 lerp2(f32x2 a, f32x2 b, f32x2 w) { return fma2(w, sub2(b, a), a); }
__device__ __forceinline__ float lerp1(float a, float b, float w) { return __fmaf_rn(w, b - a, a); }

// Bias-compensated sum of squared differences of one source over the sample rows dy = 0 and dy = +1 of the 3x3 patch,
// cheap version: texel rows r1..r3 of the 4x4 block (4 texels each; the R lanes (z, w) of rows r1 and r2 carry R of
// rows (r1, r2) and (r2, r3)), the bias block at b1, per-sample weights W0..W2 = (xw, yw) of d = -1, 0, +1.  Every
// sample, bias and difference is formed exactly as in the error analysis above (x-lerps, then the y-lerp, then the two
// subtractions), so each of the 18 terms is within 0.56 of the exact path's.  The destination patch tile and ps.dBias
// carry +0.5 (loadDstTile / loadPixelState with addend 0.5).
template <int RP, int CP>
__device__ __forceinline__ float ssdLowerRows(const float4* r1, const float4* r2, const float4* r3, const float4* b1,
                                             int W, const PixelState& ps, f32x2 W0, f32x2 W1, f32x2 W2) {
  const float xw[3] = {lo2(W0), lo2(W1), lo2(W2)};
  const float yw1 = hi2(W1), yw2 = hi2(W2);  // y weights of the rows dy = 0 and dy = +1
  const f32x2 wy1 = pk(yw1, yw1), wy2 = pk(yw2, yw2);
  // bias sample (centre sample's footprint): (B, G) packed, R scalar
  f32x2 biasBG;
  float biasR;
  {
    const float4 q00 = __ldg(b1), q01 = __ldg(b1 + 1), q10 = __ldg(b1 + W), q11 = __ldg(b1 + W + 1);
    const f32x2 wx2 = pk(xw[1], xw[1]);
    const f32x2 top = lerp2(pk(q00.x, q00.y), pk(q01.x, q01.y), wx2);
    const f32x2 bot = lerp2(pk(q10.x, q10.y), pk(q11.x, q11.y), wx2);
    biasBG = sub2(pk(ps.dBias[0], ps.dBias[1]), lerp2(top, bot, wy1));
    biasR = ps.dBias[2] - lerp1(lerp1(q00.z, q01.z, xw[1]), lerp1(q10.z, q11.z, xw[1]), yw1);
  }
  f32x2 acc = pk(0.f, 0.f);
  float accR = 0.f;
  float4 A1 = __ldg(r1), A2 = __ldg(r2), A3 = __ldg(r3);
#pragma unroll
  for (int c = 0; c < 3; ++c) {  // dx = c - 1: texel columns c and c + 1
    const float4 B1 = __ldg(r1 + c + 1), B2 = __ldg(r2 + c + 1), B3 = __ldg(r3 + c + 1);
    const f32x2 wx2 = pk(xw[c], xw[c]);
    const f32x2 x1 = lerp2(pk(A1.x, A1.y), pk(B1.x, B1.y), wx2), x2 = lerp2(pk(A2.x, A2.y), pk(B2.x, B2.y), wx2);
    const f32x2 x3 = lerp2(pk(A3.x, A3.y), pk(B3.x, B3.y), wx2);
    const f32x2 xr12 = lerp2(pk(A1.z, A1.w), pk(B1.z, B1.w), wx2), xr23 = lerp2(pk(A2.z, A2.w), pk(B2.z, B2.w), wx2);
    // row dy = 0 (texel rows r1, r2), then row dy = +1 (texel rows r2, r3)
    const f32x2 s1 = lerp2(x1, x2, wy1), s2 = lerp2(x2, x3, wy2);
    const float sr1 = lerp1(lo2(xr12), hi2(xr12), yw1), sr2 = lerp1(lo2(xr23), hi2(xr23), yw2);
    const f32x2 u1 = sub2(sub2(*reinterpret_cast<const f32x2*>(ps.bg + 1 * RP + c * CP), s1), biasBG);
    const f32x2 u2 = sub2(sub2(*reinterpret_cast<const f32x2*>(ps.bg + 2 * RP + c * CP), s2), biasBG);
    const float ur1 = (ps.rr[1 * RP + c * CP].x - sr1) - biasR, ur2 = (ps.rr[2 * RP + c * CP].x - sr2) - biasR;
    acc = fma2(u1, u1, acc);
    accR = __fmaf_rn(ur1, ur1, accR);
    acc = fma2(u2, u2, acc);
    accR = __fmaf_rn(ur2, ur2, accR);
    A1 = B1;
    A2 = B2;
    A3 = B3;
  }
  return (lo2(acc) + hi2(acc)) + accR;
}

// Lower bound of computeCost's result from per-source lower bounds of the unbiased sums (before the 1/65535^2 scale),
// accumulated as the sources arrive.  The reference keeps the `keep` = max(1, n - 2) sources with the smallest
// (biased, unbiased) pairs (Derp.cpp:204-215); whichever they are, their unbiased sums add up to at least the sum of the
// `keep` smallest lower bounds, so no kept-set decision is needed.  `rest` adds every bound that leaves, or never
// enters, the two largest: only kept-size bounds are summed, never a total minus the dropped ones, whose rounding (half
// an ulp of the total, up to 2^14 when a dropped source mismatches at full scale) could exceed a small kept sum.  With
// non-negative terms only, the factor 1 - 2^-16 covers the fp32 roundings of both computations (sums, scale, the two
// divisions and the multiplication of Derp.cpp:216-225: < 5e-6 relative together).
struct KeptBound {
  float t1 = 0.f, t2 = 0.f;  // the two largest lower bounds
  float rest = 0.f;          // sum of the others
  __device__ __forceinline__ void push(float b) {
    rest += fminf(b, t2);
    if (b > t1) {
      t2 = t1;
      t1 = b;
    } else if (b > t2) {
      t2 = b;
    }
  }
  __device__ __forceinline__ float cost(int n, int keep, float conf) const {
    const float kept = n == 1 ? t1 : (n == 2 ? t2 : rest);
    const float scaleFactor = 1.0f / (65535.0f * 65535.0f);
    const float k = (float)keep;
    return ((kept * scaleFactor) / k) * (1.0f / k) / conf * 0.9999847412109375f;  // 1 - 2^-16
  }
};

// Index of the lowest set bit of a non-zero visibility mask.
__device__ __forceinline__ int lowestSetBit(uint32_t m) { return __ffs(m) - 1; }
__device__ __forceinline__ int lowestSetBit(uint64_t m) { return __ffsll(m) - 1; }

// computeCost (Derp.cpp:104-226).  `cams` points to shared memory.  Returns the cost; confidence is
// ps.conf when the return value is not FLT_MAX, 0 otherwise.
// Mask: the visibility mask's type, one bit per camera: uint32_t for rigs of up to 32 cameras, uint64_t up to 64.
//
// Structure (instruction-issue bound kernel):
//   phase A  cone test of every source -> bitmask (short independent fp64 chains, unrolled);
//   phase B  for each set bit: the fp64 projection of the NEXT source is issued in the same basic block as
//            the fp32 SSD of the CURRENT one, so the long dependent fp64 chain (sqrt, atan2, divide) and the
//            two dependent gathers (warp entry -> 4x4 block) hide behind each other.
// SSD fast path: the 36 taps of the nine 2x2 footprints are one interior 4x4 block read column by column
// (= the reference's accumulation order, dx outer / dy inner).  Channels B,G ride the two lanes of the
// two-lane helpers; channel R rides them as (sample dy=-1, sample dy=0) thanks to the table's w lane
// holding R of the texel below; the dy=+1 R sample is scalar.  Weights are formed per sample exactly like
// the reference, so the result is bit-identical to the generic per-tap path.
// RP / CP: row and column pitch (in float2) of the thread's 3x3 destination patch in shared memory —
// (kTileW, 1) for the dense CTA tile, (3*256, 256) for the per-thread patches of the compacted kernels.
// TX: table texel type (float4 for the dense sweep, uint2 = 4 x u16 for the compacted kernels).
// LOWER = true: the LOWER-BOUND pass of the filtered sweep (derp_refine.cuh).  Visibility, projection, warp fetch and
// sample positions are the exact path's; the SSD is replaced by a lower bound of the bias-compensated sum from two of
// the three sample rows (ssdLowerRows, 16 gathers instead of 20), the selection slots by registers (KeptBound), and the
// return value is a number that is <= the exact cost (0 = "unknown", FLT_MAX = no source).
template <class Mask, int RP, int CP, class TX = float4, bool LOWER = false>
__device__ __forceinline__ float evalCost(const CostView& v, const DevCamera* __restrict__ cams,
                                          const PixelState& ps, float disparity, unsigned* hits) {
  const double depth = (double)(1.0f / disparity);
  const DevCamera& cd = cams[v.self];
  const double wx = cd.pos[0] + ps.dir[0] * depth;
  const double wy = cd.pos[1] + ps.dir[1] * depth;
  const double wz = cd.pos[2] + ps.dir[2] * depth;
  const int W = v.W, H = v.H;
  const size_t plane = (size_t)W * H;
  const float one = v.one, b23 = v.b23;
  const f32x2 one2 = pk(one, one), b232 = pk(b23, b23), half2 = pk(0.5f, 0.5f);

  Mask mask = 0;
#pragma unroll 4
  for (int s = 0; s < v.S; ++s)
    if (insideCone(cams[s], wx, wy, wz)) mask |= Mask(1) << s;
  mask &= ~(Mask(1) << v.self);

  // (biased, unbiased) SSD of every contributing source: this thread's column of the [slot][thread] array in shared
  // memory, S - 1 slots (sized at launch), so no evaluation ever touches local memory.
  int n = 0;
  bool unknown = false;  // LOWER only: a source took the generic (border) path, no bound is formed
  KeptBound kb;          // LOWER only: the per-source lower bounds, accumulated in registers
  auto pushPair = [&](float b, float u) {
    ps.sel[n * ps.selStride] = make_float2(b, u);
    ++n;
  };
  // The four warp-table taps of a projected point (getPixelBilinear on the Vec2f table, CvUtil.h:107-120) and its
  // bilinear weights.  A point inside the sensor has coordinates >= 0, so the RZ rounding applies; for a point
  // outside (!ok) the clamped, harmless fetch result is discarded by the caller.
  struct WarpTaps {
    float2 p00, p01, p10, p11;
    float xw, yw;
  };
  auto fetchWarp = [&](int s, const SrcPoint& sp) {
    const f32x2 P = pk(sp.x, sp.y);
    const f32x2 T = roundBiased2(P, half2, b232);
    const f32x2 Wt = add2(sub2(P, sub2(T, b232)), half2);  // (xw, yw) = p - round(p) + 0.5
    const int wxi = __float_as_int(lo2(T)) - 0x4B000000, wyi = __float_as_int(hi2(T)) - 0x4B000000;
    const float2* wt = v.projWarp + s * plane;
    const int x0 = clampIdx(wxi - 1, W - 1), x1 = clampIdx(wxi, W - 1);
    const int y0 = clampIdx(wyi - 1, H - 1), y1 = clampIdx(wyi, H - 1);
    WarpTaps t;
    t.p00 = __ldg(wt + (size_t)y0 * W + x0);
    t.p01 = __ldg(wt + (size_t)y0 * W + x1);
    t.p10 = __ldg(wt + (size_t)y1 * W + x0);
    t.p11 = __ldg(wt + (size_t)y1 * W + x1);
    t.xw = lo2(Wt);
    t.yw = hi2(Wt);
    return t;
  };
  if (mask) {
    int s = lowestSetBit(mask);
    mask &= mask - 1;
    SrcPoint cur = projectToSource(cams[s], wx, wy, wz, W, H);
    while (true) {
      // Tail (!more): the exact path re-projects the same source, harmlessly, to keep its main block straight-line
      // code.  The lower-bound pass skips that projection: in a warp's last iteration no lane needs it, and measured
      // on the headline sweep the branch costs less than the fp64 projection it saves.
      const int sNext = mask ? lowestSetBit(mask) : s;
      const bool more = mask != 0;
      mask &= mask - 1;
      // ---- current source: warp entry ---------------------------------------------------------------------
      float2 pd;
      {
        const WarpTaps tp = fetchWarp(s, cur);
        const float2 p00 = tp.p00, p01 = tp.p01, p10 = tp.p10, p11 = tp.p11;
        const float xw = tp.xw, yw = tp.yw;
        const float xm = 1 - xw, ym = 1 - yw;
        const f32x2 r = bilerp2(pk(p00.x, p00.y), pk(p01.x, p01.y), pk(p10.x, p10.y), pk(p11.x, p11.y),
                                pk(xm * ym, xm * ym), pk(xw * ym, xw * ym), pk(xm * yw, xm * yw), pk(xw * yw, xw * yw), one2);
        pd.x = lo2(r);
        pd.y = hi2(r);
      }
      const float xDstSrc = pd.x + 0.5f, yDstSrc = pd.y + 0.5f;
      // ---- footprint of the nine samples: (x,y) pairs for d = -1, 0, +1 ----------------------------------
      const f32x2 C = pk(xDstSrc, yDstSrc);
      const f32x2 P0 = add2(C, pk(-1.0f, -1.0f)), P2 = add2(C, pk(1.0f, 1.0f));  // xDstSrc + dx as float adds
      const f32x2 T0 = roundBiased2(P0, half2, b232), T1 = roundBiased2(C, half2, b232), T2 = roundBiased2(P2, half2, b232);
      const f32x2 W0 = add2(sub2(P0, sub2(T0, b232)), half2), W1 = add2(sub2(C, sub2(T1, b232)), half2),
                  W2 = add2(sub2(P2, sub2(T2, b232)), half2);
      const int xi0 = __float_as_int(lo2(T0)) - 0x4B000000, yi0 = __float_as_int(hi2(T0)) - 0x4B000000;
      const int xi1 = __float_as_int(lo2(T1)) - 0x4B000000, yi1 = __float_as_int(hi2(T1)) - 0x4B000000;
      const int xi2 = __float_as_int(lo2(T2)) - 0x4B000000, yi2 = __float_as_int(hi2(T2)) - 0x4B000000;
      const int X0 = xi0 - 1, Y0 = yi0 - 1;
      // the RZ rounding needs 0 <= p < 2^22; NaN fails every comparison -> slow path, which rejects it
      const bool fast = (xDstSrc >= 1.5f) & (yDstSrc >= 1.5f) & (xDstSrc < 4.0e6f) & (yDstSrc < 4.0e6f) &
          (xi1 == xi0 + 1) & (xi2 == xi0 + 2) & (yi1 == yi0 + 1) & (yi2 == yi0 + 2) & (X0 + 3 <= W - 1) & (Y0 + 3 <= H - 1);
      const TX* srcColor = TablesOf<TX>::color(v) + s * plane;
      const TX* srcBiasImg = TablesOf<TX>::bias(v) + s * plane;
      SrcPoint nxt;
      if (cur.ok) {
        if (fast) {
          // ---- main block: 20 gathers + fp32 SSD of source s, fp64 projection of source sNext --------------
          const size_t off = (size_t)Y0 * W + X0;
          const TX* r0 = srcColor + off;
          const TX* r1 = r0 + W;
          const TX* r2 = r1 + W;
          const TX* r3 = r2 + W;
          const TX* b1 = srcBiasImg + off + W + 1;  // bias sample = centre sample's 2x2 footprint
          if constexpr (LOWER) {
            if (more) nxt = projectToSource(cams[sNext], wx, wy, wz, W, H);
            // lower bound of the source's exact unbiased sum, see ssdLowerRows and KeptBound
            const float rU = sqrtApprox(ssdLowerRows<RP, CP>(r1, r2, r3, b1, W, ps, W0, W1, W2));
            const float ul = fmaxf(rU - kErrURows, 0.0f);
            kb.push(ul * ul);
            ++n;
          } else {
          const float4 q00 = ldTexel(b1), q01 = ldTexel(b1 + 1), q10 = ldTexel(b1 + W), q11 = ldTexel(b1 + W + 1);
          float4 colA[4], colB[4];
          colA[0] = ldTexel(r0);
          colA[1] = ldTexel(r1);
          colA[2] = ldTexel(r2);
          colA[3] = ldTexel(r3);
          nxt = projectToSource(cams[sNext], wx, wy, wz, W, H);
          // y weights: per sample row r (dy = r-1): yw, 1-yw; rows 0,1 also as a lane pair for channel R
          const float yw0 = hi2(W0), yw1 = hi2(W1), yw2 = hi2(W2);
          const float ym0 = 1 - yw0, ym1 = 1 - yw1, ym2 = 1 - yw2;
          const f32x2 ywP = pk(yw0, yw1), ymP = pk(ym0, ym1);
          const float xwv[3] = {lo2(W0), lo2(W1), lo2(W2)};
          // bias = float(dstBias) - float(srcBias): both carry +2^23, the difference is exact
          f32x2 biasBG;
          float biasR;
          {
            const float xwc = xwv[1], xwm = 1 - xwc;
            const float w00 = xwm * ym1, w01 = xwc * ym1, w10 = xwm * yw1, w11 = xwc * yw1;
            const f32x2 sbg = addrz2(bilerp2(pk(q00.x, q00.y), pk(q01.x, q01.y), pk(q10.x, q10.y), pk(q11.x, q11.y),
                                            pk(w00, w00), pk(w01, w01), pk(w10, w10), pk(w11, w11), one2), b232);
            biasBG = sub2(pk(ps.dBias[0], ps.dBias[1]), sbg);
            biasR = ps.dBias[2] - truncBiased(bilerp1(q00.z, q01.z, q10.z, q11.z, w00, w01, w10, w11));
          }
          const f32x2 biasRR = pk(biasR, biasR);
          float sB = 0.0f, sU = 0.0f;
#pragma unroll
          for (int c = 0; c < 3; ++c) {  // dx = c-1: texel columns c and c+1
            colB[0] = ldTexel(r0 + c + 1);
            colB[1] = ldTexel(r1 + c + 1);
            colB[2] = ldTexel(r2 + c + 1);
            colB[3] = ldTexel(r3 + c + 1);
            const float xwc = xwv[c], xwm = 1 - xwc;
            const f32x2 xwc2 = pk(xwc, xwc), xwm2 = pk(xwm, xwm);
            // weights of samples dy=-1,0 as pairs (lane = sample), dy=+1 scalar: w00=(1-xw)(1-yw) ...
            const f32x2 w00P = mul2(ymP, xwm2), w01P = mul2(ymP, xwc2), w10P = mul2(ywP, xwm2), w11P = mul2(ywP, xwc2);
            const float w00s = xwm * ym2, w01s = xwc * ym2, w10s = xwm * yw2, w11s = xwc * yw2;
            // channel R of samples dy=-1 and dy=0 in one go: the texels' (z,w) lanes are (R(row), R(row+1))
            const f32x2 sR01 = addrz2(bilerp2(pk(colA[0].z, colA[0].w), pk(colB[0].z, colB[0].w), pk(colA[1].z, colA[1].w),
                                              pk(colB[1].z, colB[1].w), w00P, w01P, w10P, w11P, one2), b232);
            const float sR2 = truncBiased(bilerp1(colA[2].z, colB[2].z, colA[3].z, colB[3].z, w00s, w01s, w10s, w11s));
            const f32x2 pR01 = *reinterpret_cast<const f32x2*>(ps.rr + c * CP);
            const float pR2 = ps.rr[2 * RP + c * CP].x;
            const f32x2 dR01 = sub2(pR01, sR01);
            const f32x2 uR01 = sub2(dR01, biasRR);
            const f32x2 ddR01 = mul2(dR01, dR01), uuR01 = mul2(uR01, uR01);
            const float dR2 = pR2 - sR2, uR2 = dR2 - biasR;
            const float ddR[3] = {lo2(ddR01), hi2(ddR01), dR2 * dR2};
            const float uuR[3] = {lo2(uuR01), hi2(uuR01), uR2 * uR2};
#pragma unroll
            for (int r = 0; r < 3; ++r) {  // dy = r-1: texel rows r and r+1; channels (B,G) on the two lanes
              const float w00 = r == 0 ? lo2(w00P) : (r == 1 ? hi2(w00P) : w00s);
              const float w01 = r == 0 ? lo2(w01P) : (r == 1 ? hi2(w01P) : w01s);
              const float w10 = r == 0 ? lo2(w10P) : (r == 1 ? hi2(w10P) : w10s);
              const float w11 = r == 0 ? lo2(w11P) : (r == 1 ? hi2(w11P) : w11s);
              const f32x2 sBG = addrz2(bilerp2(pk(colA[r].x, colA[r].y), pk(colB[r].x, colB[r].y), pk(colA[r + 1].x, colA[r + 1].y),
                                               pk(colB[r + 1].x, colB[r + 1].y), pk(w00, w00), pk(w01, w01), pk(w10, w10),
                                               pk(w11, w11), one2), b232);
              const f32x2 pBG = *reinterpret_cast<const f32x2*>(ps.bg + r * RP + c * CP);
              const f32x2 dBG = sub2(pBG, sBG);
              const f32x2 uBG = sub2(dBG, biasBG);
              const f32x2 dd = mul2(dBG, dBG), uu = mul2(uBG, uBG);
              // cv::Matx::dot order (d0*d0 + d1*d1) + d2*d2, then ssd += s (DerpUtil.cpp:150-151)
              const float s1 = addp(ddR[r], addp(hi2(dd), lo2(dd), one), one);
              const float s2 = addp(uuR[r], addp(hi2(uu), lo2(uu), one), one);
              sB += s1;
              sU += s2;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) colA[j] = colB[j];
          }
          const float scaleFactor = 1.0f / (65535.0f * 65535.0f);
          pushPair(sB * scaleFactor, sU * scaleFactor);
          }
        } else {
          if (!LOWER || more) nxt = projectToSource(cams[sNext], wx, wy, wz, W, H);
          if constexpr (LOWER) {
            if (!(isnan(xDstSrc) || isnan(yDstSrc))) {  // the source contributes, through the generic path
              unknown = true;
              ++n;
            }
          } else {
            float slowB, slowU;
            if (ssdSlowPath(srcColor, srcBiasImg, W, H, ps.bg, ps.rr, RP, CP, ps.dBias[0], ps.dBias[1], ps.dBias[2], xDstSrc,
                            yDstSrc, &slowB, &slowU))
              pushPair(slowB, slowU);
          }
        }
      } else {
        if (!LOWER || more) nxt = projectToSource(cams[sNext], wx, wy, wz, W, H);
      }
      if (!more) break;
      cur = nxt;
      s = sNext;
    }
  }
  *hits += n;
  if (n < 1) return FLT_MAX;  // kMinOverlappingCams - 1
  const int keep = n - 2 > 1 ? n - 2 : 1;
  if constexpr (LOWER) {
    if (unknown) return 0.0f;
    return kb.cost(n, keep, ps.conf);
  }
  float cost;
  if (n <= 3) {
    // keep == 1: nth_element(v, v+1, v+n) on <= 3 elements is an insertion sort, v[0] = the smallest pair
    float2 m = ps.sel[0];
    for (int i = 1; i < n; ++i) {
      const float2 t = ps.sel[i * ps.selStride];
      if (pairLess(t.x, t.y, m.x, m.y)) m = t;
    }
    cost = 0.0f + m.y;
  } else if (n <= kSelSlots) {
    // table-driven selection: host-validated on every permutation (tests/test_host_units.py), GPU-validated by the
    // parity suite; it declines ties and NaNs, which take the general algorithm
    static_assert(kSelSlots <= kSelTabMaxN, "the table path covers every evaluation that fits the shared-memory slots");
    // the 15-compare instance when no lane of the warp that got here holds more than 6 pairs
    const bool small = __reduce_max_sync(__activemask(), (unsigned)n) <= 6u;
    const bool done = small ? robustSumTable<6>(SmemPairs{ps.sel, ps.selStride}, n, keep, v.selTab, &cost)
                            : robustSumTable<8>(SmemPairs{ps.sel, ps.selStride}, n, keep, v.selTab, &cost);
    if (!done) cost = robustSum(SmemPairs{ps.sel, ps.selStride}, n, keep);
  } else {  // more than kSelTabMaxN sources: the general algorithm on the shared-memory slots
    cost = robustSum(SmemPairs{ps.sel, ps.selStride}, n, keep);
  }
  cost /= (float)keep;
  const float trustCoef = 1.0f / (float)keep;
  return cost * trustCoef / ps.conf;
}

}  // namespace derp
