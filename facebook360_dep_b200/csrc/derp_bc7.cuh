// derp_bc7.cuh — BC7 colour blocks for ConvertToBinary's default colour format (SURVEY §8(f) rank 4, colour half).
//
// What it replaces: bc7_util::compressBC7 (source/conversion/BC7Util.h:45-98) = gamma-correct and pack the image to
// RGBA8, then CompressBlocksBC7 with GetProfile_veryfast (ispc_texcomp.cpp:61-93) of the ISPC texture compressor the
// reference vendors (source/thirdparty/bc7_compressor/ISPCTextureCompressor/ispc/ispc_texcomp/kernel.ispc:615-2036).
// With that profile and an opaque 3-channel surface the encoder tries, per 4 x 4 block:
//   * the two-subset modes 1 and 3: all 64 partitions are ranked by a bound on the residual left after fitting one line
//     per subset (kernel.ispc:906-970, 1395-1414), the best 3 (mode 1) / 1 (mode 3) are tried (:1278-1296), the winner of
//     each mode is refined by least squares 2 / 1 times (:1197-1261, 1330-1352);
//   * mode 6 (one line, 7-bit endpoints + p-bit, 4-bit indexes) with one refinement (:1656-1688);
//   and keeps whichever has the smallest squared error, mode 6 winning only when strictly better.
// The arithmetic below follows the reference's operation order, its x86 float->int conversions and its endpoint
// quantisation as compiled by the reference's build (ISPC.cmake:4, --opt=fast-math: `x / 255f` is `x * fl(1/255)`),
// with ONE documented difference: where that build replaces `a / b` by `a * rcp(b)` and calls `rsqrt()` (RCPPS / RSQRTPS
// estimates + one Newton step, low bits CPU-vendor dependent) this code divides and takes 1 / sqrt in IEEE arithmetic.
// The outputs therefore agree with the reference build block for block except where such a last-bit difference flips a
// decision (tests/test_bc7.py measures the identity rate and compares decoded error).
//
// One thread encodes one block (the block lives in 48 registers); every function is __host__ __device__ so that the CPU
// test suite can run the same code through derp_test_bc7_blocks_host (a test hook: the apps only call the CUDA entry).
#pragma once
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>

namespace derp {
namespace bc7 {

#ifdef __CUDACC__
#define BC7_FN __host__ __device__ __forceinline__
// The stages called from several places (line fit, index choice, least-squares refit) are NOT inlined on the device and
// their per-pixel loops stay rolled: fully inlined and unrolled the kernel is hundreds of KB of code and stalls on
// instruction fetch.
#define BC7_STAGE __host__ __device__ __noinline__
#else  // plain C++ build of the same functions: oracle/bc7_x86.cpp (test infrastructure)
#define BC7_FN inline
#define BC7_STAGE inline
#endif
#define BC7_PIXEL_LOOP _Pragma("unroll 2")

// Division and reciprocal square root.  Product: IEEE.  -DDERP_BC7_X86_ESTIMATES (host only, used by the test build
// oracle/bc7_x86.cpp): the instruction sequences the reference's ispc build emits for `a / b` and rsqrt() — RCPPS / RSQRTPS
// + one Newton step — so that a test can show the two encoders agree byte for byte once the arithmetic is the same.
#if defined(DERP_BC7_X86_ESTIMATES) && !defined(__CUDA_ARCH__)
}  // namespace bc7
}  // namespace derp
#include <xmmintrin.h>
namespace derp {
namespace bc7 {
inline float divide(float a, float b) {
  const float iv = _mm_cvtss_f32(_mm_rcp_ss(_mm_set_ss(b)));
  return a * ((2.0f - b * iv) * iv);
}
inline float inverseSqrt(float v) {
  const float is = _mm_cvtss_f32(_mm_rsqrt_ss(_mm_set_ss(v)));
  return ((3.0f - (v * is) * is) * is) * 0.5f;
}
#else
BC7_FN float divide(float a, float b) { return a / b; }
BC7_FN float inverseSqrt(float v) { return 1.0f / sqrtf(v); }
#endif

// ---- format data (BC7 specification): subset-1 pixel masks and subset-1 anchor pixels of the 64 two-subset partitions ----
#define BC7_SUBSET1_MASKS                                                                                             \
  {                                                                                                                   \
    0xCCCC, 0x8888, 0xEEEE, 0xECC8, 0xC880, 0xFEEC, 0xFEC8, 0xEC80, 0xC800, 0xFFEC, 0xFE80, 0xE800, 0xFFE8, 0xFF00,   \
        0xFFF0, 0xF000, 0xF710, 0x008E, 0x7100, 0x08CE, 0x008C, 0x7310, 0x3100, 0x8CCE, 0x088C, 0x3110, 0x6666,       \
        0x366C, 0x17E8, 0x0FF0, 0x718E, 0x399C, 0xAAAA, 0xF0F0, 0x5A5A, 0x33CC, 0x3C3C, 0x55AA, 0x9696, 0xA55A,       \
        0x73CE, 0x13C8, 0x324C, 0x3BDC, 0x6996, 0xC33C, 0x9966, 0x0660, 0x0272, 0x04E4, 0x4E40, 0x2720, 0xC936,       \
        0x936C, 0x39C6, 0x639C, 0x9336, 0x9CC6, 0x817E, 0xE718, 0xCCF0, 0x0FCC, 0x7744, 0xEE22                        \
  }
#define BC7_SUBSET1_ANCHORS                                                                                           \
  {                                                                                                                   \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 2, 8, 2, 2, 8, 8, 15, 2, 8, 2, 2, 8, 8, 2, 2, \
        15, 15, 6, 8, 2, 8, 15, 15, 2, 8, 2, 2, 2, 15, 15, 6, 6, 2, 6, 8, 15, 15, 2, 2, 15, 15, 15, 15, 15, 2, 2, 15  \
  }
#ifdef __CUDACC__
__constant__ uint16_t kSubset1MasksDev[64] = BC7_SUBSET1_MASKS;
__constant__ uint8_t kSubset1AnchorsDev[64] = BC7_SUBSET1_ANCHORS;
#endif
static const uint16_t kSubset1MasksHost[64] = BC7_SUBSET1_MASKS;
static const uint8_t kSubset1AnchorsHost[64] = BC7_SUBSET1_ANCHORS;

BC7_FN uint32_t subset1Mask(int part) {
#ifdef __CUDA_ARCH__
  return kSubset1MasksDev[part];
#else
  return kSubset1MasksHost[part];
#endif
}
BC7_FN int subset1Anchor(int part) {
#ifdef __CUDA_ARCH__
  return kSubset1AnchorsDev[part];
#else
  return kSubset1AnchorsHost[part];
#endif
}
// interpolation weight of index q among 2^bits levels (the specification's tables {0,21,43,64}, {0,9,...,64}, {0,4,...,64})
template <int kBits>
BC7_FN int weight(int q) {
  constexpr int kMax = (1 << kBits) - 1;
  return (q * 64 + kMax / 2) / kMax;
}

// ---- x86 semantics the reference build relies on ----
// CVTTPS2DQ: truncation; NaN and out-of-range give INT_MIN (a zero-length line makes the projection 0/0 or x/0)
BC7_FN int truncX86(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN; }
BC7_FN float minPs(float a, float b) { return a < b ? a : b; }  // MINPS a, b
BC7_FN float maxPs(float a, float b) { return a > b ? a : b; }  // MAXPS a, b
BC7_FN float clampPs(float v, float lo, float hi) { return minPs(maxPs(v, lo), hi); }
BC7_FN int clampInt(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
BC7_FN float sq(float v) { return v * v; }

// The 16 pixels of a block, values 0..255 as floats: px(channel R / G / B, pixel y * 4 + x).  On the device they live in
// shared memory, [channel * 16 + pixel][thread] (conflict-free: consecutive threads, consecutive words), so that the loops
// over pixels can stay rolled and the stages can be real functions; on the host a plain array.
struct HostPixels {
  float v[3][16];
  BC7_FN float operator()(int c, int k) const { return v[c][k]; }
};
#ifdef __CUDACC__
constexpr int kBc7Threads = 128;
constexpr int kBc7MinCtas = 2;  // resident CTAs per SM bc7Kernel is compiled for (register cap)
__shared__ float bc7Tile[48 * kBc7Threads];  // 24 KB per CTA; a thread only ever touches its own 48 words: no barriers
struct SharedPixels {
  __device__ __forceinline__ float operator()(int c, int k) const { return bc7Tile[(c * 16 + k) * kBc7Threads + threadIdx.x]; }
};
#endif

// ---- first and second moments of the pixels selected by a 16-bit mask (kernel.ispc:762-802) ----
struct Moments {
  float rr, rg, rb, gg, gb, bb, r, g, b, n;
};
template <class Px>
BC7_FN Moments momentsOf(const Px& px, uint32_t mask) {
  Moments m = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  BC7_PIXEL_LOOP
  for (int k = 0; k < 16; ++k) {
    const float in = (float)((mask >> k) & 1u);
    const float r = px(0, k) * in, g = px(1, k) * in, b = px(2, k) * in;
    m.n += in;
    m.r += r;
    m.g += g;
    m.b += b;
    m.rr += r * r;
    m.rg += r * g;
    m.rb += r * b;
    m.gg += g * g;
    m.gb += g * b;
    m.bb += b * b;
  }
  return m;
}
BC7_FN Moments minus(const Moments& a, const Moments& b) {
  Moments m = {a.rr - b.rr, a.rg - b.rg, a.rb - b.rb, a.gg - b.gg, a.gb - b.gb,
               a.bb - b.bb, a.r - b.r,   a.g - b.g,   a.b - b.b,   a.n - b.n};
  return m;
}

// ---- covariance (kernel.ispc:804-822), scaled to unit range and regularised (:833-853, 906-921) ----
struct Cov {
  float rr, rg, rb, gg, gb, bb;
};
BC7_FN Cov scaledCovariance(const Moments& m) {
  Cov c;
  c.rr = m.rr - divide(m.r * m.r, m.n);
  c.rg = m.rg - divide(m.r * m.g, m.n);
  c.rb = m.rb - divide(m.r * m.b, m.n);
  c.gg = m.gg - divide(m.g * m.g, m.n);
  c.gb = m.gb - divide(m.g * m.b, m.n);
  c.bb = m.bb - divide(m.b * m.b, m.n);
  const float unit = 1.0f / (256 * 256), eps = 0.001f * 0.001f;
  c.rr *= unit;
  c.rg *= unit;
  c.rb *= unit;
  c.gg *= unit;
  c.gb *= unit;
  c.bb *= unit;
  c.rr += eps;
  c.gg += eps;
  c.bb += eps;
  return c;
}
BC7_FN void symv(const Cov& c, const float (&v)[3], float (&out)[3]) {
  out[0] = c.rr * v[0] + c.rg * v[1] + c.rb * v[2];
  out[1] = c.rg * v[0] + c.gg * v[1] + c.gb * v[2];
  out[2] = c.rb * v[0] + c.gb * v[1] + c.bb * v[2];
}
// power iteration from (1, 1, 1), renormalised after every second step (kernel.ispc:206-228)
template <int kSteps>
BC7_FN void principalAxis(const Cov& c, float (&axis)[3]) {
  float v[3] = {1, 1, 1};
#pragma unroll
  for (int i = 0; i < kSteps; ++i) {
    float a[3];
    symv(c, v, a);
    v[0] = a[0];
    v[1] = a[1];
    v[2] = a[2];
    if (i & 1) {
      float norm2 = 0;
      norm2 += a[0] * a[0];
      norm2 += a[1] * a[1];
      norm2 += a[2] * a[2];
      const float inv = inverseSqrt(norm2);
      v[0] *= inv;
      v[1] *= inv;
      v[2] *= inv;
    }
  }
  axis[0] = v[0];
  axis[1] = v[1];
  axis[2] = v[2];
}
// trace minus an estimate of the largest eigenvalue: what one line cannot explain (kernel.ispc:906-938)
BC7_FN float residualBound(const Moments& m) {
  const Cov c = scaledCovariance(m);
  float axis[3], w[3];
  principalAxis<4>(c, axis);
  symv(c, axis, w);
  float len2 = 0;
  len2 += sq(w[0]);
  len2 += sq(w[1]);
  len2 += sq(w[2]);
  float bound = c.rr + c.gg + c.bb;
  bound -= sqrtf(len2);
  return maxPs(bound, 0.0f);
}

// ---- one line per subset: end points on the principal axis, clamped to the byte range (kernel.ispc:856-904) ----
template <class Px>
BC7_STAGE void fitLine(const Px& px, uint32_t mask, float (&ends)[2][3]) {
  const Moments m = momentsOf(px, mask);
  const Cov c = scaledCovariance(m);
  const float mean[3] = {divide(m.r, m.n), divide(m.g, m.n), divide(m.b, m.n)};
  float axis[3];
  principalAxis<8>(c, axis);
  float lo = INFINITY, hi = -INFINITY;
  BC7_PIXEL_LOOP
  for (int k = 0; k < 16; ++k) {
    if (!((mask >> k) & 1u)) continue;
    float t = 0;
    t += axis[0] * (px(0, k) - mean[0]);
    t += axis[1] * (px(1, k) - mean[1]);
    t += axis[2] * (px(2, k) - mean[2]);
    lo = minPs(lo, t);
    hi = maxPs(hi, t);
  }
  if (hi - lo < 1.0f) {  // keep the end points apart
    lo -= 0.5f;
    hi += 0.5f;
  }
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    ends[0][p] = clampPs(lo * axis[p] + mean[p], 0.0f, 255.0f);
    ends[1][p] = clampPs(hi * axis[p] + mean[p], 0.0f, 255.0f);
  }
}

// ---- end-point quantisation with parity bits (kernel.ispc:982-1051) ----
// value with the given parity closest (in the reference's arithmetic) to e, on a grid of `top` + 1 steps
template <int kTop>  // 255: 7 bits + parity (modes 3, 6); 127: 6 bits + parity (mode 1)
BC7_FN int quantiseWithParity(float e, int parity) {
  const float inv255 = 1.0f / 255.0f;  // the reference build multiplies by the rounded reciprocal
  const int v = truncX86((e * inv255 * (float)kTop - (float)parity) * 0.5f + 0.5f) * 2 + parity;
  return clampInt(v, parity, kTop - 1 + parity);
}
BC7_FN int expand7(int v) {  // 7-bit end point -> byte (kernel.ispc:975-980)
  const int s = v << 1;
  return s + (s >> 7);
}
// modes 3 and 6: every end point has its own parity bit
BC7_FN void quantiseEnd8(const float (&e)[3], int (&q)[3]) {
  int q0[3], q1[3];
  float err0 = 0, err1 = 0;
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    q0[p] = quantiseWithParity<255>(e[p], 0);
    q1[p] = quantiseWithParity<255>(e[p], 1);
    err0 += sq(e[p] - (float)q0[p]);
    err1 += sq(e[p] - (float)q1[p]);
  }
#pragma unroll
  for (int p = 0; p < 3; ++p) q[p] = err0 < err1 ? q0[p] : q1[p];
}
// mode 1: the two end points of a subset share one parity bit
BC7_FN void quantisePair7(const float (&e)[2][3], int (&q)[2][3]) {
  int q0[2][3], q1[2][3];
  float err0 = 0, err1 = 0;
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      q0[j][p] = quantiseWithParity<127>(e[j][p], 0);
      q1[j][p] = quantiseWithParity<127>(e[j][p], 1);
      err0 += sq(e[j][p] - (float)expand7(q0[j][p]));
      err1 += sq(e[j][p] - (float)expand7(q1[j][p]));
    }
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int p = 0; p < 3; ++p) q[j][p] = err0 < err1 ? q0[j][p] : q1[j][p];
}

// A candidate encoding of the block in a two-subset mode (or mode 6: subset 1 empty)
struct Lines {
  int q[2][2][3];   // [subset][end][channel] quantised end points (mode 1: 7 bits, modes 3 / 6: 8 bits incl. parity)
  uint32_t idx[2];  // 16 x 4-bit pixel indexes
};
template <int kMode>
BC7_FN void quantiseLines(const float (&ends)[2][2][3], int kSubsets, Lines& out, float (&deq)[2][2][3]) {
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    if (s >= kSubsets) {  // mode 6 has one line; keep the unused slot defined
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int p = 0; p < 3; ++p) {
          out.q[s][j][p] = 0;
          deq[s][j][p] = 0;
        }
      continue;
    }
    if (kMode == 1) {
      quantisePair7(ends[s], out.q[s]);
    } else {
      quantiseEnd8(ends[s][0], out.q[s][0]);
      quantiseEnd8(ends[s][1], out.q[s][1]);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int p = 0; p < 3; ++p) deq[s][j][p] = (float)(kMode == 1 ? expand7(out.q[s][j][p]) : out.q[s][j][p]);
  }
}

// ---- pixel indexes against dequantised end points, returns the squared error (kernel.ispc:1132-1192) ----
template <int kBits, class Px>
BC7_STAGE float chooseIndexes(const Px& px, const float (&deq)[2][2][3], uint32_t subset1, uint32_t (&idx)[2]) {
  constexpr int kLevels = 1 << kBits;
  float total = 0;
  uint64_t packed = 0;
  BC7_PIXEL_LOOP
  for (int k = 0; k < 16; ++k) {
    const bool second = (subset1 >> k) & 1u;
    const float v[3] = {px(0, k), px(1, k), px(2, k)};
    float a[3], b[3];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      a[p] = second ? deq[1][0][p] : deq[0][0][p];
      b[p] = second ? deq[1][1][p] : deq[0][1][p];
    }
    float along = 0, len2 = 0;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      along += (v[p] - a[p]) * (b[p] - a[p]);
      len2 += sq(b[p] - a[p]);
    }
    along /= len2;  // `/=` stays a true division in the reference build (DIVPS)
    const int upper = clampInt(truncX86(along * (float)kLevels + 0.5f), 1, kLevels - 1);
    const int w0 = weight<kBits>(upper - 1), w1 = weight<kBits>(upper);
    float err0 = 0, err1 = 0;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      const float d0 = (float)(int)(((float)(64 - w0) * a[p] + (float)w0 * b[p] + 32.0f) * (1.0f / 64.0f));
      const float d1 = (float)(int)(((float)(64 - w1) * a[p] + (float)w1 * b[p] + 32.0f) * (1.0f / 64.0f));
      err0 += sq(d0 - v[p]);
      err1 += sq(d1 - v[p]);
    }
    int err = (int)err1, q = upper;  // the reference accumulates the error through an int
    if (err0 < err1) {
      err = (int)err0;
      q = upper - 1;
    }
    packed += (uint64_t)q << (4 * k);
    total += (float)err;
  }
  idx[0] = (uint32_t)packed;
  idx[1] = (uint32_t)(packed >> 32);
  return total;
}

// ---- least-squares end points for fixed indexes (kernel.ispc:1197-1261) ----
template <int kBits, class Px>
BC7_STAGE void refitLine(const Px& px, const uint32_t (&idx)[2], uint32_t mask, float (&ends)[2][3]) {
  constexpr int kTop = (1 << kBits) - 1;
  float xb[3] = {0, 0, 0}, sum[3] = {0, 0, 0};
  float sumQ = 0, sumQQ = 0, count = 0;
  const uint64_t packed = (uint64_t)idx[0] | ((uint64_t)idx[1] << 32);
  BC7_PIXEL_LOOP
  for (int k = 0; k < 16; ++k) {
    if (!((mask >> k) & 1u)) continue;
    const float q = (float)(int)((packed >> (4 * k)) & 15u);
    const float v[3] = {px(0, k), px(1, k), px(2, k)};
    const float x = (float)(int)((float)kTop - q);
    sumQ += q;
    sumQQ += q * q;
    count += 1;
#pragma unroll
    for (int p = 0; p < 3; ++p) sum[p] += v[p];
#pragma unroll
    for (int p = 0; p < 3; ++p) xb[p] += x * v[p];
  }
  float yb[3];
#pragma unroll
  for (int p = 0; p < 3; ++p) yb[p] = (float)kTop * sum[p] - xb[p];
  const float cxx = count * sq((float)kTop) - (float)(2 * kTop) * sumQ + sumQQ;
  const float cyy = sumQQ;
  const float cxy = (float)kTop * sumQ - sumQQ;
  const float det = cxx * cyy - cxy * cxy;
  const float scale = divide((float)kTop, det);
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    ends[0][p] = (xb[p] * cyy - yb[p] * cxy) * scale;
    ends[1][p] = (yb[p] * cxx - xb[p] * cxy) * scale;
  }
  if (fabsf(det) < 0.001f) {  // all indexes equal: both ends at the mean
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      ends[0][p] = divide(sum[p], count);
      ends[1][p] = ends[0][p];
    }
  }
}

// ---- bit stream ----
struct Stream {
  uint64_t lo, hi;
  int pos;
  BC7_FN void put(uint32_t v, int bits) {
    if (pos < 64) {
      lo |= (uint64_t)v << pos;
      if (pos + bits > 64) hi |= (uint64_t)v >> (64 - pos);
    } else {
      hi |= (uint64_t)v << (pos - 64);
    }
    pos += bits;
  }
};
BC7_FN uint32_t indexAt(const uint32_t (&idx)[2], int k) { return ((k < 8 ? idx[0] : idx[1]) >> (4 * (k & 7))) & 15u; }

// modes 1 and 3 (kernel.ispc:1707-1732, 1806-1876): each subset's anchor index must have its top bit clear — if not, the
// subset's end points are exchanged and its indexes mirrored — and is stored one bit shorter
template <int kMode>
BC7_FN void packTwoSubsets(Lines c, int part, uint32_t (&out)[4]) {
  constexpr int kBits = kMode == 1 ? 3 : 2, kLevels = 1 << kBits;
  const uint32_t subset1 = subset1Mask(part);
  const int anchor1 = subset1Anchor(part);
  uint32_t mirrored = 0;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int anchor = s ? anchor1 : 0;
    if ((int)indexAt(c.idx, anchor) >= kLevels / 2) {
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        const int t = c.q[s][0][p];
        c.q[s][0][p] = c.q[s][1][p];
        c.q[s][1][p] = t;
      }
      mirrored |= s ? subset1 : (~subset1 & 0xFFFFu);
    }
  }
  Stream w = {0, 0, 0};
  w.put(1u << kMode, kMode + 1);
  w.put((uint32_t)part & 63u, 6);
#pragma unroll
  for (int p = 0; p < 3; ++p)
#pragma unroll
    for (int e = 0; e < 4; ++e) w.put((uint32_t)c.q[e >> 1][e & 1][p] >> 1, kMode == 1 ? 6 : 7);
  if (kMode == 1) {
    w.put((uint32_t)c.q[0][0][0] & 1u, 1);
    w.put((uint32_t)c.q[1][0][0] & 1u, 1);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) w.put((uint32_t)c.q[e >> 1][e & 1][0] & 1u, 1);
  }
  BC7_PIXEL_LOOP
  for (int k = 0; k < 16; ++k) {
    uint32_t q = indexAt(c.idx, k);
    if ((mirrored >> k) & 1u) q = (uint32_t)(kLevels - 1) - q;
    w.put(q, (k == 0 || k == anchor1) ? kBits - 1 : kBits);
  }
  out[0] = (uint32_t)w.lo;
  out[1] = (uint32_t)(w.lo >> 32);
  out[2] = (uint32_t)w.hi;
  out[3] = (uint32_t)(w.hi >> 32);
}
// mode 6 (kernel.ispc:1693-1705, 1940-1964); alpha end points are 7 bits + the colour parity bit
BC7_FN void packMode6(const int (&q)[2][3], const int (&alpha)[2], const uint32_t (&idx)[2], uint32_t (&out)[4]) {
  int e0[4] = {q[0][0], q[0][1], q[0][2], alpha[0]}, e1[4] = {q[1][0], q[1][1], q[1][2], alpha[1]};
  uint32_t i0 = idx[0], i1 = idx[1];
  if ((i0 & 15u) >= 8u) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int t = e0[p];
      e0[p] = e1[p];
      e1[p] = t;
    }
    i0 = 0xFFFFFFFFu - i0;
    i1 = 0xFFFFFFFFu - i1;
  }
  Stream w = {0, 0, 0};
  w.put(64u, 7);
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    w.put((uint32_t)e0[p] >> 1, 7);
    w.put((uint32_t)e1[p] >> 1, 7);
  }
  w.put((uint32_t)e0[0] & 1u, 1);
  w.put((uint32_t)e1[0] & 1u, 1);
  w.put(i0 & 15u, 3);
#pragma unroll
  for (int k = 1; k < 8; ++k) w.put((i0 >> (4 * k)) & 15u, 4);
#pragma unroll
  for (int k = 0; k < 8; ++k) w.put((i1 >> (4 * k)) & 15u, 4);
  out[0] = (uint32_t)w.lo;
  out[1] = (uint32_t)(w.lo >> 32);
  out[2] = (uint32_t)w.hi;
  out[3] = (uint32_t)(w.hi >> 32);
}

// ---- a two-subset mode over a short list of partitions, then refinement of the winner (kernel.ispc:1278-1362) ----
template <int kMode, class Px>
BC7_FN float tryTwoSubsets(const Px& px, int part0, int part1, int part2, int count, int refinements, Lines& best,
                           int& bestPart) {
  constexpr int kBits = kMode == 1 ? 3 : 2;
  float bestErr = INFINITY;
  bestPart = part0;
  for (int t = 0; t < count; ++t) {
    const int part = t == 0 ? part0 : (t == 1 ? part1 : part2);
    const uint32_t subset1 = subset1Mask(part);
    float ends[2][2][3], deq[2][2][3];
    fitLine(px, ~subset1 & 0xFFFFu, ends[0]);
    fitLine(px, subset1, ends[1]);
    Lines c;
    quantiseLines<kMode>(ends, 2, c, deq);
    const float err = chooseIndexes<kBits>(px, deq, subset1, c.idx);
    if (err < bestErr) {
      bestErr = err;
      best = c;
      bestPart = part;
    }
  }
  const uint32_t subset1 = subset1Mask(bestPart);
  for (int it = 0; it < refinements; ++it) {
    float ends[2][2][3], deq[2][2][3];
    refitLine<kBits>(px, best.idx, ~subset1 & 0xFFFFu, ends[0]);
    refitLine<kBits>(px, best.idx, subset1, ends[1]);
    Lines c;
    quantiseLines<kMode>(ends, 2, c, deq);
    const float err = chooseIndexes<kBits>(px, deq, subset1, c.idx);
    if (err < bestErr) {
      bestErr = err;
      best = c;
    }
  }
  return bestErr;
}

// alpha end point of mode 6 for an opaque surface: the reference quantises 255 (then, after a refinement, the dequantised
// value) on the 8-bit grid with the colour end point's parity (kernel.ispc:982-1021 with p = 3)
BC7_FN int quantiseAlpha(float a, int parity) { return quantiseWithParity<255>(a, parity); }

// ---- one block: the veryfast profile on an opaque RGB surface (kernel.ispc:1969-1976, ispc_texcomp.cpp:61-93) ----
template <class Px>
BC7_FN void encodeBlock(const Px& px, uint32_t (&out)[4]) {
  float bestErr = INFINITY;
  out[0] = out[1] = out[2] = out[3] = 0;

  // rank the 64 partitions by the residual bound; keep the three smallest keys (partition + 64 * integer bound), in order
  {
    const Moments all = momentsOf(px, 0xFFFFu);
    int key0 = INT_MAX, key1 = INT_MAX, key2 = INT_MAX;
#pragma unroll 1
    for (int part = 0; part < 64; ++part) {
      const Moments first = momentsOf(px, ~subset1Mask(part) & 0xFFFFu);
      float bound = 0;
      bound += residualBound(first);
      bound += residualBound(minus(all, first));
      const int key = part + truncX86(sqrtf(bound) * 256.0f) * 64;
      if (key < key0) {
        key2 = key1;
        key1 = key0;
        key0 = key;
      } else if (key < key1) {
        key2 = key1;
        key1 = key;
      } else if (key < key2) {
        key2 = key;
      }
    }
    Lines lines;
    int part;
    float err = tryTwoSubsets<1>(px, key0 & 63, key1 & 63, key2 & 63, 3, 2, lines, part);
    if (err < bestErr) {
      bestErr = err;
      packTwoSubsets<1>(lines, part, out);
    }
    err = tryTwoSubsets<3>(px, key0 & 63, key0 & 63, key0 & 63, 1, 1, lines, part);
    if (err < bestErr) {
      bestErr = err;
      packTwoSubsets<3>(lines, part, out);
    }
  }

  // mode 6
  {
    float ends[2][2][3], deq[2][2][3];
    fitLine(px, 0xFFFFu, ends[0]);
    Lines c;
    quantiseLines<6>(ends, 1, c, deq);
    int alpha[2] = {quantiseAlpha(255.0f, c.q[0][0][0] & 1), quantiseAlpha(255.0f, c.q[0][1][0] & 1)};
    float err = chooseIndexes<4>(px, deq, 0u, c.idx);
    {  // one refinement, taken unconditionally
      refitLine<4>(px, c.idx, 0xFFFFu, ends[0]);
      quantiseLines<6>(ends, 1, c, deq);
      alpha[0] = quantiseAlpha((float)alpha[0], c.q[0][0][0] & 1);
      alpha[1] = quantiseAlpha((float)alpha[1], c.q[0][1][0] & 1);
      err = chooseIndexes<4>(px, deq, 0u, c.idx);
    }
    if (err < bestErr) {
      bestErr = err;
      packMode6(c.q[0], alpha, c.idx, out);
    }
  }
}


#ifdef __CUDACC__
// ---- K18: one thread per 4 x 4 block ----------------------------------------------------------------------------------
// Source forms: (a) the RGBA8 surface CompressBlocksBC7 receives; (b) the image as cv::imread(IMREAD_UNCHANGED) holds it
// (B, G, R[, A] interleaved, 8 or 16 bits per channel) with BC7Util.h's conversion + gamma correction + packing fused in
// through a lookup table indexed by the stored channel value (256 or 65 536 entries, built on the host with the host's
// powf: the reference's own call).  A warp reads 32 neighbouring blocks: 512 (RGBA8) contiguous bytes per image row, and
// writes 512 contiguous bytes of blocks.  Bound: instruction issue (about 4 x 10^4 instructions per block against 64 + 16
// bytes of traffic).
struct Rgba8Source {
  const uint8_t* rgba;  // width * 4 bytes per row
  int width;
  __device__ __forceinline__ void load(int bx, int by, float* mine) const {
#pragma unroll
    for (int y = 0; y < 4; ++y) {
      const uint32_t* row = reinterpret_cast<const uint32_t*>(rgba + ((size_t)(by * 4 + y) * width + (size_t)bx * 4) * 4);
      uint32_t t[4];
      if ((width & 3) == 0) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(row));
        t[0] = v.x;
        t[1] = v.y;
        t[2] = v.z;
        t[3] = v.w;
      } else {
#pragma unroll
        for (int x = 0; x < 4; ++x) t[x] = __ldg(row + x);
      }
#pragma unroll
      for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int c = 0; c < 3; ++c) mine[(c * 16 + y * 4 + x) * kBc7Threads] = (float)(int)((t[x] >> (8 * c)) & 255u);
    }
  }
};
template <typename T>
struct BgrSource {
  const T* bgr;  // width * channels values per row
  int width, channels;
  const uint8_t* lut;  // stored value -> gamma-corrected byte
  __device__ __forceinline__ void load(int bx, int by, float* mine) const {
#pragma unroll
    for (int y = 0; y < 4; ++y)
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const T* t = bgr + ((size_t)(by * 4 + y) * width + (size_t)bx * 4 + x) * channels;
#pragma unroll
        for (int c = 0; c < 3; ++c) mine[(c * 16 + y * 4 + x) * kBc7Threads] = (float)__ldg(lut + t[2 - c]);
      }
  }
};
template <typename Source>
__global__ void __launch_bounds__(kBc7Threads, kBc7MinCtas) bc7Kernel(Source src, int width, int blocksX, int blocksY, uint8_t* out) {
  const int b = blockIdx.x * kBc7Threads + threadIdx.x;
  if (b >= blocksX * blocksY) return;
  const int bx = b % blocksX, by = b / blocksX;
  src.load(bx, by, bc7Tile + threadIdx.x);
  const SharedPixels px = {};
  uint32_t data[4];
  encodeBlock(px, data);
  // the reference's store_data: block row `by` starts at byte by * width * 4 (kernel.ispc:152-159)
  uint32_t* dst = reinterpret_cast<uint32_t*>(out + (size_t)by * width * 4 + (size_t)bx * 16);
  if ((width & 3) == 0) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(data[0], data[1], data[2], data[3]);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[i] = data[i];
  }
}
#endif  // __CUDACC__

// host instantiation for the CPU test hook (not reachable from the apps)
inline void encodeSurfaceOnHost(const uint8_t* rgba, int width, int height, uint8_t* out) {
  for (int by = 0; by < height / 4; ++by)
    for (int bx = 0; bx < width / 4; ++bx) {
      HostPixels px;
      for (int y = 0; y < 4; ++y)
        for (int x = 0; x < 4; ++x) {
          const uint8_t* t = rgba + ((size_t)(by * 4 + y) * width + (size_t)bx * 4 + x) * 4;
          for (int p = 0; p < 3; ++p) px.v[p][y * 4 + x] = (float)t[p];
        }
      uint32_t data[4];
      encodeBlock(px, data);
      std::memcpy(out + (size_t)by * width * 4 + (size_t)bx * 16, data, 16);
    }
}

// bc7_util::gammaCorrect (BC7Util.h:41-43) of the value cv_util::convertTo gives a stored channel value
// (CvUtil.h:196-207: value * (1.0f / max) in float), for every stored value
inline void gammaTable(int bitsPerChannel, float gamma, uint8_t* lut) {
  const int n = 1 << bitsPerChannel;
  const float scale = 1.0f / (float)(n - 1);
  for (int v = 0; v < n; ++v) lut[v] = (uint8_t)(std::pow((float)v * scale, gamma) * 255.0f + 0.5f);
}

}  // namespace bc7
}  // namespace derp
