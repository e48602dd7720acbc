// sm_90a kernels of the depth path.  One thread per destination pixel unless stated; a warp
// covers 32 consecutive x so that the gathers of neighbouring lanes land in neighbouring texels.
// Camera structs are staged into shared memory once per CTA.
#pragma once

#include <cfloat>
#include <cstdint>

#include "derp_cost.cuh"
#include "derp_divconst.cuh"
#include "derp_rng.cuh"

namespace derp {

constexpr int kBlockX = 32, kBlockY = 8;  // 256 threads
// resident CTAs per SM requested for the cost kernels: 3 -> 80 registers, 24 warps/SM
constexpr int kCostMinCtas = 3;

__device__ __forceinline__ void stageCameras(DevCamera* sm, const DevCamera* __restrict__ g, int n) {
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int nt = blockDim.x * blockDim.y;
  const int words = n * (int)(sizeof(DevCamera) / sizeof(double));
  const double* src = reinterpret_cast<const double*>(g);
  double* dst = reinterpret_cast<double*>(sm);
  for (int i = tid; i < words; i += nt) dst[i] = src[i];
  __syncthreads();
}

// Adds (evals, hits) of the currently converged lanes to the global work counters with one
// atomic pair per warp.
__device__ __forceinline__ void addCounters(unsigned long long* counters, unsigned evals, unsigned hits) {
  const unsigned m = __activemask();
  const unsigned e = __reduce_add_sync(m, evals);
  const unsigned h = __reduce_add_sync(m, hits);
  if ((threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) {
    atomicAdd(counters, (unsigned long long)e);
    atomicAdd(counters + 1, (unsigned long long)h);
  }
}

// ---- K1: generateFovMasks (DerpUtil.cpp:239-276) ------------------------------------------------
__global__ void fovMaskKernel(const DevCamera* __restrict__ cam, int W, int H, uint8_t* __restrict__ mask) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  // normalised camera: p = (x + .5, y + .5) / size (DerpUtil.cpp:245-251)
  const double px = (x + 0.5) / W, py = (y + 0.5) / H;
  mask[(size_t)y * W + x] = !outsideImageCircle(*cam, px, py);
}

// ---- K2: computeWarpDstToSrc (ImageUtil.cpp:142-167) for all sources of one destination ---------
// projWarp(dst, s) = computeWarpDstToSrc(camSrc, camDst): iterates SOURCE pixels, stores where the
// destination sees them at infinity (Derp.cpp:970).  camsPx = cameras rescaled to the level size.
__global__ void projWarpKernel(const DevCamera* __restrict__ camsPx, int S, int self, int W, int H,
                               float2* __restrict__ projWarp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const float nan = __int_as_float(0x7fc00000);
  float2 out = make_float2(nan, nan);
  if (s != self) {
    const DevCamera& from = camsPx[s];
    const DevCamera& to = camsPx[self];
    const double px = x + 0.5, py = y + 0.5;
    if (!outsideImageCircle(from, px, py)) {
      double dir[3];
      pixelRay(from, px, py, dir);
      const double wx = from.pos[0] + dir[0] * 1e4, wy = from.pos[1] + dir[1] * 1e4, wz = from.pos[2] + dir[2] * 1e4;
      double qx, qy;
      if (sees(to, wx, wy, wz, &qx, &qy)) out = make_float2((float)(qx - 0.5f), (float)(qy - 0.5f));
    }
  }
  projWarp[(size_t)s * W * H + (size_t)y * W + x] = out;
}

// ---- K2b: projWarpInv(dst, s) = computeWarpDstToSrc(camDst, camSrc) (Derp.cpp:971) -------------------------
// Destination pixel -> source pixel at infinity, OpenCV convention (-0.5), NaN where unseen.  Like projWarp it
// depends on the rig and the level size only, so both maps are kept across frames when they fit in HBM
// (DerpCtx geometry cache) and the per-frame work of reprojectColors is the pure gather below.
__global__ void warpInvKernel(const DevCamera* __restrict__ camsPx, int S, int self, int W, int H,
                              float2* __restrict__ warpInv) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const float nan = __int_as_float(0x7fc00000);
  float2 out = make_float2(nan, nan);
  if (s != self) {
    const DevCamera& from = camsPx[self];
    const DevCamera& to = camsPx[s];
    const double px = x + 0.5, py = y + 0.5;
    if (!outsideImageCircle(from, px, py)) {
      double dir[3];
      pixelRay(from, px, py, dir);
      const double wx = from.pos[0] + dir[0] * 1e4, wy = from.pos[1] + dir[1] * 1e4, wz = from.pos[2] + dir[2] * 1e4;
      double qx, qy;
      if (sees(to, wx, wy, wz, &qx, &qy)) out = make_float2((float)(qx - 0.5f), (float)(qy - 0.5f));
    }
  }
  warpInv[(size_t)s * W * H + (size_t)y * W + x] = out;
}

// ---- K3: reprojectColors -> project (Derp.cpp:978-1003, DerpUtil.cpp:199-205) --------------------
// cv::remap(src colour, projWarpInv, INTER_CUBIC, BORDER_CONSTANT 0).
// wtab = OpenCV's 32x32x16 float bicubic table (built on the host exactly as imgwarp.cpp does).
__device__ __forceinline__ int cvRoundQ5(float v) {
  // cvRound(v * 32) with x86 semantics: NaN / out-of-range -> INT_MIN
  const float s = v * 32.0f;
  if (!(s == s) || s >= 2147483648.0f || s < -2147483648.0f) return INT_MIN;
  return __float2int_rn(s);
}

__device__ __forceinline__ float roundSatU16(float v) {
  int r = __float2int_rn(v);  // cvRound, then saturate_cast<ushort>; stored as an integer-valued float
  r = r < 0 ? 0 : (r > 65535 ? 65535 : r);
  return (float)r;
}

__device__ __forceinline__ unsigned roundSatU16i(float v) {
  int r = __float2int_rn(v);  // cvRound, then saturate_cast<ushort>
  return (unsigned)(r < 0 ? 0 : (r > 65535 ? 65535 : r));
}

// wtab1 = the 32 x 4 one-dimensional coefficient rows; OpenCV's 2-D table entry (fy, fx)[k1][k2] is the fp32 product
// wtab1[fy][k1] * wtab1[fx][k2] (initInterTab2D), formed here from two 16-byte shared-memory loads instead of 16
// scattered table reads.  Output: 4 x u16 texels (B | G << 16, R); the R-below lane is filled by the bias kernels.
__global__ void reprojectKernel(const float2* __restrict__ warpInv, int S, int self, int W, int H,
                                const uint2* __restrict__ color, const float* __restrict__ wtab1,
                                uint2* __restrict__ projColor16) {
  __shared__ float4 tab[32];
  {
    const int t = threadIdx.y * blockDim.x + threadIdx.x;
    if (t < 32) tab[t] = __ldg(reinterpret_cast<const float4*>(wtab1) + t);
  }
  __syncthreads();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const size_t plane = (size_t)W * H;
  const size_t p = (size_t)y * W + x;
  if (s == self) {  // Derp.cpp:989-991: the destination's own colour
    const uint2 t = color[s * plane + p];
    projColor16[s * plane + p] = make_uint2(t.x, t.y & 0xffffu);
    return;
  }
  const float2 m = __ldg(warpInv + s * plane + p);
  const float mx = m.x, my = m.y;
  const int sxq = cvRoundQ5(mx), syq = cvRoundQ5(my);
  int ix = sxq >> 5, iy = syq >> 5;
  ix = ix < -32768 ? -32768 : (ix > 32767 ? 32767 : ix);  // saturate_cast<short>
  iy = iy < -32768 ? -32768 : (iy > 32767 ? 32767 : iy);
  const int sx = ix - 1, sy = iy - 1;
  const float4 tx = tab[sxq & 31], ty = tab[syq & 31];
  const float wy[4] = {ty.x, ty.y, ty.z, ty.w};
  const uint2* S0 = color + s * plane;
  float sum0, sum1, sum2;
  if ((unsigned)sx < (unsigned)max(W - 3, 0) && (unsigned)sy < (unsigned)max(H - 3, 0)) {
    // interior: row-wise 4-term sums, accumulated row by row (imgwarp.cpp remapBicubic)
    sum0 = sum1 = sum2 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint2* row = S0 + (size_t)(sy + i) * W + sx;
      const Texel a = unpack(__ldg(row)), b = unpack(__ldg(row + 1)), c = unpack(__ldg(row + 2)),
                  d = unpack(__ldg(row + 3));
      const float w0 = wy[i] * tx.x, w1 = wy[i] * tx.y, w2 = wy[i] * tx.z, w3 = wy[i] * tx.w;
      const float r0 = a.b * w0 + b.b * w1 + c.b * w2 + d.b * w3;
      const float r1 = a.g * w0 + b.g * w1 + c.g * w2 + d.g * w3;
      const float r2 = a.r * w0 + b.r * w1 + c.r * w2 + d.r * w3;
      if (i == 0) {
        sum0 = r0;
        sum1 = r1;
        sum2 = r2;
      } else {
        sum0 += r0;
        sum1 += r1;
        sum2 += r2;
      }
    }
  } else {
    if (sx >= W || sx + 4 <= 0 || sy >= H || sy + 4 <= 0) {
      projColor16[s * plane + p] = make_uint2(0u, 0u);
      return;
    }
    // border: taps outside contribute the constant 0; one sequential sum (imgwarp.cpp)
    const float wx[4] = {tx.x, tx.y, tx.z, tx.w};
    sum0 = sum1 = sum2 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int yi = sy + i;
      if ((unsigned)yi >= (unsigned)H) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int xj = sx + j;
        if ((unsigned)xj >= (unsigned)W) continue;
        const Texel t = unpack(__ldg(S0 + (size_t)yi * W + xj));
        const float ww = wy[i] * wx[j];
        sum0 += (t.b - 0.f) * ww;
        sum1 += (t.g - 0.f) * ww;
        sum2 += (t.r - 0.f) * ww;
      }
    }
  }
  projColor16[s * plane + p] = make_uint2(roundSatU16i(sum0) | (roundSatU16i(sum1) << 16), roundSatU16i(sum2));
}

__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// ---- K4: colorBias = cv::blur 3x3 on u16x3 (DerpUtil.cpp:208-210) for all S planes -----------------
// Input: the 4 x u16 reprojection (B | G << 16, R) written by reprojectKernel.  The 9-term sums are plain integer sums,
// as in OpenCV's row/column filter; saturate_cast<ushort>(sum * (1.0/9)) == (sum + 4) / 9 for integer sums (no exact .5
// cases).  Two output formats, one per consumer:
//  * biasKernel: float4 tables for the dense sweep / evalCost / the getters — projColor = (B, G, R, R of the texel
//    below), projBias = (B, G, R, 0) as integer-valued floats; the w lane lets the cost kernel run channel R of two
//    vertically adjacent samples on the two lanes of the fp32 lane-pair arithmetic (derp_cost.cuh);
//  * bias16Kernel: the same two tables as 4 x u16 for the compacted fine-level kernels; projColor16 is the input
//    itself, completed IN PLACE with the R-below lane (bits 16..31 of .y).  Concurrent readers of a texel being
//    completed see either version of the 32-bit word and use only its low half, which does not change.
struct BoxSum {
  unsigned b, g, r, cx, cy, below;
};
__device__ __forceinline__ BoxSum boxSum3(const uint2* img, int W, int H, int x, int y) {
  BoxSum o{0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
  for (int j = -1; j <= 1; ++j) {
    const int yy = reflect101(y + j, H);
#pragma unroll
    for (int i = -1; i <= 1; ++i) {
      const int xx = reflect101(x + i, W);
      const uint2 t = img[(size_t)yy * W + xx];
      o.b += t.x & 0xffffu;
      o.g += t.x >> 16;
      o.r += t.y & 0xffffu;
      if (i == 0 && j == 0) {
        o.cx = t.x;
        o.cy = t.y & 0xffffu;
      }
      if (i == 0 && j == 1) o.below = (y + 1 < H) ? (t.y & 0xffffu) : 0u;
    }
  }
  o.b = (o.b + 4) / 9;
  o.g = (o.g + 4) / 9;
  o.r = (o.r + 4) / 9;
  return o;
}

__global__ void biasKernel(int W, int H, const uint2* in, float4* __restrict__ color, float4* __restrict__ bias) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const BoxSum o = boxSum3(in + (size_t)s * W * H, W, H, x, y);
  const size_t q = (size_t)s * W * H + (size_t)y * W + x;
  bias[q] = make_float4((float)o.b, (float)o.g, (float)o.r, 0.f);
  color[q] = make_float4((float)(o.cx & 0xffffu), (float)(o.cx >> 16), (float)o.cy, (float)o.below);
}

__global__ void bias16Kernel(int W, int H, uint2* color16, uint2* __restrict__ bias16) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const BoxSum o = boxSum3(color16 + (size_t)s * W * H, W, H, x, y);
  const size_t q = (size_t)s * W * H + (size_t)y * W + x;
  bias16[q] = make_uint2(o.b | (o.g << 16), o.r);
  color16[q] = make_uint2(o.cx, o.cy | (o.below << 16));
}

// ---- K5: computeImageVariance (DerpUtil.cpp:214-237) for all S planes ---------------------------
__global__ void varianceKernel(int W, int H, const uint2* __restrict__ in, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int s = blockIdx.z;
  if (x >= W || y >= H) return;
  const uint2* img = in + (size_t)s * W * H;
  const float alpha = 1.0f / 65535.0f;
  double s1[3] = {0, 0, 0}, s2[3] = {0, 0, 0};
#pragma unroll
  for (int j = -1; j <= 1; ++j) {
    const int yy = reflect101(y + j, H);
    double r1[3] = {0, 0, 0}, r2[3] = {0, 0, 0};
#pragma unroll
    for (int i = -1; i <= 1; ++i) {
      const int xx = reflect101(x + i, W);
      const Texel t = unpack(__ldg(img + (size_t)yy * W + xx));
      const float f0 = t.b * alpha, f1 = t.g * alpha, f2 = t.r * alpha;
      r1[0] += (double)f0;
      r1[1] += (double)f1;
      r1[2] += (double)f2;
      r2[0] += (double)(f0 * f0);
      r2[1] += (double)(f1 * f1);
      r2[2] += (double)(f2 * f2);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      s1[c] += r1[c];
      s2[c] += r2[c];
    }
  }
  const double scale = 1.0 / 9;
  float vc[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float mean = (float)(s1[c] * scale);
    const float msq = (float)(s2[c] * scale);
    vc[c] = msq - mean * mean;
  }
  out[(size_t)s * W * H + (size_t)y * W + x] = vc[0] * 0.3333f + vc[1] * 0.3334f + vc[2] * 0.3333f;
}

// ---- layout conversion ----------------------------------------------------------------------------
__global__ void packColorKernel(size_t n, const uint16_t* __restrict__ bgr, uint2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t b = bgr[i * 3], g = bgr[i * 3 + 1], r = bgr[i * 3 + 2];
  out[i] = make_uint2(b | (g << 16), r);
}
__global__ void unpackColorKernel(size_t n, const uint2* __restrict__ in, uint16_t* __restrict__ bgr) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint2 t = in[i];
  bgr[i * 3] = (uint16_t)(t.x & 0xffffu);
  bgr[i * 3 + 1] = (uint16_t)(t.x >> 16);
  bgr[i * 3 + 2] = (uint16_t)(t.y & 0xffffu);
}
__global__ void unpackTexelF32Kernel(size_t n, const float4* __restrict__ in, uint16_t* __restrict__ bgr) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 t = in[i];
  bgr[i * 3] = (uint16_t)t.x;
  bgr[i * 3 + 1] = (uint16_t)t.y;
  bgr[i * 3 + 2] = (uint16_t)t.z;
}
template <typename T>
__global__ void fillKernel(size_t n, T* p, T v) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---- K6: fused sphere sweep + cost + winner-takes-all (Derp.cpp:230-356) ------------------------
// grid.z = candidate chunk.  Every thread sweeps its chunk in index order with a strict-< running
// minimum, then merges across chunks with a 64-bit atomicMin on (cost bits << 32 | index): for
// non-negative floats the bit pattern is monotone, so the merge keeps the lowest cost and, among
// equal costs, the lowest index — exactly the reference's first-strict-minimum scan.
struct SweepArgs : DstArgs {
  const float* disparities;  // [D] candidate table (probeDisparity)
  int D, chunk;
  unsigned long long* best;   // [H][W] packed
  unsigned long long* counters;  // [0] cost evaluations, [1] source hits
};

// Launched with 32 x BY threads: BY = kSweepMaxRows (20 => one 640-thread CTA per SM at 96 registers) on levels of
// >= 1024 rows, 10 on smaller ones; a taller CTA shares more texel rows between its warps (per-warp footprint (BY+3)/BY
// rows instead of 11/8).  Rigs of more than 42 cameras get shorter CTAs, whose S - 1 selection slots per thread still fit
// in shared memory (DerpCtx::sweepRows).
constexpr int kSweepMinCtas = 1;
template <class Mask>
__global__ void __launch_bounds__(32 * kSweepMaxRows, kSweepMinCtas) sweepKernel(const SweepArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* tile = reinterpret_cast<float*>(cams + a.v.S);
  stageCameras(cams, a.v.cams, a.v.S);
  loadDstTile(tile, a.v, blockIdx.x * kBlockX, blockIdx.y * blockDim.y);
  const int W = a.v.W, H = a.v.H;
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  unsigned hits = 0, evals = 0;
  if (x >= 1 && x < W - 1 && y >= 1 && y < H - 1) {
    const size_t p = (size_t)y * W + x;
    const bool active = a.fov[p] && (!a.fg || a.fg[p]);
    if (active) {
      PixelState ps;
      loadPixelState(a.v, cams[a.v.self], tile, x, y, ps);
      const float bgd = a.bg ? a.bg[p] : 0.f;
      const int c0 = blockIdx.z * a.chunk;
      const int c1 = min(a.D, c0 + a.chunk);
      float bestCost = FLT_MAX;
      int bestIdx = -1;
      for (int c = c0; c < c1; ++c) {
        const float d = __ldg(a.disparities + c);
        if (a.bg && !(bgd < d)) continue;  // closerMask (Derp.cpp:240-243)
        const float cost = evalCost<Mask, kTileW, 1>(a.v, cams, ps, d, &hits);
        ++evals;
        if (cost < bestCost) {
          bestCost = cost;
          bestIdx = c;
        }
      }
      if (bestIdx >= 0) {
        const unsigned long long packed =
            ((unsigned long long)__float_as_uint(bestCost) << 32) | (unsigned long long)(unsigned)bestIdx;
        atomicMin(a.best + p, packed);
      }
    }
  }
  addCounters(a.counters, evals, hits);
}

// WTA write-back (Derp.cpp:306-356) for interior pixels
__global__ void sweepFinalizeKernel(int W, int H, const uint8_t* __restrict__ fov, const uint8_t* __restrict__ fg,
                                    const float* __restrict__ bg, const float* __restrict__ variance,
                                    const float* __restrict__ disparities, float minDisparity,
                                    const unsigned long long* __restrict__ best, float* __restrict__ disp,
                                    float* __restrict__ cost, float* __restrict__ conf, int* __restrict__ idxOut,
                                    unsigned* __restrict__ uncovered) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < 1 || x >= W - 1 || y < 1 || y >= H - 1) return;
  const size_t p = (size_t)y * W + x;
  if (!fov[p]) {
    disp[p] = __int_as_float(0x7fc00000);
    if (idxOut) idxOut[p] = -2;
    return;
  }
  if (fg && !fg[p]) {
    disp[p] = bg[p];
    if (idxOut) idxOut[p] = -3;
    return;
  }
  const unsigned long long b = best[p];
  const unsigned idx = (unsigned)(b & 0xffffffffull);
  if (idx == 0xffffffffu) {
    atomicAdd(uncovered, 1u);
    disp[p] = minDisparity;
    cost[p] = FLT_MAX;
    conf[p] = 0.f;
    if (idxOut) idxOut[p] = -1;
  } else {
    disp[p] = disparities[idx];
    cost[p] = __uint_as_float((unsigned)(b >> 32));
    conf[p] = fmaxf(variance[p], kMinVarF);
    if (idxOut) idxOut[p] = (int)idx;
  }
}

// Extend disparities to the 1-px margin (Derp.cpp:359-381)
__global__ void extendBorderKernel(int W, int H, const uint8_t* __restrict__ fg, const float* __restrict__ bg,
                                   float* __restrict__ disp, float* __restrict__ cost, float* __restrict__ conf,
                                   int* __restrict__ idxOut) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = 2 * W + 2 * (H - 2);
  if (i >= per) return;
  int x, y;
  if (i < W) {
    x = i;
    y = 0;
  } else if (i < 2 * W) {
    x = i - W;
    y = H - 1;
  } else {
    const int k = i - 2 * W;
    y = 1 + (k >> 1);
    x = (k & 1) ? W - 1 : 0;
  }
  const size_t p = (size_t)y * W + x;
  if (fg && !fg[p]) {
    disp[p] = bg[p];
    if (idxOut) idxOut[p] = -3;
    return;
  }
  const size_t qq = (size_t)max(1, min(y, H - 2)) * W + max(1, min(x, W - 2));
  disp[p] = disp[qq];
  cost[p] = cost[qq];
  conf[p] = conf[qq];
  if (idxOut) idxOut[p] = idxOut[qq];
}

// ---- derp_eval_cost: one hypothesis per pixel ------------------------------------------------------
template <class Mask>
__global__ void __launch_bounds__(kBlockX* kBlockY, kCostMinCtas)
    evalCostKernel(const CostView v, const float* __restrict__ disparity, float* __restrict__ outCost,
                   float* __restrict__ outConf, unsigned long long* counters) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* tile = reinterpret_cast<float*>(cams + v.S);
  stageCameras(cams, v.cams, v.S);
  loadDstTile(tile, v, blockIdx.x * kBlockX, blockIdx.y * kBlockY);
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  if (x >= v.W || y >= v.H) return;
  const size_t p = (size_t)y * v.W + x;
  float co = __int_as_float(0x7fc00000), cf = co;
  if (x >= 1 && x < v.W - 1 && y >= 1 && y < v.H - 1) {
    PixelState ps;
    loadPixelState(v, cams[v.self], tile, x, y, ps);
    unsigned hits = 0;
    co = evalCost<Mask, kTileW, 1>(v, cams, ps, disparity[p], &hits);
    cf = (co == FLT_MAX) ? 0.f : ps.conf;
    addCounters(counters, 1u, hits);
  }
  if (outCost) outCost[p] = co;
  if (outConf) outConf[p] = cf;
}

// ---- active-pixel compaction for the fine-level stages ---------------------------------------------------
// randomProposal and pingPong skip pixels outside the FOV / foreground mask and below a variance threshold
// (Derp.cpp:765-789, 422-437).  With one thread per pixel those lanes idle while their neighbours run ~10^4
// instructions per cost evaluation, so the stages first build the list of active pixels (row scan ->
// row offsets -> scatter) and then run one thread per ACTIVE pixel.  `prefix` doubles as the per-row draw
// index of randomProposal's sequential RNG (see below).
__global__ void activeScanKernel(int W, int H, const uint8_t* __restrict__ fov, const uint8_t* __restrict__ fg,
                                 const float* __restrict__ variance, float varThresh, int* __restrict__ prefix,
                                 int* __restrict__ rowCount) {
  // one warp per row
  const int y = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (y >= H) return;
  int running = 0;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane;
    bool proc = false;
    if (x >= 1 && x < W - 1 && y >= 1 && y < H - 1) {
      const size_t p = (size_t)y * W + x;
      proc = fov[p] && (!fg || fg[p]) && !(variance[p] < varThresh);
    }
    const unsigned m = __ballot_sync(0xffffffffu, proc);
    if (x < W) prefix[(size_t)y * W + x] = proc ? running + __popc(m & ((1u << lane) - 1u)) : -1;
    running += __popc(m);
  }
  if (lane == 0) rowCount[y] = running;
}

// exclusive scan of the row counts (H <= a few thousand: one CTA); rowOffset[H] = total
__global__ void rowOffsetKernel(int H, const int* __restrict__ rowCount, int* __restrict__ rowOffset) {
  __shared__ int warpSums[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < H; base += blockDim.x) {
    const int i = base + tid;
    int v = i < H ? rowCount[i] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += n;
    }
    if (lane == 31) warpSums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      int ws = lane < (blockDim.x >> 5) ? warpSums[lane] : 0;
      int wi = ws;
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += n;
      }
      warpSums[lane] = wi - ws;  // exclusive
    }
    __syncthreads();
    const int excl = carry + warpSums[wid] + incl - v;
    if (i < H) rowOffset[i] = excl;
    __syncthreads();
    if (tid == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
  if (tid == 0) rowOffset[H] = carry;
}

// The list is ordered TILE-major (32x8 pixel tiles, rows inside a tile): the 256 consecutive entries a CTA of the
// compacted kernels works on then come from one or two adjacent tiles, so its warps gather from vertically
// adjacent texel rows and share them in L1 like the dense sweep does (row-major order shares fewer).
__global__ void tileCountKernel(int W, int H, const int* __restrict__ prefix, int* __restrict__ tileCount) {
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  const bool act = x < W && y < H && prefix[(size_t)y * W + x] >= 0;
  const int n = __syncthreads_count(act);
  if (threadIdx.x == 0 && threadIdx.y == 0) tileCount[blockIdx.y * gridDim.x + blockIdx.x] = n;
}

__global__ void activeScatterKernel(int W, int H, const int* __restrict__ prefix, const int* __restrict__ tileOffset,
                                    int* __restrict__ list) {
  __shared__ int rowCount[kBlockY];
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  const bool act = x < W && y < H && prefix[(size_t)y * W + x] >= 0;
  const unsigned m = __ballot_sync(0xffffffffu, act);
  if (threadIdx.x == 0) rowCount[threadIdx.y] = __popc(m);
  __syncthreads();
  int off = tileOffset[blockIdx.y * gridDim.x + blockIdx.x];
  for (int r = 0; r < (int)threadIdx.y; ++r) off += rowCount[r];
  if (act) list[off + __popc(m & ((1u << threadIdx.x) - 1u))] = y * W + x;
}

// ---- K7: randomProposal (Derp.cpp:750-824) -----------------------------------------------------------
// The reference walks each row sequentially with one minstd_rand0 per row (seed y*level) and draws
// exactly numProposals values for every processed pixel.  Whether a pixel is processed depends only
// on masks and variance, so the draw index of pixel x is numProposals * (#processed pixels left of
// x) = numProposals * prefix[x]: the row scan + LCG skip-ahead makes the row parallel and bit-identical.
struct ProposalArgs : DstArgs {
  const int* prefix;
  const int* list;       // active pixels
  const int* listCount;  // &rowOffset[H]
  float* disp;
  float* cost;
  float* conf;
  int numProposals, level;
  float minDispGlobal, maxDisp;
  unsigned long long* counters;
};

// pixels outside the foreground mask take the background disparity (Derp.cpp:768-771)
__global__ void backgroundFillKernel(int W, int H, const uint8_t* __restrict__ fov, const uint8_t* __restrict__ fg,
                                     const float* __restrict__ bg, float* __restrict__ disp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < 1 || x >= W - 1 || y < 1 || y >= H - 1) return;
  const size_t p = (size_t)y * W + x;
  if (fov[p] && !fg[p]) disp[p] = bg[p];
}

template <class Mask>
__global__ void __launch_bounds__(kPatchThreads, kPatchMinCtas) proposalKernel(const ProposalArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* patches = reinterpret_cast<float*>(cams + a.v.S);
  const int count = *a.listCount;
  if (blockIdx.x * kPatchThreads >= count) return;  // whole CTA idle: skip the camera staging too
  stageCameras(cams, a.v.cams, a.v.S);
  const int W = a.v.W;
  // grid-stride over the active list (the launch covers the longest possible list: normally one trip)
  unsigned hits = 0, evals = 0;
  for (int i = blockIdx.x * kPatchThreads + threadIdx.x; i < count; i += gridDim.x * kPatchThreads) {
  const int p = a.list[i];
  const int y = p / W, x = p - y * W;
  PixelState ps;
  loadPixelStateCompact<kPatchThreads>(a.v, cams[a.v.self], patches, x, y, ps);
  float currDisp = a.disp[p];
  float currCost = evalCost<Mask, kPatchRP, kPatchCP, uint2>(a.v, cams, ps, currDisp, &hits);
  float currConf = (currCost == FLT_MAX) ? 0.f : ps.conf;
  const float costThresh = fminf(0.5f * currCost, 5.0f);
  const float minDisp = a.bg ? a.bg[p] : a.minDispGlobal;
  const float maxDisp = a.maxDisp;
  float amplitude = (maxDisp - minDisp) / 2.0f;
  MinstdRand0 rng;
  rng.seed((unsigned)(y * a.level));
  rng.discard((unsigned long long)a.prefix[p] * (unsigned long long)a.numProposals);
#pragma unroll 1
  for (int k = 0; k < a.numProposals; ++k) {
    const float lo = fmaxf(minDisp, currDisp - amplitude);
    const float hi = fminf(maxDisp, currDisp + amplitude);
    const float propDisp = rng.uniform(lo, hi);
    const float propCost = evalCost<Mask, kPatchRP, kPatchCP, uint2>(a.v, cams, ps, propDisp, &hits);
    if (propCost < currCost && propCost < costThresh) {
      currCost = propCost;
      currDisp = propDisp;
      currConf = (propCost == FLT_MAX) ? 0.f : ps.conf;
      amplitude /= 2.0f;
    }
  }
  a.disp[p] = currDisp;
  a.cost[p] = currCost;
  a.conf[p] = currConf;
  evals += (unsigned)(1 + a.numProposals);
  }
  addCounters(a.counters, evals, hits);
}

// ---- K8: pingPongRectangle (Derp.cpp:403-478), one Jacobi iteration ------------------------------------
struct PingPongArgs : DstArgs {
  const float* disp;        // read
  const uint8_t* changed;   // read
  float* dispRes;           // write
  float* costRes;           // write (INF where skipped)
  uint8_t* changedNext;     // write: disp != dispRes
  const int* list;
  const int* listCount;
  unsigned long long* counters;
  unsigned long long* counters2;  // nullable: a second tally of the same work (profiling)
};

// every pixel: the values a skipped pixel ends up with (Derp.cpp:420-437, 486-487, 525-529)
__global__ void pingPongInitKernel(int W, int H, const uint8_t* __restrict__ fov, const uint8_t* __restrict__ fg,
                                   const float* __restrict__ bg, const float* __restrict__ disp,
                                   float* __restrict__ dispRes, float* __restrict__ costRes,
                                   uint8_t* __restrict__ changedNext) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  const float old = disp[p];
  float res = old;
  const bool interior = x >= 1 && x < W - 1 && y >= 1 && y < H - 1;
  if (interior && fov[p] && fg && !fg[p]) res = bg[p];
  dispRes[p] = res;
  costRes[p] = __int_as_float(0x7f800000);  // +INF
  changedNext[p] = (old != res) ? 1 : 0;
}

template <class Mask>
__global__ void __launch_bounds__(kPingThreads, kPingMinCtas) pingPongKernel(const PingPongArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* patches = reinterpret_cast<float*>(cams + a.v.S);
  const int count = *a.listCount;
  if (blockIdx.x * kPingThreads >= count) return;
  stageCameras(cams, a.v.cams, a.v.S);
  const int W = a.v.W, H = a.v.H;
  unsigned hits = 0, evals = 0;
  for (int i = blockIdx.x * kPingThreads + threadIdx.x; i < count; i += gridDim.x * kPingThreads) {
  const int p = a.list[i];
  const int y = p / W, x = p - y * W;
  PixelState ps;
  loadPixelStateCompact<kPingThreads>(a.v, cams[a.v.self], patches, x, y, ps);
  const float old = a.disp[p];
  float bestCost = __int_as_float(0x7f800000);
  float bestDisp = old;
  const float backgroundDisparity = a.bg ? a.bg[p] : 0.f;
#pragma unroll 1
  for (int k = 0; k < 9; ++k) {
    // candidateTemplateOriginal (DerpUtil.h:34-43): centre, 4-neighbours, 4 diagonals at +-2
    // offsets + 2 packed as nibbles, k = 0..8:  x: 0,-1,1,0,0,-2,2,-2,2   y: 0,0,0,-1,1,-2,-2,2,2
    const int ox = (int)((0x404022312ull >> (4 * k)) & 0xF) - 2;
    const int oy = (int)((0x440031222ull >> (4 * k)) & 0xF) - 2;
    const int xx = clampIdx(x + ox, W - 1), yy = clampIdx(y + oy, H - 1);
    const size_t q = (size_t)yy * W + xx;
    if (!a.fov[q]) continue;
    const float d = a.disp[q];
    if (d >= backgroundDisparity && a.changed[q]) {
      const float cost = evalCost<Mask, 3 * kPingThreads, kPingThreads, uint2>(a.v, cams, ps, d, &hits);
      ++evals;
      if (cost < bestCost) {
        bestCost = cost;
        bestDisp = d;
      }
    }
  }
  a.dispRes[p] = bestDisp;
  a.costRes[p] = bestCost;
  a.changedNext[p] = (old != bestDisp) ? 1 : 0;
  }
  addCounters(a.counters, evals, hits);
  if (a.counters2) addCounters(a.counters2, evals, hits);
}

// ---- K9: handleDisparityMismatch (Derp.cpp:553-720) for one destination ----------------------------------
struct MismatchArgs {
  int W, H, S, self;
  const DevCamera* cams;
  const float* dispAll;      // [S][H][W] all cameras' disparity (dst list == camera list)
  const float* variance;     // destination's
  const uint8_t* fov;
  const uint8_t* fg;
  float varNoiseFloor, varHighThresh;
  float* dispNew;            // [H][W]
  uint8_t* mask;             // [H][W]
};

__global__ void __launch_bounds__(kBlockX* kBlockY) mismatchKernel(const MismatchArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  stageCameras(cams, a.cams, a.S);
  const int W = a.W, H = a.H;
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  const size_t plane = (size_t)W * H;
  const float nan = __int_as_float(0x7fc00000);
  if (!a.fov[p]) {
    a.dispNew[p] = nan;
    return;
  }
  const float dispCurr = a.dispAll[a.self * plane + p];
  int nMatch = 0, nMis = 0;
  float mis[kMaxCams];  // disparities of the disagreeing sources: at most S - 1 of them
  if (!a.fg || a.fg[p]) {
    const DevCamera& cd = cams[a.self];
    double dir[3];
    pixelRay(cd, (x + 0.5) / W, (y + 0.5) / H, dir);
    const double depth = (double)(1.0f / dispCurr);
    const double wx = cd.pos[0] + dir[0] * depth, wy = cd.pos[1] + dir[1] * depth, wz = cd.pos[2] + dir[2] * depth;
    for (int s = 0; s < a.S; ++s) {
      if (s == a.self) continue;
      double px, py;
      if (!sees(cams[s], wx, wy, wz, &px, &py)) continue;
      px *= W;
      py *= H;
      const float dSrc = sampleF32(a.dispAll + s * plane, W, H, (float)px, (float)py);
      const float dMin = (1.0f - 0.1f) * dispCurr, dMax = (1.0f + 0.1f) * dispCurr;
      if (dMin <= dSrc && dSrc <= dMax) ++nMatch;
      else mis[nMis++] = dSrc;
    }
  }
  if (nMatch + nMis == 0) {
    a.mask[p] = 0;
    a.dispNew[p] = dispCurr;
    return;
  }
  const float var = a.variance[p];
  if (nMatch >= 1 || a.varHighThresh < var || var < a.varNoiseFloor) {
    a.mask[p] = 0;
    a.dispNew[p] = dispCurr;
  } else {
    a.mask[p] = 1;
    for (int i = 1; i < nMis; ++i) {  // ascending sort
      const float vv = mis[i];
      int j = i - 1;
      while (j >= 0 && vv < mis[j]) {
        mis[j + 1] = mis[j];
        --j;
      }
      mis[j + 1] = vv;
    }
    int closer = 0;
    for (; closer < nMis; ++closer)
      if (mis[closer] >= dispCurr) break;
    const float m = mis[closer / 2];
    a.dispNew[p] = (m < dispCurr) ? m : dispCurr;  // std::min(dispCurr, m)
  }
}

// ---- K10: generalizedJointBilateralFilter<float, Vec3w> (TemporalBilateralFilter.h:39-124) ----------
// mask = fov & fg; output copied only onto foreground pixels (Derp.cpp:900).
// One CTA filters a 32 x 8 block from a shared-memory tile with a `radius` halo: an entry holds the guide
// already scaled to [0,1] (the per-tap `colour * guideFactor` of the reference, hoisted: same fp32 product) and
// the image value, so a tap is one 16-byte shared load instead of three global loads + unpack + 3 multiplies.
// The two per-tap divisions by constants use divBy (derp_divconst.cuh).  The tap loop keeps the reference's
// order (v outer, u inner) and its left-to-right sums.
constexpr size_t kBilMaxSmem = 48 * 1024;  // tiles up to radius 17; wider filters take bilateralWideKernel
struct GuideU16 {  // packed u16 BGR texels, factor 1/65535
  const uint2* g;
  __device__ __forceinline__ float3 load(size_t q) const {
    const float f = 1 / 65535.0f;
    const Texel t = unpack(__ldg(g + q));
    return make_float3(t.b * f, t.g * f, t.r * f);
  }
};
struct GuideF32 {  // float BGR in [0,1], factor 1/1.0f (UpsampleDisparity.cpp: PixelType = Vec3f)
  const float* g;
  __device__ __forceinline__ float3 load(size_t q) const {
    const float f = 1 / 1.0f;
    return make_float3(g[q * 3] * f, g[q * 3 + 1] * f, g[q * 3 + 2] * f);
  }
};

template <class Guide>
__global__ void __launch_bounds__(kBlockX* kBlockY)
    bilateralKernel(int W, int H, const float* __restrict__ image, const Guide guide, const uint8_t* __restrict__ mask0,
                    const uint8_t* __restrict__ mask1, int radius, DivConst three, DivConst denom, float w0, float w1,
                    float w2, float* __restrict__ out) {
  extern __shared__ float4 bilTile[];
  const int TW = kBlockX + 2 * radius, TH = kBlockY + 2 * radius;
  uint8_t* tmask = reinterpret_cast<uint8_t*>(bilTile + TW * TH);
  const int bx = blockIdx.x * kBlockX - radius, by = blockIdx.y * kBlockY - radius;
  const int tid = threadIdx.y * kBlockX + threadIdx.x;
  for (int i = tid; i < TW * TH; i += kBlockX * kBlockY) {
    const int ty = i / TW, tx = i - ty * TW;
    const size_t q = (size_t)clampIdx(by + ty, H - 1) * W + clampIdx(bx + tx, W - 1);
    const float3 g = guide.load(q);
    bilTile[i] = make_float4(g.x, g.y, g.z, __ldg(image + q));
    tmask[i] = (mask0[q] && (!mask1 || mask1[q])) ? 1 : 0;
  }
  __syncthreads();
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  const int ci = (threadIdx.y + radius) * TW + threadIdx.x + radius;
  const float4 c = bilTile[ci];
  if (!tmask[ci]) {
    out[p] = c.w;  // dest = image where unmasked; non-fg pixels keep their value anyway
    return;
  }
  float sumWeight = 0.0f, weightedAvg = 0.0f;
  for (int v = -radius; v <= radius; ++v) {
    const int row = ci + v * TW;
#pragma unroll 4
    for (int u = -radius; u <= radius; ++u) {
      if (!tmask[row + u]) continue;
      const float4 n = bilTile[row + u];
      const float d0 = c.x - n.x, d1 = c.y - n.y, d2 = c.z - n.z;
      const float colorDiffSq = w0 * (d0 * d0) + w1 * (d1 * d1) + w2 * (d2 * d2);
      const float weight = expf(divBy(divBy(-colorDiffSq, three), denom));
      sumWeight += weight;
      weightedAvg += weight * n.w;
    }
  }
  out[p] = (sumWeight != 0.0f) ? weightedAvg / sumWeight : c.w;
}

// Same filter without the tile, for radii whose halo does not fit shared memory (UpsampleDisparity at 8x:
// radius = scale^2 + 1 = 65, UpsampleDisparityLib.cpp:93-96).
template <class Guide>
__global__ void bilateralWideKernel(int W, int H, const float* __restrict__ image, const Guide guide,
                                    const uint8_t* __restrict__ mask0, const uint8_t* __restrict__ mask1, int radius,
                                    DivConst three, DivConst denom, float w0, float w1, float w2, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  const float self = image[p];
  if (!(mask0[p] && (!mask1 || mask1[p]))) {
    out[p] = self;
    return;
  }
  const float3 c = guide.load(p);
  float sumWeight = 0.0f, weightedAvg = 0.0f;
  for (int v = -radius; v <= radius; ++v) {
    const int sy = clampIdx(y + v, H - 1);
    for (int u = -radius; u <= radius; ++u) {
      const size_t q = (size_t)sy * W + clampIdx(x + u, W - 1);
      if (!(mask0[q] && (!mask1 || mask1[q]))) continue;
      const float3 n = guide.load(q);
      const float d0 = c.x - n.x, d1 = c.y - n.y, d2 = c.z - n.z;
      const float colorDiffSq = w0 * (d0 * d0) + w1 * (d1 * d1) + w2 * (d2 * d2);
      const float weight = expf(divBy(divBy(-colorDiffSq, three), denom));
      sumWeight += weight;
      weightedAvg += weight * __ldg(image + q);
    }
  }
  out[p] = (sumWeight != 0.0f) ? weightedAvg / sumWeight : self;
}

// ---- K11: maskedMedianBlur radius 1 (CvUtil.h:336-385) ----------------------------------------------
__global__ void medianKernel(int W, int H, const float* __restrict__ mat, const float* __restrict__ background,
                             const uint8_t* __restrict__ fov, const uint8_t* __restrict__ fg,
                             float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  if (!(fov[p] && (!fg || fg[p]))) {
    out[p] = background ? background[p] : 0.0f;
    return;
  }
  float vals[9];
  int n = 0;
  for (int yy = y - 1; yy <= y + 1; ++yy)
    for (int xx = x - 1; xx <= x + 1; ++xx) {
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const size_t q = (size_t)yy * W + xx;
      if (!(fov[q] && (!fg || fg[q]))) continue;
      const float v = mat[q];
      if (isnan(v) || v == 0) continue;
      // sorted insert
      int j = n++;
      while (j > 0 && v < vals[j - 1]) {
        vals[j] = vals[j - 1];
        --j;
      }
      vals[j] = v;
    }
  float r = 0.0f;
  if (n > 0) {
    const int m = n / 2;
    r = (n & 1) ? vals[m] : (float)((double)(vals[m - 1] + vals[m]) / 2.0);
  }
  out[p] = r;
}

// ---- K12: maskFov (Derp.cpp:940-951) -----------------------------------------------------------------
__global__ void maskFovKernel(size_t n, const uint8_t* __restrict__ fov, float* __restrict__ disp) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !fov[i]) disp[i] = __int_as_float(0x7fc00000);
}

__global__ void copyWhereKernel(size_t n, const uint8_t* __restrict__ mask, const float* __restrict__ src,
                                float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (!mask || mask[i])) dst[i] = src[i];
}

// ---- K13: upsampling (UpsampleDisparityLib.cpp:98-147) ---------------------------------------------------
// cv::resize INTER_LANCZOS4: separable, 8 taps, index-clamped; tap tables come from the host.
__global__ void nanToKernel(size_t n, const float* __restrict__ in, float v, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float f = in[i];
    out[i] = (f != f) ? v : f;
  }
}
__global__ void lanczosHKernel(int sw, int sh, int dw, const float* __restrict__ src, const int* __restrict__ xofs,
                               const float* __restrict__ alpha, float* __restrict__ rows) {
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (dx >= dw || y >= sh) return;
  const float* S = src + (size_t)y * sw;
  const float* a = alpha + (size_t)dx * 8;
  const int sx = xofs[dx];
  float v;
  if (sx - 3 >= 0 && sx + 4 < sw) {
    v = S[sx - 3] * a[0] + S[sx - 2] * a[1] + S[sx - 1] * a[2] + S[sx] * a[3] + S[sx + 1] * a[4] +
        S[sx + 2] * a[5] + S[sx + 3] * a[6] + S[sx + 4] * a[7];
  } else {
    v = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) v += S[clampIdx(sx + j - 3, sw - 1)] * a[j];
  }
  rows[(size_t)y * dw + dx] = v;
}
__global__ void lanczosVKernel(int sh, int dw, int dh, const float* __restrict__ rows, const int* __restrict__ yofs,
                               const float* __restrict__ beta, float* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || dy >= dh) return;
  const float* b = beta + (size_t)dy * 8;
  const int sy = yofs[dy];
  float r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = rows[(size_t)clampIdx(sy - 3 + k, sh - 1) * dw + x];
  dst[(size_t)dy * dw + x] = r[0] * b[0] + r[1] * b[1] + r[2] * b[2] + r[3] * b[3] + r[4] * b[4] + r[5] * b[5] +
      r[6] * b[6] + r[7] * b[7];
}
// masked path: NaN outside coarse mask -> INTER_NEAREST -> NaN outside fine mask
__global__ void nearestMaskedKernel(int sw, int sh, int dw, int dh, const float* __restrict__ src,
                                    const uint8_t* __restrict__ maskC, const uint8_t* __restrict__ maskUp,
                                    const int* __restrict__ xofs, const int* __restrict__ yofs,
                                    float* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  const size_t q = (size_t)yofs[y] * sw + xofs[x];
  float v = maskC[q] ? src[q] : __int_as_float(0x7fc00000);
  if (!maskUp[(size_t)y * dw + x]) v = __int_as_float(0x7fc00000);
  dst[(size_t)y * dw + x] = v;
}
// replaceNans (UpsampleDisparityLib.cpp:54-91): spiral search, then background fill
__global__ void replaceNansKernel(int W, int H, const float* __restrict__ dispUp, const float* __restrict__ bg,
                                  const uint8_t* __restrict__ maskUp, const short2* __restrict__ spiral, int nSpiral,
                                  float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  float v = dispUp[p];
  if (maskUp[p] && !(v > 0)) {
    for (int i = 0; i < nSpiral; ++i) {
      const short2 o = spiral[i];
      const float d = dispUp[(size_t)clampIdx(y + o.y, H - 1) * W + clampIdx(x + o.x, W - 1)];
      if (d > 0) {
        v = d;
        break;
      }
    }
  }
  if (isnan(v) || v == 0) v = bg[p];
  out[p] = v;
}

// ---- K14: temporalJointBilateralFilter (TemporalBilateralFilter.h:126-215) ------------------------------------
struct TemporalArgs {
  int W, H, T, frameOffset, radius;
  const uint2* guides;    // [T][H][W] texels
  const float* disps;     // [T][H][W]
  const uint8_t* masks;   // [T][H][W]
  float w0, w1, w2;
  DivConst maxPix, sig2;  // 65535.0f and sigma^2 (TemporalBilateralFilter.h:176-185)
  float* out;
};
__global__ void temporalKernel(const TemporalArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= a.W || y >= a.H) return;
  const size_t plane = (size_t)a.W * a.H;
  const size_t p = (size_t)y * a.W + x;
  if (!a.masks[a.frameOffset * plane + p]) {
    a.out[p] = a.disps[a.frameOffset * plane + p];
    return;
  }
  const uint2 rt = __ldg(a.guides + a.frameOffset * plane + p);
  const int r0 = (int)(rt.x & 0xffffu), r1 = (int)(rt.x >> 16), r2 = (int)(rt.y & 0xffffu);
  float weightedSumPix = 0.0f, sumWeight = 0.0f;
  for (int t = 0; t < a.T; ++t) {
    const float dt = a.disps[t * plane + p];  // centre pixel of frame t (TemporalBilateralFilter.h:165)
    for (int u = -a.radius; u <= a.radius; ++u) {
      const int sx = clampIdx(x + u, a.W - 1);
      for (int v = -a.radius; v <= a.radius; ++v) {
        const int sy = clampIdx(y + v, a.H - 1);
        const size_t q = (size_t)sy * a.W + sx;
        if (!a.masks[t * plane + q]) continue;
        const uint2 st = __ldg(a.guides + t * plane + q);
        // (ushort - ushort) is exact in int; int -> float conversion rounds to nearest like the CPU
        const float e0 = divBy((float)(r0 - (int)(st.x & 0xffffu)), a.maxPix);
        const float e1 = divBy((float)(r1 - (int)(st.x >> 16)), a.maxPix);
        const float e2 = divBy((float)(r2 - (int)(st.y & 0xffffu)), a.maxPix);
        const float weightedDiff = a.w0 * (e0 * e0) + a.w1 * (e1 * e1) + a.w2 * (e2 * e2);
        const float weight = expf(divBy(-weightedDiff, a.sig2));
        weightedSumPix += dt * weight;
        sumWeight += weight;
      }
    }
  }
  a.out[p] = weightedSumPix / sumWeight;
}


// ---- GenerateForegroundMasks (source/render/BackgroundSubtractionUtil.h:20-59) ---------------------------------------
// cv::GaussianBlur 3 x 3, sigma 0, u16 x 3: (1 2 1; 2 4 2; 1 2 1) / 16 in fixed point, round half up, REFLECT_101
__global__ void gaussian3Kernel(const uint16_t* __restrict__ src, int w, int h, uint16_t* __restrict__ dst) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (e >= w * 3) return;
  const int x = e / 3, c = e - x * 3;
  const int ys[3] = {reflect101(y - 1, h), y, reflect101(y + 1, h)};
  const int xs[3] = {reflect101(x - 1, w), x, reflect101(x + 1, w)};
  unsigned s = 0;
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) s += (unsigned)((j == 1 ? 2 : 1) * (i == 1 ? 2 : 1)) * src[((size_t)ys[j] * w + xs[i]) * 3 + c];
  dst[((size_t)y * w + x) * 3 + c] = (uint16_t)((s + 8u) >> 4);
}
// cv::GaussianBlur((2 r + 1)^2, sigma 0) on u16 x 3 for any radius up to kGaussMaxRadius (derp_gaussian_blur): OpenCV's
// bit-exact fixed-point path.  Taps carry 16 fraction bits and sum to 2^16 (built on the host, gaussTaps in derp_b200.cu).
// The row pass keeps exact u32 sums (at most 65535 * 2^16); the column pass sums those in u64 and rounds with
// (s + 2^31) >> 32.  Borders are REFLECT_101, folded as often as an image smaller than the kernel needs.
constexpr int kGaussMaxRadius = 64;
struct GaussTaps {
  int r;
  uint32_t k[2 * kGaussMaxRadius + 1];  // k[r - i] == k[r + i]
};
__device__ __forceinline__ int reflect101Fold(int p, int len) {  // == reflect101, in closed form: period 2 (len - 1)
  if (len == 1) return 0;
  const int period = 2 * (len - 1);
  p = abs(p) % period;
  return p < len ? p : period - p;
}
// Row pass: one block per kGaussRowPixels pixels of a row; the row segment and its aprons are staged in shared memory as
// u32 elements (interleaved like the image, so consecutive threads read consecutive words)
constexpr int kGaussRowPixels = 256;
__global__ void __launch_bounds__(256) gaussRowKernel(const uint16_t* __restrict__ src, int w, int h, GaussTaps t,
                                                      uint32_t* __restrict__ rows) {
  extern __shared__ uint32_t sRow[];
  const int r = t.r, x0 = blockIdx.x * kGaussRowPixels;
  const int px = min(kGaussRowPixels, w - x0), ne = 3 * (px + 2 * r);
  for (int y = blockIdx.y; y < h; y += gridDim.y) {  // the grid's y extent is capped at 65535 rows
    const uint16_t* S = src + (size_t)y * w * 3;
    for (int e = threadIdx.x; e < ne; e += blockDim.x) {
      const int p = e / 3, c = e - 3 * p;
      sRow[e] = S[reflect101Fold(x0 - r + p, w) * 3 + c];
    }
    __syncthreads();
    uint32_t* D = rows + ((size_t)y * w + x0) * 3;
    for (int e = threadIdx.x; e < 3 * px; e += blockDim.x) {
      const uint32_t* s = sRow + e + 3 * r;  // the output element's own tap
      uint32_t sum = t.k[r] * s[0];
      for (int i = 1; i <= r; ++i) sum += t.k[r - i] * (s[-3 * i] + s[3 * i]);  // < 2^32: the taps sum to 2^16
      D[e] = sum;
    }
    __syncthreads();
  }
}
// Column pass: a block covers kGaussColElems elements of kGaussColRows output rows and stages the rows it reads
constexpr int kGaussColElems = 32, kGaussColRows = 64, kGaussColThreadsY = 8;
__global__ void __launch_bounds__(kGaussColElems* kGaussColThreadsY) gaussColKernel(const uint32_t* __restrict__ rows, int w,
                                                                                   int h, GaussTaps t,
                                                                                   uint16_t* __restrict__ dst) {
  extern __shared__ uint32_t sCol[];
  const int r = t.r, n = 3 * w, tx = threadIdx.x;
  const int e = blockIdx.x * kGaussColElems + tx, y0 = blockIdx.y * kGaussColRows;
  const int ny = min(kGaussColRows, h - y0), nr = ny + 2 * r;
  for (int j = threadIdx.y; j < nr; j += kGaussColThreadsY)
    sCol[j * kGaussColElems + tx] = e < n ? rows[(size_t)reflect101Fold(y0 - r + j, h) * n + e] : 0u;
  __syncthreads();
  if (e >= n) return;
  for (int j = threadIdx.y; j < ny; j += kGaussColThreadsY) {
    const uint32_t* s = sCol + j * kGaussColElems + tx;
    unsigned long long sum = 0;
    for (int i = 0; i <= 2 * r; ++i) sum += (unsigned long long)t.k[i] * s[i * kGaussColElems];
    dst[(size_t)(y0 + j) * n + e] = (uint16_t)((sum + (1ull << 31)) >> 32);
  }
}
// mask = || float(template) - float(frame) ||_2 > threshold; cv::norm accumulates the squares in double
__global__ void foregroundDiffKernel(size_t n, const uint16_t* __restrict__ templ, const uint16_t* __restrict__ frame, float threshold,
                                     uint8_t* __restrict__ mask) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float alpha = 1.0f / 65535.0f;
  double s = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float d = fabsf((float)templ[i * 3 + c] * alpha - (float)frame[i * 3 + c] * alpha);
    s += (double)d * (double)d;
  }
  mask[i] = sqrt(s) > (double)threshold ? 1 : 0;
}
// cv::dilate / cv::erode with a k x k rectangle anchored at k / 2; border taps never win
__global__ void morphRectKernel(const uint8_t* __restrict__ src, int w, int h, int k, int dilate, uint8_t* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int a = k / 2;
  unsigned v = dilate ? 0u : 255u;
  for (int j = -a; j < k - a; ++j) {
    const int yy = y + j;
    if (yy < 0 || yy >= h) continue;
    for (int i = -a; i < k - a; ++i) {
      const int xx = x + i;
      if (xx < 0 || xx >= w) continue;
      const unsigned t = src[(size_t)yy * w + xx];
      v = dilate ? max(v, t) : min(v, t);
    }
  }
  dst[(size_t)y * w + x] = (uint8_t)v;
}

}  // namespace derp
