// cv::resize(src, dsize, INTER_AREA) [then cv::threshold(., t, 255, THRESH_BINARY)] of interleaved images of 8-bit, 16-bit
// or float samples with 1, 3 or 4 channels, either direction (derp_resize_area, derp_downscale_area): OpenCV 4.13's
// modules/imgproc/src/resize.cpp restated path by path, one thread per destination sample.  Built with -fmad=false, so
// every product and sum is rounded on its own like the C++ (SSE baseline, no FMA) it restates.
//   * integer ratios (resizeAreaFast_): 2 x 2 on 8- and 16-bit samples is (a + b + c + d + 2) >> 2; 2 x 2 on floats with 1
//     or 4 channels is the SIMD body ((a + b) + (c + d)) * 0.25f, except the scalar tail of a 1-channel row (the last
//     dw % kCvF32Lanes samples); everything else is the sum of the kx * ky samples in row order times 1.f / (kx * ky) --
//     an int for 8-bit, a float fed by exact int groups of four for 16-bit, a float fed by float groups of four for float
//     (CV_ENABLE_UNROLLED: sum += ((s0 + s1) + s2) + s3);
//   * other ratios when no axis grows (ResizeArea_Invoker<T, float>): separable weighted sums in float in the table order
//     of computeResizeAreaTab (built on the host, areaTaps in derp_b200.cu);
//   * an axis grows (INTER_AREA's bilinear variant, resizeGeneric_ with HResizeLinear / VResizeLinear, used for both axes):
//     two taps per axis at s = floor(d * scale); floats and 16-bit weight in float, rows first, cvRound and saturation at
//     the end; 8-bit in fixed point with weights round(w * 2048), exact int rows and the SIMD rounding of the columns.
// The functions below are __host__ __device__ so that the arithmetic is one piece of code wherever it runs.
#pragma once

#include <cmath>
#include <cstdint>
#include <type_traits>

#ifdef __CUDACC__
#define DERP_RESIZE_HD __host__ __device__ __forceinline__
#else
#define DERP_RESIZE_HD inline
#endif

namespace derp {

// float lanes of OpenCV's baseline SIMD width (128-bit SSE) in ResizeAreaFastVec_SIMD_32f
constexpr int kCvF32Lanes = 4;
// INTER_RESIZE_COEF_SCALE: the fixed-point unit of 8-bit linear weights
constexpr int kResizeCoefScale = 2048;

// One output sample's two taps on one axis of the bilinear variant: source index s (s + 1 is clipped by the caller), float
// weights (1 - f, f) and their fixed-point form for 8-bit images
struct LinearTap {
  int s;
  float w0, w1;
  int i0, i1;
};

DERP_RESIZE_HD int cvRoundF(float v) {  // cvRound: to nearest, ties to even
#ifdef __CUDA_ARCH__
  return __float2int_rn(v);
#else
  return (int)std::lrintf(v);
#endif
}

// saturate_cast<T>(v), then the optional binary threshold (v > t ? 255 : 0)
template <typename T>
DERP_RESIZE_HD T thresholded(T v, int t) {
  if (t < 0) return v;
  if constexpr (std::is_same<T, float>::value)
    return v > (float)t ? 255.f : 0.f;
  else
    return (int)v > t ? (T)255 : (T)0;
}
template <typename T>
DERP_RESIZE_HD T saturateF(float v) {
  if constexpr (std::is_same<T, float>::value) {
    return v;
  } else {
    constexpr int hi = std::is_same<T, uint8_t>::value ? 255 : 65535;
    const int r = cvRoundF(v);
    return (T)(r < 0 ? 0 : (r > hi ? hi : r));
  }
}

// resizeAreaFast_: destination sample (dx, c) of row dy at integer ratios kx, ky; row = sw * C samples
template <typename T, int C>
DERP_RESIZE_HD T areaFastAt(const T* src, int sw, int dw, int dx, int c, int dy, int kx, int ky) {
  const size_t row = (size_t)sw * C;
  const T* S = src + (size_t)dy * ky * row + (size_t)dx * kx * C + c;
  if (kx == 2 && ky == 2) {
    if constexpr (!std::is_same<T, float>::value) {
      return (T)(((int)S[0] + (int)S[C] + (int)S[row] + (int)S[row + C] + 2) >> 2);
    } else if (C == 4 || (C == 1 && dx < dw / kCvF32Lanes * kCvF32Lanes)) {
      return ((S[0] + S[C]) + (S[row] + S[row + C])) * 0.25f;
    }
  }
  const int area = kx * ky;
  const float scale = 1.f / (float)area;
  auto at = [&](int k) { return S[(size_t)(k / kx) * row + (size_t)(k % kx) * C]; };
  if constexpr (std::is_same<T, uint8_t>::value) {
    int sum = 0;
    for (int k = 0; k < area; ++k) sum += at(k);
    return saturateF<T>((float)sum * scale);
  } else {
    float sum = 0.f;
    int k = 0;
    for (; k <= area - 4; k += 4) {
      if constexpr (std::is_same<T, uint16_t>::value)
        sum = sum + (float)((int)at(k) + (int)at(k + 1) + (int)at(k + 2) + (int)at(k + 3));
      else
        sum = sum + (((at(k) + at(k + 1)) + at(k + 2)) + at(k + 3));
    }
    for (; k < area; ++k) sum = sum + (float)at(k);
    return saturateF<T>(sum * scale);
  }
}

// ResizeArea_Invoker<T, float>: xs / xa are the source column and weight of each horizontal tap, xo[dx] .. xo[dx + 1] its
// taps; the same for rows.  The first destination row starts from sum = 0 (0 + t: a -0 becomes +0); every later row
// ASSIGNS its first product (resize.cpp: sum[dx] = beta * buf[dx]), as one OpenCV thread does over the whole image.
template <typename T, int C>
DERP_RESIZE_HD T areaGeneralAt(const T* src, int sw, int dx, int c, int dy, const int* xo, const int* xs, const float* xa,
                               const int* yo, const int* ys, const float* ya) {
  const int k0 = xo[dx], k1 = xo[dx + 1];
  float sum = 0.f;
  for (int j = yo[dy]; j < yo[dy + 1]; ++j) {
    const T* S = src + (size_t)ys[j] * sw * C + c;
    float buf = 0.f;
    for (int k = k0; k < k1; ++k) buf = buf + (float)S[(size_t)xs[k] * C] * xa[k];
    const float t = ya[j] * buf;
    sum = (j == yo[dy] && dy != 0) ? t : sum + t;
  }
  return saturateF<T>(sum);
}

// resizeGeneric_ in area mode: columns dx >= xmax (s + 1 past the last column) take S[s] * ONE, the rest both taps even at
// weight 0; rows s and min(s + 1, sh - 1) always both.
template <typename T, int C>
DERP_RESIZE_HD T areaEnlargeAt(const T* src, int sw, int sh, int dx, int c, int dy, const LinearTap* xt, int xmax,
                               const LinearTap* yt) {
  const LinearTap tx = xt[dx], ty = yt[dy];
  const int r0 = ty.s, r1 = ty.s + 1 < sh ? ty.s + 1 : sh - 1;
  const T* A = src + (size_t)r0 * sw * C + (size_t)tx.s * C + c;
  const T* B = src + (size_t)r1 * sw * C + (size_t)tx.s * C + c;
  const bool two = dx < xmax;
  if constexpr (std::is_same<T, uint8_t>::value) {
    const int h0 = two ? (int)A[0] * tx.i0 + (int)A[C] * tx.i1 : (int)A[0] * kResizeCoefScale;
    const int h1 = two ? (int)B[0] * tx.i0 + (int)B[C] * tx.i1 : (int)B[0] * kResizeCoefScale;
    return (uint8_t)((((ty.i0 * (h0 >> 4)) >> 16) + ((ty.i1 * (h1 >> 4)) >> 16) + 2) >> 2);
  } else {
    const float h0 = two ? (float)A[0] * tx.w0 + (float)A[C] * tx.w1 : (float)A[0] * 1.f;
    const float h1 = two ? (float)B[0] * tx.w0 + (float)B[C] * tx.w1 : (float)B[0] * 1.f;
    return saturateF<T>(h0 * ty.w0 + h1 * ty.w1);
  }
}

#ifdef __CUDACC__
// One thread per destination sample e = dx * C + c; blockIdx.y strides over rows (the grid's y extent is capped)
template <typename T, int C>
__global__ void areaResizeFastKernel(const T* __restrict__ src, int sw, T* __restrict__ dst, int dw, int dh, int kx, int ky,
                                     int thr) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;  // dw * C <= INT_MAX: no wrap in the last block
  if (e >= (unsigned)(dw * C)) return;
  const int dx = (int)(e / C), c = (int)(e - (unsigned)dx * C);
  for (int dy = blockIdx.y; dy < dh; dy += gridDim.y)
    dst[(size_t)dy * dw * C + e] = thresholded(areaFastAt<T, C>(src, sw, dw, dx, c, dy, kx, ky), thr);
}
template <typename T, int C>
__global__ void areaResizeKernel(const T* __restrict__ src, int sw, T* __restrict__ dst, int dw, int dh,
                                 const int* __restrict__ xo, const int* __restrict__ xs, const float* __restrict__ xa,
                                 const int* __restrict__ yo, const int* __restrict__ ys, const float* __restrict__ ya,
                                 int thr) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;  // dw * C <= INT_MAX: no wrap in the last block
  if (e >= (unsigned)(dw * C)) return;
  const int dx = (int)(e / C), c = (int)(e - (unsigned)dx * C);
  for (int dy = blockIdx.y; dy < dh; dy += gridDim.y)
    dst[(size_t)dy * dw * C + e] = thresholded(areaGeneralAt<T, C>(src, sw, dx, c, dy, xo, xs, xa, yo, ys, ya), thr);
}
template <typename T, int C>
__global__ void areaEnlargeKernel(const T* __restrict__ src, int sw, int sh, T* __restrict__ dst, int dw, int dh,
                                  const LinearTap* __restrict__ xt, int xmax, const LinearTap* __restrict__ yt, int thr) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;  // dw * C <= INT_MAX: no wrap in the last block
  if (e >= (unsigned)(dw * C)) return;
  const int dx = (int)(e / C), c = (int)(e - (unsigned)dx * C);
  for (int dy = blockIdx.y; dy < dh; dy += gridDim.y)
    dst[(size_t)dy * dw * C + e] = thresholded(areaEnlargeAt<T, C>(src, sw, sh, dx, c, dy, xt, xmax, yt), thr);
}
#endif

}  // namespace derp
