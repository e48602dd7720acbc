// ORACLE — TEST INFRASTRUCTURE ONLY.  What the reference's RigSimulator.cpp (and the headers it includes:
// BoundingVolumeHierarchy.h, RaytracingPrimitives.h) uses beyond ../refshim and ../sweepshim.  rigsim.mk appends this
// header to its generated copy of ../refshim/opencv2/core.hpp, in which the stand-in's resize is renamed resizeShim and
// its aborting vconcat is dropped.  The arithmetic follows OpenCV 4's matx.hpp and resize.cpp:
//   * norm(Vec): the sum of squares accumulated in double from 0, then std::sqrt (normL2Sqr<_Tp, double>);
//   * Vec / float: each element times the float 1.f / alpha;
//   * resize INTER_AREA on float images by an integer factor k (resizeAreaFast_): factor 2 with 1 or 4 channels takes
//     the SIMD body ((a + b) + (c + d)) * 0.25f; otherwise the k * k samples of a cell, in row order, are added to a
//     float sum in groups of four (sum += ((s0 + s1) + s2) + s3, then the remainder one by one) and the sum is
//     multiplied by 1.f / (k * k).  tests/golden/rigsim_vectors.npz pins this to cv2 4.13.
#pragma once
#include <cmath>
#include <cstring>

namespace cv {
typedef Vec<int, 3> Vec3i;

template <class T, int N>
inline double norm(const Vec<T, N>& a) {
  double s = 0;
  for (int i = 0; i < N; ++i) s += (double)a.val[i] * (double)a.val[i];
  return std::sqrt(s);
}

template <class T, int N>
inline Vec<T, N> operator/(const Vec<T, N>& a, float alpha) {
  const float s = 1.f / alpha;
  Vec<T, N> r;
  for (int i = 0; i < N; ++i) r.val[i] = saturate_cast<T>(a.val[i] * s);
  return r;
}

// MatExpr a * s assigned to a Mat: convertTo(dst, -1, s) on 32F, i.e. each element times (float)s
inline Mat_<float> operator*(const Mat_<float>& a, double s) { return a * (float)s; }

inline void resize(const Mat& src, Mat& dst, Size dsize, double fx, double fy, int interpolation) {
  const int cn = src.channels();
  if (interpolation != INTER_AREA || src.depth() != CV_32F || dsize.width < 1 || dsize.height < 1) {
    resizeShim(src, dst, dsize, fx, fy, interpolation);
    return;
  }
  const int kx = src.cols / dsize.width, ky = src.rows / dsize.height;
  if (kx != ky || kx * dsize.width != src.cols || ky * dsize.height != src.rows)
    shimUnsupported("INTER_AREA other than by one integer factor on both axes");
  Mat out(dsize.height, dsize.width, src.type());
  const float* S = src.ptr<float>();
  float* D = out.ptr<float>();
  const size_t row = (size_t)src.cols * cn;
  const int k = kx, area = k * k;
  const float scale = 1.f / area;
  for (int y = 0; y < dsize.height; ++y)
    for (int x = 0; x < dsize.width; ++x)
      for (int c = 0; c < cn; ++c) {
        const float* s0 = S + (size_t)y * k * row + (size_t)x * k * cn + c;
        float v;
        if (k == 2 && (cn == 1 || cn == 4)) {
          v = ((s0[0] + s0[cn]) + (s0[row] + s0[row + cn])) * 0.25f;
        } else {
          float sum = 0;
          int i = 0;
          auto at = [&](int j) { return s0[(size_t)(j / k) * row + (size_t)(j % k) * cn]; };
          for (; i <= area - 4; i += 4) sum += at(i) + at(i + 1) + at(i + 2) + at(i + 3);
          for (; i < area; ++i) sum += at(i);
          v = sum * scale;
        }
        D[((size_t)y * dsize.width + x) * cn + c] = v;
      }
  dst = out;
}

inline void vconcat(const Mat& a, const Mat& b, Mat& dst) {
  if (a.type() != b.type() || a.cols != b.cols) shimUnsupported("vconcat of Mats of different types or widths");
  Mat out(a.rows + b.rows, a.cols, a.type());
  const size_t na = a.total() * a.elemSize(), nb = b.total() * b.elemSize();
  std::memcpy(out.data, a.data, na);
  std::memcpy(out.data + na, b.data, nb);
  dst = out;
}
}  // namespace cv

#include <Eigen/Geometry>
namespace Eigen {
typedef Matrix<float, 3, 1> Vector3f;
template <class M>
struct Map;
template <class S, int N>
struct Map<const Matrix<S, N, 1>> {
  const S* p;
  explicit Map(const S* p) : p(p) {}
  template <class T>
  Matrix<T, N, 1> cast() const {
    Matrix<T, N, 1> r;
    for (int i = 0; i < N; ++i) r.v[i] = (T)p[i];
    return r;
  }
};
// Eigen promotes a float scalar to the double matrix's scalar type (promote_scalar_arg)
template <int N>
inline Matrix<double, N, 1> operator*(float s, const Matrix<double, N, 1>& m) { return m * (double)s; }
}  // namespace Eigen
