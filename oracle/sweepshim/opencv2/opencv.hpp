// ORACLE — TEST INFRASTRUCTURE ONLY.  The <opencv2/opencv.hpp> umbrella for GenerateEquirect.cpp, plus what the two
// sweep-view apps use beyond ../refshim: cv::putText (declared; aborts if called — the bridges never draw the depth
// label) and Vec / int with matx.hpp's rule (Vec(a, 1. / alpha, Matx_ScaleOp()): each element times the fp64
// reciprocal, then saturate_cast to the element type).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <string>

#include <opencv2/core.hpp>
#include <opencv2/highgui.hpp>
#include <opencv2/imgproc.hpp>

namespace cv {
typedef Point_<float> Point2f;
struct Scalar {  // Scalar_<double>: four doubles, converted to a Vec element by element with saturate_cast
  double val[4];
  Scalar(double v0 = 0, double v1 = 0, double v2 = 0, double v3 = 0) : val{v0, v1, v2, v3} {}
  template <class T, int N>
  operator Vec<T, N>() const {
    Vec<T, N> r;
    for (int i = 0; i < N && i < 4; ++i) r.val[i] = saturate_cast<T>(val[i]);
    return r;
  }
};
enum { FONT_HERSHEY_PLAIN = 1 };
inline void putText(const Mat&, const std::string&, Point_<float>, int, double, Scalar) {
  std::fprintf(stderr, "refshim: cv::putText is not implemented\n");
  std::abort();
}
template <class T, int N>
inline Vec<T, N> operator/(const Vec<T, N>& a, int alpha) {
  const double s = 1. / alpha;
  Vec<T, N> r;
  for (int i = 0; i < N; ++i) r.val[i] = saturate_cast<T>(a.val[i] * s);
  return r;
}
}  // namespace cv
