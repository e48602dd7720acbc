// Interval arithmetic for the device's proofs of the reference's decisions, shared by derp_sweepview.cuh
// (ProjectEquirectsToCameras) and derp_riganalysis.cuh (RigAnalyzer), and the rig point both prove things about.
//
// The device's transcendentals are not glibc's to the last bit, so where a decision depends on one, the device repeats
// the chain on intervals and decides only when the interval proves the decision; otherwise the host recomputes the case
// with the same DERP_HD code and the C library.  Every IEEE operation of a chain is bracketed by its round-down and
// round-up results (exact arithmetic lies between them, and round-to-nearest of any point of the operands' intervals
// does too, the operations being monotone in each operand over the intervals where they are applied).  Each
// transcendental result t is widened by (device bound + host bound + 1) ulp of |t|, the + 1 covering the difference
// between the ulp at t and at the exact value, plus, for sin / cos, the width of their argument's interval (both are
// 1-Lipschitz).  Device bounds: the CUDA C++ Programming Guide's maximum ulp errors (double sin, cos, atan, asin, atan2:
// 2; acosf: 2; atan2f: 3).  Host bound: glibc's published maxima for x86_64 ("Known Maximum Errors in Math Functions")
// are at most 1 ulp for these; 2 is budgeted.
#pragma once

#include "derp_camera.cuh"

namespace derp {

// rig({x + .5, y + .5}, depth) = position + ray * depth (Camera.h:141-143, ParametrizedLine::pointAt)
DERP_HD void rigPoint(const DevCamera& c, int x, int y, double depth, double* w) {
  double dir[3];
  pixelRay(c, x + 0.5, y + 0.5, dir);
  for (int k = 0; k < 3; ++k) w[k] = c.pos[k] + dir[k] * depth;
}

#if defined(__CUDACC__)
struct Iv {
  double lo, hi;
};
constexpr double kTwoPi = 2 * M_PI;
constexpr int kHostUlps = 2;
constexpr int kSinUlps = 2 + kHostUlps + 1, kAtanUlps = 2 + kHostUlps + 1;  // double sin, cos, atan, asin
constexpr int kAtan2Ulps = 2 + kHostUlps + 1;                              // double atan2
constexpr int kAcosfUlps = 2 + kHostUlps + 1, kAtan2fUlps = 3 + kHostUlps + 1;

// extra + k ulp of a double function's result t, rounded up (ulp(t) <= 2^-52 |t|; 2^-1074 below the normal range)
__device__ __forceinline__ double errD(double t, int k, double extra) {
  return __dadd_ru(__dmul_ru(k * 0x1p-52, __dadd_ru(fabs(t), extra)), __dadd_ru(extra, k * 0x1p-1074));
}
__device__ __forceinline__ Iv widenD(double t, int k, double extra) {
  const double e = errD(t, k, extra);
  return Iv{__dadd_rd(t, -e), __dadd_ru(t, e)};
}
// the same for a float function, in double (ulp(t) <= 2^-23 |t|; 2^-149 below the normal range)
__device__ __forceinline__ Iv widenF(float t, int k) {
  const double e = __dadd_ru(__dmul_ru(k * 0x1p-23, fabs((double)t)), k * 0x1p-149);
  return Iv{__dadd_rd(t, -e), __dadd_ru(t, e)};
}
__device__ __forceinline__ Iv ivAdd(Iv a, Iv b) { return Iv{__dadd_rd(a.lo, b.lo), __dadd_ru(a.hi, b.hi)}; }
__device__ __forceinline__ Iv ivScale(Iv a, double s) {  // a * s, s a point
  return s >= 0 ? Iv{__dmul_rd(a.lo, s), __dmul_ru(a.hi, s)} : Iv{__dmul_rd(a.hi, s), __dmul_ru(a.lo, s)};
}
__device__ __forceinline__ Iv ivDivPos(Iv a, double d) { return Iv{__ddiv_rd(a.lo, d), __ddiv_ru(a.hi, d)}; }  // d > 0
__device__ __forceinline__ Iv ivSqr(Iv a) {
  if (a.lo >= 0) return Iv{__dmul_rd(a.lo, a.lo), __dmul_ru(a.hi, a.hi)};
  if (a.hi <= 0) return Iv{__dmul_rd(a.hi, a.hi), __dmul_ru(a.lo, a.lo)};
  return Iv{0.0, fmax(__dmul_ru(a.lo, a.lo), __dmul_ru(a.hi, a.hi))};
}
// a / d with d a positive interval
__device__ __forceinline__ Iv ivDiv(Iv a, Iv d) {
  return Iv{fmin(__ddiv_rd(a.lo, d.lo), __ddiv_rd(a.lo, d.hi)), fmax(__ddiv_ru(a.hi, d.lo), __ddiv_ru(a.hi, d.hi))};
}
__device__ __forceinline__ Iv ivFloat(Iv a) { return Iv{__double2float_rd(a.lo), __double2float_ru(a.hi)}; }

// rigPoint on intervals: sensorToCamera's branches depend only on exactly computed values (the sensor point, its norm
// and undistort's result), so the interval follows the same branch as any IEEE evaluation
__device__ __forceinline__ void rigPointIv(const DevCamera& c, int px, int py, double depth, Iv* w) {
  const double sx = (px + 0.5 - c.principal[0]) / c.focal[0];
  const double sy = (py + 0.5 - c.principal[1]) / c.focal[1];
  const double squaredNorm = sx * sx + sy * sy;
  Iv u[3];
  if (squaredNorm == 0) {
    u[0] = u[1] = Iv{0.0, 0.0};
    u[2] = Iv{-1.0, -1.0};
  } else {
    const double norm = sqrt(squaredNorm);
    const double r = undistort(c, norm);
    double theta, eTheta = 0;  // theta +- eTheta holds the host's theta
    if (c.type == DERP_CAM_FTHETA) {
      theta = r;
    } else if (c.type == DERP_CAM_RECTILINEAR) {
      theta = atan(r);
      eTheta = errD(theta, kAtanUlps, 0);
    } else if (c.type == DERP_CAM_EQUISOLID) {
      if (r <= 2) {
        const double a = asin(r / 2);
        theta = 2 * a;
        eTheta = 2 * errD(a, kAtanUlps, 0);
      } else {
        theta = 3.14159265358979323846;
      }
    } else {
      if (r <= 1) {
        theta = asin(r);
        eTheta = errD(theta, kAtanUlps, 0);
      } else {
        theta = 3.14159265358979323846 / 2;
      }
    }
    const Iv s = widenD(sin(theta), kSinUlps, eTheta), co = widenD(cos(theta), kSinUlps, eTheta);
    const Iv f = ivDivPos(s, norm);
    u[0] = ivScale(f, sx);
    u[1] = ivScale(f, sy);
    u[2] = Iv{-co.hi, -co.lo};
  }
  for (int k = 0; k < 3; ++k) {
    const Iv d = ivAdd(ivAdd(ivScale(u[0], c.rot[k]), ivScale(u[1], c.rot[3 + k])), ivScale(u[2], c.rot[6 + k]));
    w[k] = ivAdd(Iv{c.pos[k], c.pos[k]}, ivScale(d, depth));
  }
}
#endif

}  // namespace derp
