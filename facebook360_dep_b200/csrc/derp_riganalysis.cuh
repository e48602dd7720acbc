// RigAnalyzer's coverage counts (include/derp_riganalysis.h): per point, the number of cameras that see it.
//
// The DERP_HD functions are the reference's loops (RigAnalyzer.cpp:346-460, 557-589) over derp::sees; the host runs
// them with the C library, for the points the device leaves undecided and for the CPU tests.  The device kernels run
// one thread per point and decide a camera only when the decision is provably the reference's:
//   - RECTILINEAR, EQUISOLID and ORTHOGRAPHIC cameras at an exact point: Camera::sees is IEEE arithmetic (products,
//     sums, quotients, sqrt; -fmad=false keeps them uncontracted), so derp::sees gives the reference's bits.
//   - FTHETA cameras, and every camera in camera mode, whose point rig({x + .5, y + .5}, distance) is only known to an
//     interval (rigPointIv): seesIv repeats Camera::sees on intervals (derp_interval.cuh's rounding argument and ulp
//     bounds; atan2 over the box of its arguments has its extremes at the corners, being monotone in each argument
//     away from the origin).  A camera is decided when the interval fixes the FOV branch, the sensor test and, for
//     timing, the float t; an interval that contains NaN or does not fix them leaves the point to the host.
//   - Timing: minTimingDiff is the least fl(|t_i - t_j|) over pairs of seeing cameras (or 1.0).  Over sorted t the
//     least pairwise difference is an adjacent one, and rounding is monotone, so the device sorts t into a local list of
//     kTimingCap entries and takes adjacent differences; a point seen by more cameras, or with a NaN t (whose
//     differences the reference's std::min skips), goes to the host.
#pragma once

#include "derp_camera.cuh"
#include "derp_interval.cuh"

namespace derp {
namespace rig {

// ---- the reference's per-point loops (host and tests) ---------------------------------------------------------------
// saveEquirect's per-pixel loop (RigAnalyzer.cpp:398-419); t: scratch for n floats
DERP_HD int countTiming(const DevCamera* cams, int n, double x, double y, double z, float* t, double* minTimingDiff) {
  int count = 0;
  for (int i = 0; i < n; ++i) {
    double px, py;
    if (sees(cams[i], x, y, z, &px, &py)) t[count++] = (float)(py / cams[i].res[1]);
  }
  double m = 1.0;
  for (int i = 0; i < count; ++i)
    for (int j = i + 1; j < count; ++j) {
      const double d = fabsf(t[i] - t[j]);
      m = d < m ? d : m;  // std::min(m, d): a NaN d leaves m
    }
  *minTimingDiff = m;
  return count;
}

DERP_HD int countSees(const DevCamera* cams, int n, double x, double y, double z) {
  int count = 0;
  for (int i = 0; i < n; ++i) {
    double px, py;
    if (sees(cams[i], x, y, z, &px, &py)) ++count;
  }
  return count;
}

// saveCamera's pixel (RigAnalyzer.cpp:359-368); edge2: cam's image-circle edge, squared (imageCircleEdge2)
DERP_HD int countCameraPixel(const DevCamera* cams, int n, int cam, double edge2, int x, int y, double distance) {
  const DevCamera& c = cams[cam];
  const double px = x + 0.5, py = y + 0.5;
  if (!c.defaultFov) {  // isOutsideImageCircle (Camera.h:166-178)
    const double sx = (px - c.principal[0]) / c.focal[0], sy = (py - c.principal[1]) / c.focal[1];
    if (sx * sx + sy * sy >= edge2) return 0;
  }
  double w[3];
  rigPoint(c, x, y, distance, w);
  return countSees(cams, n, w[0], w[1], w[2]);
}

// |cameraToSensor(0, sinFov, -cosFov)|^2, the image-circle edge; on the host, so FTHETA's atan2 is the C library's
inline double imageCircleEdge2(const DevCamera& c) {
  const double sinFov = sqrt(1 - c.cosFov * c.cosFov);
  double ex, ey;
  cameraToSensor(c, 0.0, sinFov, -c.cosFov, &ex, &ey);
  return ex * ex + ey * ey;
}

#if defined(__CUDACC__)
// ---- the device's proof ------------------------------------------------------------------------------------------
constexpr int kNotSeen = 0, kSeen = 1, kUndecided = -1;
constexpr int kTimingCap = 32;

__device__ __forceinline__ Iv ivAddPt(Iv a, double b) { return Iv{__dadd_rd(a.lo, b), __dadd_ru(a.hi, b)}; }
__device__ __forceinline__ Iv ivNeg(Iv a) { return Iv{-a.hi, -a.lo}; }
__device__ __forceinline__ Iv ivMul(Iv a, Iv b) {
  const double l0 = __dmul_rd(a.lo, b.lo), l1 = __dmul_rd(a.lo, b.hi), l2 = __dmul_rd(a.hi, b.lo),
               l3 = __dmul_rd(a.hi, b.hi);
  const double h0 = __dmul_ru(a.lo, b.lo), h1 = __dmul_ru(a.lo, b.hi), h2 = __dmul_ru(a.hi, b.lo),
               h3 = __dmul_ru(a.hi, b.hi);
  return Iv{fmin(fmin(l0, l1), fmin(l2, l3)), fmax(fmax(h0, h1), fmax(h2, h3))};
}
__device__ __forceinline__ Iv ivSqrt(Iv a) { return Iv{__dsqrt_rd(a.lo), __dsqrt_ru(a.hi)}; }  // a.lo >= 0
__device__ __forceinline__ Iv ivDot(const double* row, const Iv* v) {  // (row0 v0 + row1 v1) + row2 v2
  return ivAdd(ivAdd(ivScale(v[0], row[0]), ivScale(v[1], row[1])), ivScale(v[2], row[2]));
}
__device__ __forceinline__ bool ivOk(Iv a) { return a.lo <= a.hi; }  // false when either end is NaN

// distortFactor / distort (Camera.h:225-241) on an interval
__device__ __forceinline__ Iv distortFactorIv(const DevCamera& c, Iv r2) {
  Iv result{c.dist[2], c.dist[2]};
  result = ivAddPt(ivMul(r2, result), c.dist[1]);
  result = ivAddPt(ivMul(r2, result), c.dist[0]);
  return ivAddPt(ivMul(r2, result), 1.0);
}
__device__ __forceinline__ Iv distortIv(const DevCamera& c, Iv r) {
  r = Iv{fmin(c.distMax, r.lo), fmin(c.distMax, r.hi)};  // (distMax < r) ? distMax : r, monotone
  return ivMul(distortFactorIv(c, ivSqr(r)), r);
}

// Camera::sees on the interval w: kSeen (with the pixel row's interval in *py), kNotSeen, or kUndecided
__device__ __forceinline__ int seesIv(const DevCamera& c, const Iv* w, Iv* py) {
  Iv v[3];
  for (int k = 0; k < 3; ++k) v[k] = ivAddPt(w[k], -c.pos[k]);
  const Iv cz = ivDot(c.rot + 6, v);
  if (c.cosFov != -1) {  // isOutsideFov
    if (c.cosFov == 0) {
      if (cz.lo >= 0) return kNotSeen;
      if (!(cz.hi < 0)) return kUndecided;
    } else {
      const Iv dot = ivNeg(cz);  // dot * |dot| is increasing in dot
      const Iv lhs{__dmul_rd(dot.lo, fabs(dot.lo)), __dmul_ru(dot.hi, fabs(dot.hi))};
      const Iv rhs = ivScale(ivAdd(ivAdd(ivSqr(v[0]), ivSqr(v[1])), ivSqr(v[2])), c.cosFov * fabs(c.cosFov));
      if (lhs.hi <= rhs.lo) return kNotSeen;
      if (!(lhs.lo > rhs.hi)) return kUndecided;
    }
  }
  const Iv cx = ivDot(c.rot, v), cy = ivDot(c.rot + 3, v);
  Iv sx, sy;
  if (c.type == DERP_CAM_ORTHOGRAPHIC) {
    if (!(cz.hi < 0)) return kUndecided;  // the cz >= 0 branch is behind the default and every limited fov
    const Iv norm = ivSqrt(ivAdd(ivAdd(ivSqr(cx), ivSqr(cy)), ivSqr(cz)));
    const Iv px = ivDiv(cx, norm), pyy = ivDiv(cy, norm);
    const Iv f = distortFactorIv(c, ivAdd(ivSqr(px), ivSqr(pyy)));
    sx = ivMul(f, px);
    sy = ivMul(f, pyy);
  } else {
    const Iv xy = ivSqrt(ivAdd(ivSqr(cx), ivSqr(cy)));
    if (!(xy.lo > 0)) return kUndecided;  // next to the optical axis (distort(r) / xy may be NaN)
    Iv r;
    if (c.type == DERP_CAM_FTHETA) {
      // atan2(xy, -cz): decreasing in -cz, and monotone in xy for each -cz, so its extremes are at the box's corners;
      // each corner is widened by CUDA's 2 ulp, glibc's budgeted 2 and 1
      const Iv mz = ivNeg(cz);
      double lo = INFINITY, hi = -INFINITY;
      for (int k = 0; k < 4; ++k) {
        const Iv t = widenD(atan2((k & 1) ? xy.hi : xy.lo, (k & 2) ? mz.hi : mz.lo), kAtan2Ulps, 0);
        lo = fmin(lo, t.lo);
        hi = fmax(hi, t.hi);
      }
      r = Iv{lo, hi};
    } else if (c.type == DERP_CAM_RECTILINEAR) {
      const Iv mz = ivNeg(cz);
      if (mz.hi <= 0) {
        r = Iv{16331239353195370.0, 16331239353195370.0};
      } else if (mz.lo > 0) {
        r = ivDiv(xy, mz);
      } else {
        return kUndecided;
      }
    } else {  // EQUISOLID: 2 * sqrt((1 + cz / norm) / 2)
      const Iv norm = ivSqrt(ivAdd(ivAdd(ivSqr(cx), ivSqr(cy)), ivSqr(cz)));
      const Iv h = ivDivPos(ivAddPt(ivDiv(cz, norm), 1.0), 2.0);
      if (!(h.lo >= 0)) return kUndecided;
      r = ivScale(ivSqrt(h), 2.0);
    }
    const Iv f = ivDiv(distortIv(c, r), xy);
    sx = ivMul(f, cx);
    sy = ivMul(f, cy);
  }
  const Iv x = ivAddPt(ivScale(sx, c.focal[0]), c.principal[0]);
  const Iv y = ivAddPt(ivScale(sy, c.focal[1]), c.principal[1]);
  if (!ivOk(x) || !ivOk(y)) return kUndecided;  // NaN: seen by the reference, which the interval cannot show
  if (x.hi < 0 || x.lo >= c.res[0] || y.hi < 0 || y.lo >= c.res[1]) return kNotSeen;
  if (!(x.lo >= 0 && x.hi < c.res[0] && y.lo >= 0 && y.hi < c.res[1])) return kUndecided;
  *py = y;
  return kSeen;
}

// The number of cameras that see the exact point (x, y, z), or -1 when the point goes to the host.  With kTiming, also
// minTimingDiff in *minTiming (as a float, which holds it exactly).
template <bool kTiming>
__device__ __forceinline__ int provenCount(const DevCamera* __restrict__ cams, int n, double x, double y, double z,
                                          float* minTiming) {
  float t[kTiming ? kTimingCap : 1];
  int count = 0;
  for (int i = 0; i < n; ++i) {
    const DevCamera& c = cams[i];
    float ti = 0;
    if (c.type != DERP_CAM_FTHETA) {
      double px, py;
      if (!sees(c, x, y, z, &px, &py)) continue;
      if (kTiming) ti = (float)(py / c.res[1]);
    } else {
      const Iv w[3] = {{x, x}, {y, y}, {z, z}};
      Iv py;
      const int s = seesIv(c, w, &py);
      if (s == kUndecided) return -1;
      if (s == kNotSeen) continue;
      if (kTiming) {  // the host's y / res lies between these quotients, and rounding to float is monotone
        ti = (float)__ddiv_rd(py.lo, c.res[1]);
        if (ti != (float)__ddiv_ru(py.hi, c.res[1])) return -1;
      }
    }
    if (kTiming) {
      if (count == kTimingCap || ti != ti) return -1;
      int k = count;  // insertion into the sorted list
      for (; k > 0 && t[k - 1] > ti; --k) t[k] = t[k - 1];
      t[k] = ti;
    }
    ++count;
  }
  if (kTiming) {
    double m = 1.0;
    for (int k = 0; k + 1 < count; ++k) m = fmin(m, (double)(t[k + 1] - t[k]));
    *minTiming = (float)m;
  }
  return count;
}
#endif

}  // namespace rig
}  // namespace derp
