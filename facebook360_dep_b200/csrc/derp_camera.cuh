// Camera model of the product path (host construction + device projection), fp64.
// Replaces fb360_dep::Camera (source/util/Camera.h:32-378, Camera.cpp:30-242) for the depth path.
// All device arithmetic is written in the reference's operation order and compiled with
// -fmad=false, because the narrowed fp32 source coordinates feed a bit-exact cost.
#pragma once

#include <cmath>
#include <cstdint>

#include "../../include/derp_b200.h"

#if defined(__CUDACC__)
#define DERP_HD __host__ __device__ __forceinline__
#else
#define DERP_HD inline
#endif

namespace derp {

// 16-byte aligned and a multiple of 16 bytes long so that pairs of doubles can move with one 128-bit shared load
struct alignas(16) DevCamera {
  double pos[3];
  double cosFov;        // next to pos: the cone test reads pos, cosFov, rot[6..8]
  double rot[9];        // row-major; rows: right, up, backward (Camera.h:77-85)
  double distMax;
  double principal[2];
  double focal[2];
  double res[2];
  double dist[3];
  double pad0;
  int type;
  int defaultFov;       // cosFov == getDefaultCosFov(type) (Camera.cpp:206-208)
  int zeroDist;         // getDistortion().isZero() (Camera.h:256)
  int reserved[9];      // unused, zero
};
static_assert(sizeof(DevCamera) % 16 == 0, "DevCamera is staged with 128-bit copies");
static_assert(sizeof(DevCamera) == 240, "the size sets the cost kernels' shared memory and so the sweep's CTA height");

// ------------------------------------------------------------------------------------------------
// Host-side construction
// ------------------------------------------------------------------------------------------------
namespace host {

inline double defaultCosFov(int type) {  // Camera.cpp:183-191
  return (type == DERP_CAM_RECTILINEAR || type == DERP_CAM_ORTHOGRAPHIC) ? 0.0 : -1.0;
}

// Eigen: Matrix3 -> Quaternion -> AngleAxis -> Matrix3, what Camera::setRotation uses to
// re-unitarise the JSON rotation (Camera.cpp:77-87).
inline bool reunitarise(const double* fwd, const double* up, const double* right, double* R) {
  const double crx = right[1] * up[2] - right[2] * up[1];
  const double cry = right[2] * up[0] - right[0] * up[2];
  const double crz = right[0] * up[1] - right[1] * up[0];
  if (!(crx * fwd[0] + cry * fwd[1] + crz * fwd[2] < 0)) return false;  // must be right-handed
  double m[9];
  for (int i = 0; i < 3; ++i) {
    m[0 + i] = right[i];
    m[3 + i] = up[i];
    m[6 + i] = -fwd[i];
  }
  for (int i = 0; i < 3; ++i) {  // isUnitary(0.001)
    const double n2 = m[i] * m[i] + m[3 + i] * m[3 + i] + m[6 + i] * m[6 + i];
    if (!(std::fabs(n2 - 1.0) <= 0.001 * (n2 < 1.0 ? n2 : 1.0))) return false;
    for (int j = 0; j < i; ++j)
      if (!(std::fabs(m[i] * m[j] + m[3 + i] * m[3 + j] + m[6 + i] * m[6 + j]) <= 0.001)) return false;
  }
  double qx, qy, qz, qw;
  double t = m[0] + m[4] + m[8];
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    qw = 0.5 * t;
    t = 0.5 / t;
    qx = (m[7] - m[5]) * t;
    qy = (m[2] - m[6]) * t;
    qz = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 4]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double q[3];
    t = std::sqrt(m[i * 4] - m[j * 4] - m[k * 4] + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    qw = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
    qx = q[0];
    qy = q[1];
    qz = q[2];
  }
  double n = std::sqrt(qx * qx + qy * qy + qz * qz);
  double ang = 0, ax = 1, ay = 0, az = 0;
  if (n != 0) {
    ang = 2.0 * std::atan2(n, std::fabs(qw));
    if (qw < 0) n = -n;
    ax = qx / n;
    ay = qy / n;
    az = qz / n;
  }
  const double s = std::sin(ang), c = std::cos(ang);
  const double sx = s * ax, sy = s * ay, sz = s * az;
  const double cx = (1.0 - c) * ax, cy = (1.0 - c) * ay, cz = (1.0 - c) * az;
  double tmp;
  tmp = cx * ay;
  R[1] = tmp - sz;
  R[3] = tmp + sz;
  tmp = cx * az;
  R[2] = tmp + sy;
  R[6] = tmp - sy;
  tmp = cy * az;
  R[5] = tmp - sx;
  R[7] = tmp + sx;
  R[0] = cx * ax + c;
  R[4] = cy * ay + c;
  R[8] = cz * az + c;
  return true;
}

inline double horner(const double* c, int deg, double y) {
  double r = c[deg];
  for (int i = deg - 1; i >= 0; --i) r = r * y + c[i];
  return r;
}

// smallest positive real root of c0 + c1 y + ... (deg <= 3, c0 = 1) — Camera.cpp:131-153.
// Sign-change search over the monotone pieces + bisection to the last ulp.
inline double smallestPositiveRoot(const double* c, int deg) {
  const double inf = INFINITY;
  if (deg == 1) {
    const double r = -c[0] / c[1];
    return r > 0 ? r : inf;
  }
  double brk[3];
  int nb = 0;
  if (deg == 2) {
    const double r = -c[1] / (2 * c[2]);
    if (r > 0) brk[nb++] = r;
  } else {
    const double A = 3 * c[3], B = 2 * c[2], Cc = c[1];
    const double disc = B * B - 4 * A * Cc;
    if (disc >= 0) {
      const double sq = std::sqrt(disc);
      const double q = -0.5 * (B + (B >= 0 ? sq : -sq));
      double r1 = q / A, r2 = (q != 0) ? Cc / q : r1;
      if (r1 > r2) {
        const double t = r1;
        r1 = r2;
        r2 = t;
      }
      if (r1 > 0) brk[nb++] = r1;
      if (r2 > 0 && r2 != r1) brk[nb++] = r2;
    }
  }
  double lo = 0, flo = c[0];
  for (int i = 0; i <= nb; ++i) {
    double hi;
    if (i < nb) {
      hi = brk[i];
    } else {
      if ((c[deg] < 0) == (flo < 0)) return inf;
      hi = (lo > 0 ? lo : 1.0) * 2;
      int guard = 0;
      while ((horner(c, deg, hi) < 0) == (flo < 0) && guard++ < 2000) hi *= 2;
      if (guard >= 2000) return inf;
    }
    const double fhi = horner(c, deg, hi);
    if (fhi == 0 && i < nb) return hi;
    if ((fhi < 0) != (flo < 0)) {
      double a = lo, b = hi, fa = flo;
      for (int it = 0; it < 200; ++it) {
        const double mid = 0.5 * (a + b);
        if (mid == a || mid == b) break;
        const double fm = horner(c, deg, mid);
        if (fm == 0) return mid;
        if ((fm < 0) == (fa < 0)) {
          a = mid;
          fa = fm;
        } else {
          b = mid;
        }
      }
      return 0.5 * (a + b);
    }
    lo = hi;
    flo = fhi;
  }
  return inf;
}

inline bool makeCamera(const DerpCameraDesc& d, DevCamera* out) {
  DevCamera c{};
  if (d.type < 0 || d.type > 3) return false;
  c.type = d.type;
  for (int i = 0; i < 3; ++i) c.pos[i] = d.origin[i];
  if (!reunitarise(d.forward, d.up, d.right, c.rot)) return false;
  for (int i = 0; i < 2; ++i) {
    c.res[i] = d.resolution[i];
    c.principal[i] = d.has_principal ? d.principal[i] : d.resolution[i] / 2;
    c.focal[i] = d.focal[i];
  }
  int count = 3;
  while (count > 0 && d.distortion[count - 1] == 0) --count;
  if (count == 0) {
    c.dist[0] = c.dist[1] = c.dist[2] = 0;
    c.distMax = INFINITY;
  } else {
    double poly[4] = {1, 0, 0, 0};
    for (int i = 0; i < count; ++i) poly[i + 1] = d.distortion[i] * (2 * i + 3);
    for (int i = 0; i < 3; ++i) c.dist[i] = d.distortion[i];
    c.distMax = std::sqrt(smallestPositiveRoot(poly, count));
  }
  c.zeroDist = (c.dist[0] == 0 && c.dist[1] == 0 && c.dist[2] == 0);
  if (d.has_fov) {
    c.cosFov = std::cos(d.fov);
    if (!(c.cosFov >= defaultCosFov(d.type))) return false;  // Camera.cpp:197-200
  } else {
    c.cosFov = defaultCosFov(d.type);
  }
  c.defaultFov = (c.cosFov == defaultCosFov(d.type));
  *out = c;
  return true;
}

inline DevCamera rescaled(const DevCamera& in, double w, double h) {  // Camera.cpp:210-216
  DevCamera c = in;
  const double nr[2] = {w, h};
  for (int i = 0; i < 2; ++i) {
    c.principal[i] *= nr[i] / c.res[i];
    c.focal[i] *= nr[i] / c.res[i];
    c.res[i] = nr[i];
  }
  return c;
}

inline void normalise(DevCamera& c) {  // Camera.cpp:218-222
  for (int i = 0; i < 2; ++i) {
    c.principal[i] = c.principal[i] / c.res[i];
    c.focal[i] = c.focal[i] / c.res[i];
    c.res[i] = 1;
  }
}

}  // namespace host

// ------------------------------------------------------------------------------------------------
// Device-side projection (usable on the host too, for CPU-side unit tests of this code)
// ------------------------------------------------------------------------------------------------
DERP_HD double distortFactor(const DevCamera& c, double r2) {  // Camera.h:225-232
  double result = c.dist[2];
  result = c.dist[1] + r2 * result;
  result = c.dist[0] + r2 * result;
  return 1 + r2 * result;
}

DERP_HD double distort(const DevCamera& c, double r) {  // Camera.h:238-241
  r = (c.distMax < r) ? c.distMax : r;
  return distortFactor(c, r * r) * r;
}

DERP_HD double undistort(const DevCamera& c, double y) {  // Camera.h:243-284
  if (c.zeroDist) return y;
  if (y >= distort(c, c.distMax)) return c.distMax;
  const double smidgen = 1.0 / 1e4;
  double x0 = 0, y0 = 0, dy0 = 1;
  for (int step = 0; step < 10; ++step) {
    const double x1 = (y - y0) / dy0 + x0;
    const double y1 = distort(c, x1);
    if (fabs(y1 - y) < smidgen) return x1;
    const double dy1 = (distort(c, x1 + smidgen) - y1) / smidgen;
    x0 = x1;
    y0 = y1;
    dy0 = dy1;
  }
  return x0;
}

// atan2(y, x) for y >= 0 (y is a norm), result in [0, pi].
// Device version: one division + fdlibm's degree-11 minimax polynomial (|t| <= tan(pi/8) after folding the
// argument with atan(a/b) = pi/4 + atan((a-b)/(a+b))), coefficients as constant-bank operands.  CUDA's
// libdevice atan2 materialises ~25 64-bit immediates with two UMOVs each inside the sweep's inner loop
// (visible in the SASS); this one issues ~45 instructions in total.  Error < 1.5 ulp, i.e. the same
// tolerance class as CUDA-vs-glibc atan2 (the value is narrowed to fp32 pixel coordinates afterwards).
#if defined(__CUDACC__)
static __constant__ double kAtanT[11] = {  // static: one copy per translation unit that includes this header
    3.33333333333329318027e-01,  -1.99999999998764832476e-01, 1.42857142725034663711e-01,
    -1.11111104054623557880e-01, 9.09088713343650656196e-02,  -7.69187620504482999495e-02,
    6.66107313738753120669e-02,  -5.83357013379057348645e-02, 4.97687799461593236017e-02,
    -3.65315727442169155270e-02, 1.62858201153657823623e-02};
#endif
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ double atan2Pos(double y, double x) {
  const double ax = fabs(x);
  const double hi = fmax(ax, y), lo = fmin(ax, y);
  // region 0: lo/hi <= tan(pi/8): t = lo/hi;  region 1: t = (lo-hi)/(lo+hi), atan(lo/hi) = pi/4 + atan(t)
  const bool fold = lo > 0.41421356237309503 * hi;
  const double num = fold ? lo - hi : lo;
  const double den = fold ? lo + hi : hi;
  double t = num / den;
  if (!(den > 0)) t = 0;  // atan2(0, 0) = 0 like the C library (x = +0)
  const double z = t * t, w = z * z;
  const double s1 = z * fma(w, fma(w, fma(w, fma(w, fma(w, kAtanT[10], kAtanT[8]), kAtanT[6]), kAtanT[4]), kAtanT[2]), kAtanT[0]);
  const double s2 = w * fma(w, fma(w, fma(w, fma(w, kAtanT[9], kAtanT[7]), kAtanT[5]), kAtanT[3]), kAtanT[1]);
  double a = t - t * (s1 + s2);                       // atan(t), |t| <= 0.4143
  if (fold) a += 7.85398163397448278999e-01;          // + pi/4
  if (y > ax) a = 1.57079632679489655800e+00 - a;     // atan(y/ax) = pi/2 - atan(ax/y)
  if (x < 0) a = 3.14159265358979311600e+00 - a;      // second quadrant
  return a;
}
#else
inline double atan2Pos(double y, double x) { return atan2(y, x); }
#endif

// Camera.h:301-341. `cam` = rotation * (rig - position).
DERP_HD void cameraToSensor(const DevCamera& c, double cx, double cy, double cz, double* sx, double* sy) {
  if (c.type == DERP_CAM_FTHETA) {
    const double xy = sqrt(cx * cx + cy * cy);
    const double r = atan2Pos(xy, -cz);
    const double f = distort(c, r) / xy;
    *sx = f * cx;
    *sy = f * cy;
  } else if (c.type == DERP_CAM_RECTILINEAR) {
    const double xy = sqrt(cx * cx + cy * cy);
    double r;
    if (-cz <= 0) {
      r = 16331239353195370.0;  // tan(M_PI / 2) in IEEE double
    } else {
      r = xy / -cz;
    }
    const double f = distort(c, r) / xy;
    *sx = f * cx;
    *sy = f * cy;
  } else if (c.type == DERP_CAM_EQUISOLID) {
    const double xy = sqrt(cx * cx + cy * cy);
    const double norm = sqrt(cx * cx + cy * cy + cz * cz);
    const double r = 2 * sqrt((1 + cz / norm) / 2);
    const double f = distort(c, r) / xy;
    *sx = f * cx;
    *sy = f * cy;
  } else {
    double px, py;
    if (cz < 0) {
      const double norm = sqrt(cx * cx + cy * cy + cz * cz);
      px = cx / norm;
      py = cy / norm;
    } else {
      const double n2 = cx * cx + cy * cy;
      if (n2 > 0) {
        const double n = sqrt(n2);
        px = cx / n;
        py = cy / n;
      } else {
        px = cx;
        py = cy;
      }
    }
    const double f = distortFactor(c, px * px + py * py);
    *sx = f * px;
    *sy = f * py;
  }
}

// Camera.h:344-378
DERP_HD void sensorToCamera(const DevCamera& c, double sx, double sy, double* ux, double* uy, double* uz) {
  const double squaredNorm = sx * sx + sy * sy;
  if (squaredNorm == 0) {
    *ux = 0;
    *uy = 0;
    *uz = -1;
    return;
  }
  const double norm = sqrt(squaredNorm);
  const double r = undistort(c, norm);
  double theta;
  if (c.type == DERP_CAM_FTHETA) {
    theta = r;
  } else if (c.type == DERP_CAM_RECTILINEAR) {
    theta = atan(r);
  } else if (c.type == DERP_CAM_EQUISOLID) {
    theta = r <= 2 ? 2 * asin(r / 2) : 3.14159265358979323846;
  } else {
    theta = r <= 1 ? asin(r) : 3.14159265358979323846 / 2;
  }
  const double f = sin(theta) / norm;
  *ux = f * sx;
  *uy = f * sy;
  *uz = -cos(theta);
}

// Ray direction of a pixel in rig space: rotation^T * sensorToCamera((pixel - principal) / focal)
// (Camera.h:131-138).  rig(pixel, depth) = pos + dir * depth (Camera.h:141-143).
DERP_HD void pixelRay(const DevCamera& c, double px, double py, double* dir) {
  const double sx = (px - c.principal[0]) / c.focal[0];
  const double sy = (py - c.principal[1]) / c.focal[1];
  double ux, uy, uz;
  sensorToCamera(c, sx, sy, &ux, &uy, &uz);
  dir[0] = c.rot[0] * ux + c.rot[3] * uy + c.rot[6] * uz;
  dir[1] = c.rot[1] * ux + c.rot[4] * uy + c.rot[7] * uz;
  dir[2] = c.rot[2] * ux + c.rot[5] * uy + c.rot[8] * uz;
}

// Camera::sees (Camera.h:184-190): FOV cone test, projection, sensor bounds.
// Returns pixel coordinates in the camera's own resolution units.
DERP_HD bool sees(const DevCamera& c, double wx, double wy, double wz, double* px, double* py) {
  const double vx = wx - c.pos[0], vy = wy - c.pos[1], vz = wz - c.pos[2];
  const double camz = c.rot[6] * vx + c.rot[7] * vy + c.rot[8] * vz;
  // isOutsideFov (Camera.h:154-164); forward() = -row2, so forward.dot(v) = -camz
  if (c.cosFov != -1) {
    if (c.cosFov == 0) {
      if (camz >= 0) return false;  // isBehind
    } else {
      const double dot = -camz;
      const double n2 = vx * vx + vy * vy + vz * vz;
      if (dot * fabs(dot) <= c.cosFov * fabs(c.cosFov) * n2) return false;
    }
  }
  const double camx = c.rot[0] * vx + c.rot[1] * vy + c.rot[2] * vz;
  const double camy = c.rot[3] * vx + c.rot[4] * vy + c.rot[5] * vz;
  double sx, sy;
  cameraToSensor(c, camx, camy, camz, &sx, &sy);
  const double x = c.focal[0] * sx + c.principal[0];
  const double y = c.focal[1] * sy + c.principal[1];
  *px = x;
  *py = y;
  return !(0 > x || x >= c.res[0] || 0 > y || y >= c.res[1]);  // isOutsideSensor
}

// Camera::isOutsideImageCircle (Camera.h:166-178)
DERP_HD bool outsideImageCircle(const DevCamera& c, double px, double py) {
  if (c.defaultFov) return false;
  const double sinFov = sqrt(1 - c.cosFov * c.cosFov);
  double ex, ey;
  cameraToSensor(c, 0.0, sinFov, -c.cosFov, &ex, &ey);
  const double sx = (px - c.principal[0]) / c.focal[0];
  const double sy = (py - c.principal[1]) / c.focal[1];
  return sx * sx + sy * sy >= ex * ex + ey * ey;
}

}  // namespace derp
