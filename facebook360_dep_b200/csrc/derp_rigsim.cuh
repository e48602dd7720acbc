// RigSimulator's scene, BVH and ray tracer (include/derp_rigsim.h): the host construction, which consumes rand() in the
// reference's order, and the per-ray code shared by the trace kernel and the host (DERP_HD).  Every fp32 expression is
// written in the reference's operation order and element type, with OpenCV 4's matx.hpp rules for cv::Vec:
//   Vec / float      each element times the float 1.f / alpha
//   Vec /= double    each element times the double 1. / alpha, narrowed to float
//   Vec /= float     each element times the float 1.f / alpha
//   norm(Vec3f)      the double sqrt of the sum of squares accumulated in double
//   a.dot(b)         accumulated in float from 0
//   a.cross(b)       (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0) in float
// The library is compiled with -fmad=false, so no product is contracted into an FMA.
#pragma once

#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "derp_camera.cuh"
#include "derp_interval.cuh"
#include "../../include/derp_rigsim.h"

namespace derp {
namespace rigsim {

constexpr int kTraceThreadsX = 32, kTraceThreadsY = 4;
constexpr double kPi = 3.14159265358979323846;  // M_PI

// ---- fp32 vector arithmetic in matx.hpp's order -------------------------------------------------------------------
struct V3 {
  float x, y, z;
};
DERP_HD V3 v3(float x, float y, float z) { return V3{x, y, z}; }
DERP_HD V3 v3(const float* p) { return V3{p[0], p[1], p[2]}; }
DERP_HD V3 add(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
DERP_HD V3 sub(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
DERP_HD V3 mul(V3 a, float s) { return V3{a.x * s, a.y * s, a.z * s}; }
DERP_HD float dot(V3 a, V3 b) {
  float s = 0;
  s += a.x * b.x;
  s += a.y * b.y;
  s += a.z * b.z;
  return s;
}
DERP_HD V3 cross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
DERP_HD double norm(V3 a) {
  double s = 0;
  s += (double)a.x * (double)a.x;
  s += (double)a.y * (double)a.y;
  s += (double)a.z * (double)a.z;
  return sqrt(s);
}
DERP_HD V3 divD(V3 a, double alpha) {  // Vec /= double
  const double ia = 1. / alpha;
  return V3{(float)(a.x * ia), (float)(a.y * ia), (float)(a.z * ia)};
}

// ---- Ken Perlin's improved noise (PerlinNoise.h, after mrl.nyu.edu/~perlin/noise/) -------------------------------
// The permutation of Perlin's reference implementation; the reference repeats it to 512 entries, indexed below 512.
#define DERP_PERLIN_PERMUTATION                                                                                       \
  151, 160, 137, 91, 90, 15, 131, 13, 201, 95, 96, 53, 194, 233, 7, 225, 140, 36, 103, 30, 69, 142, 8, 99, 37, 240,   \
      21, 10, 23, 190, 6, 148, 247, 120, 234, 75, 0, 26, 197, 62, 94, 252, 219, 203, 117, 35, 11, 32, 57, 177, 33,     \
      88, 237, 149, 56, 87, 174, 20, 125, 136, 171, 168, 68, 175, 74, 165, 71, 134, 139, 48, 27, 166, 77, 146, 158,   \
      231, 83, 111, 229, 122, 60, 211, 133, 230, 220, 105, 92, 41, 55, 46, 245, 40, 244, 102, 143, 54, 65, 25, 63,    \
      161, 1, 216, 80, 73, 209, 76, 132, 187, 208, 89, 18, 169, 200, 196, 135, 130, 116, 188, 159, 86, 164, 100, 109,  \
      198, 173, 186, 3, 64, 52, 217, 226, 250, 124, 123, 5, 202, 38, 147, 118, 126, 255, 82, 85, 212, 207, 206, 59,    \
      227, 47, 16, 58, 17, 182, 189, 28, 42, 223, 183, 170, 213, 119, 248, 152, 2, 44, 154, 163, 70, 221, 153, 101,   \
      155, 167, 43, 172, 9, 129, 22, 39, 253, 19, 98, 108, 110, 79, 113, 224, 232, 178, 185, 112, 104, 218, 246, 97,   \
      228, 251, 34, 242, 193, 238, 210, 144, 12, 191, 179, 162, 241, 81, 51, 145, 235, 249, 14, 239, 107, 49, 192,    \
      214, 31, 181, 199, 106, 157, 184, 84, 204, 176, 115, 121, 50, 45, 127, 4, 150, 254, 138, 236, 205, 93, 222, 114, \
      67, 29, 24, 72, 243, 141, 128, 195, 78, 66, 215, 61, 156, 180
#if defined(__CUDACC__)
__constant__ unsigned char kPermDev[256] = {DERP_PERLIN_PERMUTATION};
#endif
static const unsigned char kPermHost[256] = {DERP_PERLIN_PERMUTATION};
#undef DERP_PERLIN_PERMUTATION

DERP_HD int perm(int i) {
#if defined(__CUDA_ARCH__)
  return kPermDev[i & 255];
#else
  return kPermHost[i & 255];
#endif
}
DERP_HD float fade(float t) { return t * t * t * (t * (t * 6 - 15) + 10); }
DERP_HD float lerp(float t, float a, float b) { return a + t * (b - a); }
DERP_HD float grad(int hash, float x, float y, float z) {
  const int h = hash & 15;
  const float u = h < 8 ? x : y;
  const float v = h < 4 ? y : h == 12 || h == 14 ? x : z;
  return ((h & 1) == 0 ? u : -u) + ((h & 2) == 0 ? v : -v);
}
// floor of a float is exact in either overload, and x - floor(x) is exact in float
DERP_HD float pnoise(float x, float y, float z) {
  const int X = (int)floorf(x) & 255, Y = (int)floorf(y) & 255, Z = (int)floorf(z) & 255;
  x -= floorf(x);
  y -= floorf(y);
  z -= floorf(z);
  const float u = fade(x), v = fade(y), w = fade(z);
  const int A = perm(X) + Y, AA = perm(A) + Z, AB = perm(A + 1) + Z;
  const int B = perm(X + 1) + Y, BA = perm(B) + Z, BB = perm(B + 1) + Z;
  return lerp(w,
              lerp(v, lerp(u, grad(perm(AA), x, y, z), grad(perm(BA), x - 1, y, z)),
                   lerp(u, grad(perm(AB), x, y - 1, z), grad(perm(BB), x - 1, y - 1, z))),
              lerp(v, lerp(u, grad(perm(AA + 1), x, y, z - 1), grad(perm(BA + 1), x - 1, y, z - 1)),
                   lerp(u, grad(perm(AB + 1), x, y - 1, z - 1), grad(perm(BB + 1), x - 1, y - 1, z - 1))));
}

// ---- the scene as the trace reads it ------------------------------------------------------------------------------
struct SceneView {
  const DerpRigsimNode* nodes;
  const int* leafTris;
  const DerpRigsimTriangle* tris;
  const uint8_t* sky;  // BGR
  int skyW, skyH;
  const uint8_t* ceil;  // BGR, NULL: no ceiling
  int ceilW, ceilH;
  double ceilPos, ceilWidth, ceilDepth;
  int marble;
  double marbleScale;
};

// rayIntersectSphereYesNo (RaytracingPrimitives.h:89-109).  A sphere with a NaN centre (an empty cluster) misses.
DERP_HD bool hitSphere(V3 o, V3 d, const DerpRigsimNode& n) {
  const V3 r = sub(v3(n.center), o);
  const float l2 = r.x * r.x + r.y * r.y + r.z * r.z;
  if (l2 < n.radius * n.radius) return true;
  const float ca = dot(r, d);
  if (ca < 0.0f) return false;
  const float h = n.radius * n.radius + ca * ca - l2;
  return h >= 0.0f;
}

// rayIntersectTriangle (RaytracingPrimitives.h:58-85): the distance of a hit, or false
DERP_HD bool hitTriangle(V3 o, V3 d, const DerpRigsimTriangle& t, float* dist) {
  const V3 e1 = v3(t.e1), e2 = v3(t.e2);
  const V3 q = cross(d, e2);
  const float a = dot(e1, q);
  if (a * a < 0.0001f) return false;
  const V3 s = mul(sub(o, v3(t.v0)), 1.f / a);
  const V3 r = cross(s, e1);
  const float b0 = dot(s, q);
  const float b1 = dot(r, d);
  const float b2 = 1.0f - b0 - b1;
  if (b0 < 0.0f || b1 < 0.0f || b2 < 0.0f) return false;
  const float dd = dot(e2, r);
  if (dd < 0.0f) return false;
  *dist = dd;
  return true;
}

// raytraceBVH (RigSimulator.cpp:169-193) without a stack: the recursion visits every child whose sphere is hit, in
// order, and keeps a hit only when it is strictly closer, so its result is the first minimum in preorder over the leaf
// triangles of the visited leaves; the walk below visits the same leaves in the same order.  Returns the scene index
// of the hit triangle or -1, with its distance in *dist (FLT_MAX on a miss).
DERP_HD int closestHit(const SceneView& s, V3 o, V3 d, float* dist) {
  float best = FLT_MAX;
  int idx = -1;
  int k = 0;
  const int end = s.nodes[0].escape;
  while (k < end) {
    const DerpRigsimNode& n = s.nodes[k];
    if (!hitSphere(o, d, n)) {
      k = n.escape;
      continue;
    }
    for (int i = 0; i < n.count; ++i) {
      const int t = s.leafTris[n.first + i];
      float dd;
      if (hitTriangle(o, d, s.tris[t], &dd) && dd < best) {
        best = dd;
        idx = t;
      }
    }
    ++k;
  }
  *dist = best;
  return idx;
}

// The sky texel of a direction (RigSimulator.cpp:224-231) from given acosf and atan2f values:
//   phi = acosf(clamp(dz, -1, 1)); theta = float(M_PI + atan2f(dy, dx));
//   sampleX = float((theta / (2 M_PI)) * cols); sampleY = float((phi / M_PI) * rows)   (double, narrowed to float)
//   row = min(int(sampleY), rows - 1); col = int(sampleX) % cols
// The narrowing matters: a double just below an integer can round up to it.  *row and *colInt (the column before the
// modulo) are non-decreasing in the two function values (theta may be a little below 0: atan2f's float -pi is below
// -M_PI; int() truncates it to column 0).  A sample outside int's range (a NaN direction, which no camera or equirect
// ray has) gives texel (0, 0); the reference's conversion to int is undefined there.
DERP_HD bool skyTexelOf(float phi, float atn, int rows, int cols, int* row, int* colInt) {
  const float theta = (float)(kPi + (double)atn);
  const float sx = (float)(((double)theta / (2.0 * kPi)) * cols);
  const float sy = (float)(((double)phi / kPi) * rows);
  if (!(sx > -2147483648.0f && sx < 2147483648.0f && sy > -2147483648.0f && sy < 2147483648.0f)) {
    *row = 0;
    *colInt = 0;
    return false;
  }
  *row = (int)sy < rows - 1 ? (int)sy : rows - 1;
  *colInt = (int)sx;
  return true;
}

inline void skyTexelHost(V3 d, int rows, int cols, int* row, int* col) {
  const float z = d.z < -1.0f ? -1.0f : d.z > 1.0f ? 1.0f : d.z;
  skyTexelOf(acosf(z), atan2f(d.y, d.x), rows, cols, row, col);
  *col %= cols;
}

#if defined(__CUDACC__)
// The device's acosf and atan2f are within 2 and 3 ulp of the exact value (CUDA C++ Programming Guide, "Mathematical
// Functions", single precision) and glibc's within the 2 derp_interval.cuh budgets.  Those are ulps of the exact value,
// so the C library's value lies in widenF of the device's with kAcosfUlps / kAtan2fUlps, a relative bound plus 1 ulp.
// (Counting float steps from the device's value would not do: just above a power of two, 2 ulp below the exact value
// are 4 steps.)  The texel is decided when both ends of the widened intervals give the same row and column before the
// modulo (then every value between does, the chain being monotone); false otherwise
__device__ __forceinline__ bool skyTexelDevice(V3 d, int rows, int cols, int* row, int* col) {
  const float z = d.z < -1.0f ? -1.0f : d.z > 1.0f ? 1.0f : d.z;
  const Iv p = ivFloat(widenF(acosf(z), kAcosfUlps)), a = ivFloat(widenF(atan2f(d.y, d.x), kAtan2fUlps));
  int r0, c0, r1, c1;
  if (!skyTexelOf((float)p.lo, (float)a.lo, rows, cols, &r0, &c0) ||
      !skyTexelOf((float)p.hi, (float)a.hi, rows, cols, &r1, &c1) || r0 != r1 || c0 != c1)
    return false;
  *row = r0;
  *col = c0 % cols;
  return true;
}
#endif

// traceRayToGetColor (RigSimulator.cpp:196-262) up to the sky texel: B, G, R (0..1) and depth.  Returns false when
// nothing but the sky is hit; the caller then finds the texel (skyTexelHost / skyTexelDevice) and calls skyColor.
DERP_HD bool traceRay(const SceneView& s, V3 o, V3 d, float* out) {
  float dist;
  const int hit = closestHit(s, o, d, &dist);
  if (s.ceil) {
    // the ceiling plane: (double - float) / float in double, narrowed; s and t in double, narrowed
    const float depth = (float)((s.ceilPos - o.z) / d.z);
    if (0 < depth && depth < dist) {
      const V3 p = add(o, mul(d, depth));
      const float cs = (float)(p.x / s.ceilWidth + 0.5);
      const float ct = (float)(p.y / s.ceilDepth + 0.5);
      if (0 <= cs && cs < 1 && 0 <= ct && ct < 1) {
        const uint8_t* c = s.ceil + ((size_t)(int)(ct * s.ceilH) * s.ceilW + (int)(cs * s.ceilW)) * 3;
        out[0] = (float)c[0] / 255;
        out[1] = (float)c[1] / 255;
        out[2] = (float)c[2] / 255;
        out[3] = depth;
        return true;
      }
    }
  }
  if (hit < 0) return false;
  const DerpRigsimTriangle& t = s.tris[hit];
  V3 base = v3(t.color);
  const V3 p = add(o, mul(d, dist));
  if (s.marble) {
    // FLAGS_marble_scale * float in double, narrowed to pnoise's float parameters
    const float f = 0.7f + 0.3f * fabsf(pnoise((float)(s.marbleScale * p.x), (float)(s.marbleScale * p.y),
                                               (float)(s.marbleScale * p.z)));
    base = mul(base, f);
  }
  V3 light = sub(v3(2.0f, 1.0f, 5.2f), p);  // kLightPos
  light = divD(light, norm(light));
  const float dl = dot(v3(t.normal), light);
  const float coef = .25f + .75f * (0.0f < dl ? dl : 0.0f);  // std::max(0.0f, dl)
  out[0] = base.x * coef;
  out[1] = base.y * coef;
  out[2] = base.z * coef;
  out[3] = dist;
  return true;
}

DERP_HD void skyColor(const SceneView& s, int row, int col, float* out) {
  const uint8_t* c = s.sky + ((size_t)row * s.skyW + col) * 3;
  out[0] = c[0] / 255.0f;
  out[1] = c[1] / 255.0f;
  out[2] = c[2] / 255.0f;
  out[3] = FLT_MAX;
}

// ---- host construction ----------------------------------------------------------------------------------------------
namespace host {

inline float randf0to1() { return float(rand()) / float(RAND_MAX); }  // MathUtil.h:23-25

// Triangle's constructor (RaytracingPrimitives.h:45-49)
inline DerpRigsimTriangle makeTriangle(V3 a, V3 b, V3 c, V3 color) {
  DerpRigsimTriangle t;
  const V3 e1 = sub(b, a), e2 = sub(c, a);
  const V3 n = divD(cross(e1, e2), norm(cross(e1, e2)));
  const V3* src[7] = {&a, &b, &c, &e1, &e2, &n, &color};
  float* dst[7] = {t.v0, t.v1, t.v2, t.e1, t.e2, t.normal, t.color};
  for (int i = 0; i < 7; ++i) {
    dst[i][0] = src[i]->x;
    dst[i][1] = src[i]->y;
    dst[i][2] = src[i]->z;
  }
  return t;
}

// The unit icosahedron: 12 vertices (+-X, 0, +-Z) cycled through the axes, X = 1 / sqrt(phi sqrt 5) and
// Z = phi X (phi the golden ratio), as float; and its 20 faces
constexpr float kIcoX = 0.525731112119133696f, kIcoZ = 0.850650808352039932f;
static const float kIcoVertex[12][3] = {
    {-kIcoX, 0, kIcoZ}, {kIcoX, 0, kIcoZ}, {-kIcoX, 0, -kIcoZ}, {kIcoX, 0, -kIcoZ}, {0, kIcoZ, kIcoX}, {0, kIcoZ, -kIcoX},
    {0, -kIcoZ, kIcoX}, {0, -kIcoZ, -kIcoX}, {kIcoZ, kIcoX, 0}, {-kIcoZ, kIcoX, 0}, {kIcoZ, -kIcoX, 0}, {-kIcoZ, -kIcoX, 0}};
static const int kIcoFace[20][3] = {{1, 4, 0},  {4, 9, 0},  {4, 5, 9},  {8, 5, 4},  {1, 8, 4},  {1, 10, 8}, {10, 3, 8},
                                    {8, 3, 5},  {3, 2, 5},  {3, 7, 2},  {3, 10, 7}, {10, 6, 7}, {6, 11, 7}, {6, 0, 11},
                                    {6, 1, 0},  {10, 1, 6}, {11, 0, 9}, {2, 11, 9}, {5, 2, 9},  {11, 2, 7}};

// Three randf0to1() calls in one cv::Vec3f(...) constructor: C++ leaves their order unspecified; g++ (x86_64), which
// builds the reference, evaluates the arguments last to first, so z is drawn first and x last.  The checker test of
// the scene pins this order against the reference's own object.
inline V3 randVec3(float (*f)()) {
  const float z = f(), y = f(), x = f();
  return v3(x, y, z);
}

inline void makeIcosahedron(std::vector<DerpRigsimTriangle>& tris, V3 center, float radius) {  // RigSimulator.cpp:145-167
  const V3 color = center.z > 0 ? v3(0, 1, 0) : randVec3(randf0to1);
  for (int i = 0; i < 20; ++i) {
    V3 v[3];
    for (int k = 0; k < 3; ++k) v[k] = add(mul(v3(kIcoVertex[kIcoFace[i][k]]), radius), center);
    tris.push_back(makeTriangle(v[0], v[1], v[2], color));
  }
}

inline void makeIcosahedronScene(const DerpRigsimSceneParams& p, std::vector<DerpRigsimTriangle>& tris) {
  for (int i = 0; i < p.num_random_icosahedrons; ++i) {  // RigSimulator.cpp:264-289
    const float minAllowed = (float)(p.min_icosahedron_dist + p.max_icosahedron_radius);
    V3 center;
    do {
      // 2.0f * (randf0to1() - 0.5) * max_dist in double, narrowed by the constructor; drawn z, y, x (see randVec3)
      double c[3];
      for (int k = 2; k >= 0; --k) c[k] = 2.0f * (randf0to1() - 0.5) * p.max_icosahedron_dist;
      center = v3((float)c[0], (float)c[1], (float)c[2]);
    } while (norm(center) < minAllowed);
    const float range = (float)(p.max_icosahedron_radius - p.min_icosahedron_radius);
    const float radius = (float)(p.min_icosahedron_radius + randf0to1() * range);
    makeIcosahedron(tris, center, radius);
  }
  if (p.red_triangle) {
    const float depth = (float)p.min_icosahedron_dist, side = 0.1f * depth;
    tris.push_back(makeTriangle(v3(depth, 0, 0), v3(depth, 0, side), v3(depth, side, 0), v3(0, 0, 1)));
  }
}

// Two cubes, the first of side 2 centred 25 m down -z, the second of side 1 at (5, 2, -20); each face pair has its
// colour (B, G, R)  (RigSimulator.cpp:291-343)
inline void makeCubesScene(std::vector<DerpRigsimTriangle>& tris) {
  static const float kVertex[8][3] = {{0, 0, 0}, {0, 0, 1}, {0, 1, 0}, {0, 1, 1},
                                      {1, 0, 0}, {1, 0, 1}, {1, 1, 0}, {1, 1, 1}};
  static const int kFace[12][3] = {{2, 0, 1}, {1, 3, 2}, {6, 2, 0}, {0, 4, 6}, {4, 0, 1}, {1, 5, 4},
                                   {3, 1, 5}, {5, 7, 3}, {7, 3, 2}, {2, 6, 7}, {5, 4, 6}, {6, 7, 5}};
  static const float kScale[2] = {2, 1};
  static const float kOffset[2][3] = {{0, 0, -25}, {5, 2, -20}};
  static const float kColor[2][6][3] = {
      {{0, 0, 1}, {0, 1, 0}, {0, 1, 1}, {1, 0, 0}, {1, 0, 1}, {1, 1, 0}},            // red green yellow blue magenta cyan
      {{0.5f, 1, 0}, {1, 0, 0.5f}, {1, 1, 1}, {0, 0.5f, 1}, {0.5f, 0.5f, 1}, {0, 0, 0}}};  // teal purple white orange salmon black
  const V3 shift = v3(-0.5f, -0.5f, -0.5f);
  for (int f = 0; f < 12; ++f)
    for (int c = 0; c < 2; ++c) {
      V3 v[3];
      for (int k = 0; k < 3; ++k) v[k] = add(mul(add(v3(kVertex[kFace[f][k]]), shift), kScale[c]), v3(kOffset[c]));
      tris.push_back(makeTriangle(v[0], v[1], v[2], v3(kColor[c][f / 2])));
    }
}

inline void makeGroundPlaneScene(const DerpRigsimSceneParams& p, std::vector<DerpRigsimTriangle>& tris) {
  const float r = 100.0f, z = (float)-p.ground_plane_dist_m;  // RigSimulator.cpp:345-358
  const V3 v[4] = {v3(-r, -r, z), v3(r, -r, z), v3(r, r, z), v3(-r, r, z)};
  tris.push_back(makeTriangle(v[0], v[1], v[2], v3(0, 0, 1)));
  tris.push_back(makeTriangle(v[3], v[0], v[2], v3(0, 0, 1)));
}

// BoundingVolumeHierarchy::makeBVH (BoundingVolumeHierarchy.h:32-112) over the scene indices `idx`, appended in
// preorder
inline void makeBVH(const std::vector<DerpRigsimTriangle>& all, const std::vector<int>& idx, int leafSize, int splitK,
                    int depth, int maxDepth, std::vector<DerpRigsimNode>& nodes, std::vector<int>& leafTris) {
  V3 cm = v3(0.0f, 0.0f, 0.0f);
  for (int i : idx) cm = add(cm, add(add(v3(all[i].v0), v3(all[i].v1)), v3(all[i].v2)));
  const float ia = 1.f / float(idx.size() * 3);  // Vec /= float; 1 / 0 = inf: an empty cluster's centre is NaN
  cm = v3(cm.x * ia, cm.y * ia, cm.z * ia);
  float radius = 0.0f;
  for (int i : idx)
    for (const float* v : {all[i].v0, all[i].v1, all[i].v2}) {
      const float d = float(norm(sub(cm, v3(v))));
      radius = radius < d ? d : radius;  // std::max
    }
  const size_t me = nodes.size();
  nodes.push_back(DerpRigsimNode{{cm.x, cm.y, cm.z}, radius, (int)leafTris.size(), 0, -1, 0});
  const int n = (int)idx.size();
  if (depth >= maxDepth || n < splitK || n < leafSize) {
    nodes[me].count = n;
    leafTris.insert(leafTris.end(), idx.begin(), idx.end());
    nodes[me].escape = (int)nodes.size();
    return;
  }
  std::vector<int> centers;
  while ((int)centers.size() < splitK) {
    const int r = (int)(rand() % (size_t)n);
    bool seen = false;
    for (int c : centers) seen |= c == r;
    if (!seen) centers.push_back(r);
  }
  std::vector<std::vector<int>> cluster(splitK);
  for (int i = 0; i < n; ++i) {
    float minDist = FLT_MAX;
    int assigned = 0;
    for (int j = 0; j < splitK; ++j) {
      const V3 diff = sub(v3(all[idx[i]].v0), v3(all[idx[centers[j]]].v0));
      const float d2 = diff.x * diff.x + diff.y * diff.y + diff.z * diff.z;
      if (d2 < minDist) {
        minDist = d2;
        assigned = j;
      }
    }
    cluster[assigned].push_back(idx[i]);
  }
  for (int j = 0; j < splitK; ++j) makeBVH(all, cluster[j], leafSize, splitK, depth + 1, maxDepth, nodes, leafTris);
  nodes[me].escape = (int)nodes.size();
}

}  // namespace host
}  // namespace rigsim
}  // namespace derp
