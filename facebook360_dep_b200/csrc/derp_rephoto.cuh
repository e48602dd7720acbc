// CanopyScene (source/render/CanopyScene.cpp) without GL, for rephotography (ComputeRephotographyErrors: cubemap,
// ipd = 0, alphaBlend = true, the on-screen fragment shader canopyFS) and the exporter (SimpleMeshRenderer: cubemap,
// equirect and perspective views, stereo eye offsets, blending on or off, the off-screen shader canopyFS_SVD), and the
// SSIM / NCC score of source/render/RephotographyUtil.h.
//
// ABI: include/derp_rephoto.h, include/derp_canopy.h; CPU checkers: tests/rephoto_oracle.cpp (rephotography) and
// tests/canopy_oracle.cpp (every canopy mode, built on the former).
// There is no GL here, so the rasteriser follows documented rules (DESIGN.md §4, K19; INTEGRATION.md):
//   - vertices: camera.rig({x + .5, y + .5}, 1.0f / disparity) at the disparity's (mesh) size, fp64 -> fp32
//     (disparityMesh); with ipd != 0, canopyVS' eye offset is subtracted per vertex in rig space (eyeOffset below);
//     primitives are the triangles of stripify's strip in draw order, prim = ((y * (mw - 1) + x) * 2 + k);
//     texVar = (1 / mw, 1 / mh) * (x + .5, y + .5) (Canopy::scale is 1 / mesh size); a triangle with a non-finite vertex
//     is dropped.
//   - views: any number, each with its own fp32 clip matrix and a W x H viewport.  clip = M * (pos, 1) with M =
//     projection * view as Eigen forms it in fp32 on the host (cube faces: all entries 0, +-1, +-p or -p - 0.2, so M is
//     exact); polygons are clipped against the near plane z >= -w only (the far plane is at infinity, side planes are
//     handled by the viewport bounding box).
//   - window coordinates in fp32; edge functions in fp64 over them; a pixel centre on an edge belongs to the triangle
//     whose oriented edge (interior on the left, y up) points down, or left when horizontal (top-left rule).
//   - depth: window z interpolated linearly in screen space, clamped to [0, 1]; GL_LEQUAL in draw order = least depth,
//     ties to the later primitive.  A fragment whose sampled alpha is 0 is discarded before the depth test.
//   - texVar: perspective-correct; dFdx / dFdy are fine derivatives over the pixel's 2x2 quad (quads at even window
//     coordinates), the helper pixels evaluating the same triangle's interpolant.
//   - texture: GL_RGBA16 (round(clamp(v, 0, 1) * 65535)) at its own size, alpha from alphaFov at that size; mips by a
//     2x2 box on the stored integers (odd edges drop their last row / column), GL_REPEAT, GL_LINEAR_MIPMAP_LINEAR with
//     the isotropic LOD of the GL spec §8.14 (no anisotropic filtering) at the sampled texture's size; log2 by a fixed
//     series so that the CPU checker computes the same level.
//   - alpha: canopyFS multiplies by the minor axis, canopyFS_SVD by sigma2 / sigma1 (svdRatio: its rule for degenerate
//     Jacobians), both by the cone.
//   - blend: with alphaBlend, w = exp(30 a) - 1 (expm1 in fp64 by a fixed series, rounded to fp32), else w = a;
//     rgb += w * rgb, a += w in camera order (fp32), then rgba / a; rephotography sets NaN to 0 (zeroOutNans), the
//     exporter keeps it (NaN alpha = no canopy, the background shows).
//   - equirect: equirectFS over the cubemap, GL_LINEAR at level 0, seamless (canopyEquirectKernel).
#pragma once

#include <cstdint>

#include "derp_camera.cuh"
#include "host/smr_host.h"

namespace derp {
namespace rephoto {

constexpr int kMaxLevels = 16;
constexpr int kFaces = 6;

struct FaceMats {
  float m[kFaces][16];  // row-major clip = M * (x, y, z, 1)
};

struct Canopy {
  const float* vtx;                 // mw * mh * 3 rig-space vertices
  const ushort4* tex[2];            // colour / disparity mip chains (B, G, R, A) of one size; either may be null
  int mw, mh;                       // mesh size (Canopy::modulo, Canopy::scale = 1 / size)
  int levels;
  int lw[kMaxLevels], lh[kMaxLevels];  // texture level sizes; level 0 scales the LOD
  long long lofs[kMaxLevels];       // texel offset of each level
  int anyZeroAlpha;                 // 0 when no texel of level 0 has alpha 0: the alpha test cannot discard
  int svd;                          // 1: canopyFS_SVD (exporter), 0: canopyFS (on screen, rephotography)
  int alphaBlend;                   // accumulateFS' alphaBlend
};

struct Tri {
  float x[3], y[3], z[3];     // window coordinates
  float q[3], uq[3], vq[3];   // 1 / w_clip and texVar / w_clip
  double area;                // signed, fp64 over the fp32 coordinates
};

struct ClipV {
  float x, y, z, w, u, v;
};

DERP_HD ClipV toClip(const float* M, float px, float py, float pz, float u, float v) {
  ClipV c;
  c.x = ((M[0] * px + M[1] * py) + M[2] * pz) + M[3];
  c.y = ((M[4] * px + M[5] * py) + M[6] * pz) + M[7];
  c.z = ((M[8] * px + M[9] * py) + M[10] * pz) + M[11];
  c.w = ((M[12] * px + M[13] * py) + M[14] * pz) + M[15];
  c.u = u;
  c.v = v;
  return c;
}

DERP_HD ClipV lerpClip(const ClipV& a, const ClipV& b, float t) {
  ClipV r;
  r.x = a.x + t * (b.x - a.x);
  r.y = a.y + t * (b.y - a.y);
  r.z = a.z + t * (b.z - a.z);
  r.w = a.w + t * (b.w - a.w);
  r.u = a.u + t * (b.u - a.u);
  r.v = a.v + t * (b.v - a.v);
  return r;
}

DERP_HD bool finite3(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

// Triangle `prim` of canopy `cv` on the face with matrix M, clipped to the near plane: 0, 1 or 2 screen triangles.
DERP_HD int setupPrim(const Canopy& cv, const float* M, int W, int H, int prim, Tri* out) {
  const int k = prim & 1, cell = prim >> 1;
  const int mw = cv.mw;
  const int cx = cell % (mw - 1), cy = cell / (mw - 1);
  // strip order: (t_x, b_x, t_x+1), (b_x, t_x+1, b_x+1)
  int id[3];
  if (k == 0) {
    id[0] = cy * mw + cx;
    id[1] = (cy + 1) * mw + cx;
    id[2] = cy * mw + cx + 1;
  } else {
    id[0] = (cy + 1) * mw + cx;
    id[1] = cy * mw + cx + 1;
    id[2] = (cy + 1) * mw + cx + 1;
  }
  const float sx = (float)(1.0 / mw), sy = (float)(1.0 / cv.mh);  // Canopy::scale (Vector2f of 1.0 / cols, rows)
  ClipV v[3];
  for (int i = 0; i < 3; ++i) {
    const float* p = cv.vtx + 3 * (size_t)id[i];
    if (!finite3(p[0], p[1], p[2])) return 0;
    const float u = sx * ((float)(id[i] % mw) + 0.5f), t = sy * ((float)(id[i] / mw) + 0.5f);
    v[i] = toClip(M, p[0], p[1], p[2], u, t);
  }
  // trivial rejects against the side planes (exact: nothing of such a triangle lies in the viewport)
  if (v[0].x > v[0].w && v[1].x > v[1].w && v[2].x > v[2].w) return 0;
  if (v[0].x < -v[0].w && v[1].x < -v[1].w && v[2].x < -v[2].w) return 0;
  if (v[0].y > v[0].w && v[1].y > v[1].w && v[2].y > v[2].w) return 0;
  if (v[0].y < -v[0].w && v[1].y < -v[1].w && v[2].y < -v[2].w) return 0;
  // near plane z >= -w (Sutherland-Hodgman; the intersection is interpolated from the inside vertex)
  ClipV poly[4];
  int n = 0;
  for (int i = 0; i < 3; ++i) {
    const ClipV& a = v[i];
    const ClipV& b = v[(i + 1) % 3];
    const float da = a.z + a.w, db = b.z + b.w;
    const bool ina = da >= 0, inb = db >= 0;
    if (ina) poly[n++] = a;
    if (ina != inb) poly[n++] = ina ? lerpClip(a, b, da / (da - db)) : lerpClip(b, a, db / (db - da));
  }
  if (n < 3) return 0;
  const float halfW = 0.5f * (float)W, halfH = 0.5f * (float)H;
  float X[4], Y[4], Z[4], Q[4], U[4], V[4];
  for (int i = 0; i < n; ++i) {
    const float iw = 1.0f / poly[i].w;
    X[i] = (poly[i].x / poly[i].w) * halfW + halfW;
    Y[i] = (poly[i].y / poly[i].w) * halfH + halfH;
    Z[i] = (poly[i].z / poly[i].w) * 0.5f + 0.5f;
    Q[i] = iw;
    U[i] = poly[i].u * iw;
    V[i] = poly[i].v * iw;
  }
  int m = 0;
  for (int f = 1; f + 1 < n; ++f) {  // fan around poly[0]
    const int idx[3] = {0, f, f + 1};
    Tri& t = out[m];
    for (int j = 0; j < 3; ++j) {
      t.x[j] = X[idx[j]];
      t.y[j] = Y[idx[j]];
      t.z[j] = Z[idx[j]];
      t.q[j] = Q[idx[j]];
      t.uq[j] = U[idx[j]];
      t.vq[j] = V[idx[j]];
    }
    const double x0 = t.x[0], y0 = t.y[0];
    t.area = ((double)t.x[1] - x0) * ((double)t.y[2] - y0) - ((double)t.x[2] - x0) * ((double)t.y[1] - y0);
    if (t.area != 0 && t.area == t.area) ++m;
  }
  return m;
}

// Barycentric weights of (px, py); returns whether the point is covered under the top-left rule.
DERP_HD bool bary(const Tri& t, double px, double py, double* l) {
  const double s = t.area > 0 ? 1.0 : -1.0;
  const double area = t.area * s;
  bool in = true;
  for (int i = 0; i < 3; ++i) {
    const int a = (i + 1) % 3, b = (i + 2) % 3;
    const double xa = t.x[a], ya = t.y[a];
    const double dx = (double)t.x[b] - xa, dy = (double)t.y[b] - ya;
    const double e = (dx * (py - ya) - dy * (px - xa)) * s;
    if (!(e > 0 || (e == 0 && (dy * s < 0 || (dy == 0 && dx * s < 0))))) in = false;
    l[i] = e / area;
  }
  return in;
}

DERP_HD void texVarAt(const Tri& t, const double* l, float* u, float* v) {
  const double iw = (l[0] * t.q[0] + l[1] * t.q[1]) + l[2] * t.q[2];
  *u = (float)(((l[0] * t.uq[0] + l[1] * t.uq[1]) + l[2] * t.uq[2]) / iw);
  *v = (float)(((l[0] * t.vq[0] + l[1] * t.vq[1]) + l[2] * t.vq[2]) / iw);
}

// log2 by frexp and the atanh series (|z| <= 1/3, 8 terms): the same value on the device and in the CPU checker
DERP_HD double log2Series(double x) {
  int e;
  const double m = frexp(x, &e);  // [0.5, 1)
  const double z = (m - 1.0) / (m + 1.0), z2 = z * z;
  double s = 1.0 / 15.0;
  s = s * z2 + 1.0 / 13.0;
  s = s * z2 + 1.0 / 11.0;
  s = s * z2 + 1.0 / 9.0;
  s = s * z2 + 1.0 / 7.0;
  s = s * z2 + 1.0 / 5.0;
  s = s * z2 + 1.0 / 3.0;
  s = s * z2 + 1.0;
  return (double)e + 2.0 * z * s * 1.4426950408889634;
}

// expm1(x) = 2^k (1 + expm1(r)) - 1 in fp64: range reduction by ln 2 (|r| <= ln2 / 2), degree-13 Taylor series; returns
// expm1(r) and k
DERP_HD double expm1Reduced(double x, double* k) {
  *k = floor(x * 1.4426950408889634 + 0.5);
  const double r = (x - *k * 6.93147180369123816490e-01) - *k * 1.90821492927058770002e-10;
  double p = 1.0 / 6227020800.0;  // 1/13!
  const double inv[12] = {1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0, 1.0 / 40320.0,
                          1.0 / 5040.0, 1.0 / 720.0, 1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0};
  for (int i = 0; i < 12; ++i) p = p * r + inv[i];
  return p * r;
}

// accumulateFS' weight exp(30 a) - 1 as expm1 in fp64 (expm1Reduced, exact ldexp), rounded to fp32: IEEE operations
// only, so that the CPU checker computes the same bits.  GL's fp32 exp(x) - 1 loses the small weights of stretched or
// cone-edge fragments to cancellation; this is the value it approximates.
DERP_HD float blendWeight(float a) {
  const double x = (double)(30.0f * a);
  double k;
  const double em1 = expm1Reduced(x, &k);
  if (k == 0) return (float)em1;
  return (float)(ldexp(1.0 + em1, (int)k) - 1.0);
}

// exp of an fp32 argument by the same series, rounded to fp32 (canopyVS' exp); |x| is clamped to 200, beyond which
// the fp32 result is 0 or inf either way
DERP_HD float expSeries(float xf) {
  if (xf != xf) return xf;
  const double x = xf < -200.0f ? -200.0 : (xf > 200.0f ? 200.0 : (double)xf);
  double k;
  const double em1 = expm1Reduced(x, &k);
  return (float)ldexp(1.0 + em1, (int)k);
}

// atan of an fp32 argument in fp64, rounded to fp32 (canopyVS' atan): atan(x) = pi/2 - atan(1/x) for |x| > 1,
// pi/4 + atan((x - 1) / (x + 1)) above tan(pi/8), then the odd Taylor series to x^43 (|x| <= 0.4143: error < 1e-17)
DERP_HD float atanSeries(float xf) {
  if (xf != xf) return xf;
  double x = xf < 0 ? -(double)xf : (double)xf;
  const bool inv = x > 1;
  if (inv) x = 1.0 / x;
  const bool shift = x > 0.41421356237309503;
  if (shift) x = (x - 1.0) / (x + 1.0);
  const double z = x * x;
  double s = -1.0 / 43.0;
  for (int n = 20; n >= 0; --n) s = s * z + ((n & 1) ? -1.0 : 1.0) / (double)(2 * n + 1);
  double r = x * s;
  if (shift) r += 0.78539816339744830962;
  if (inv) r = 1.57079632679489661923 - r;
  return (float)(xf < 0 ? -r : r);
}

// canopyVS' ipd(lat), fp32 in the shader's order
DERP_HD float ipdAtLat(float ipdm, float lat) {
  const float kPi = 3.1415926535897932384626433832795f, kA = 25, kB = 0.17f;
  const float q = lat / kPi;
  const float e1 = expSeries(kA * ((kB - 0.5f) - q)), e2 = expSeries(kA * ((kB - 0.5f) + q));
  return ipdm * expSeries(-e1 - e2);
}

// canopyVS' error(xy, z, dEst)
DERP_HD float eyeError(float x, float y, float z, float ipdm, float dEst) {
  const float h = ipdAtLat(ipdm, atanSeries(z / dEst)) / 2;
  return ((x * x + y * y) - h * h) - dEst * dEst;
}

// canopyVS' eye(p) (solve with two secant steps, then inverse(A) * p.xy): the offset the vertex moves by, in rig space
// about the rig origin, fp32 operation by operation with exp / atan by the fixed series above.  inverse(A) is
// (1 / det) * adj(A), det = 1 + k * k.
DERP_HD void eyeOffset(float ipdm, float px, float py, float pz, float* ex, float* ey) {
  const float xy2 = px * px + py * py;
  const float i0 = ipdAtLat(ipdm, atanSeries(pz / sqrtf(xy2)));
  float d0 = sqrtf(xy2 - i0 * i0);
  for (int it = 0; it < 2; ++it) {
    const float d1 = (1 + 1e-3f) * d0;
    const float e0 = eyeError(px, py, pz, ipdm, d0), e1 = eyeError(px, py, pz, ipdm, d1);
    const float de = (e1 - e0) / (d1 - d0);
    d0 = d0 - e0 / de;
  }
  const float eNorm = ipdAtLat(ipdm, atanSeries(pz / d0)) / 2;
  const float k = -d0 / eNorm;
  const float idet = 1.0f / (1.0f + k * k);
  *ex = idet * px + (idet * k) * py;
  *ey = (idet * -k) * px + idet * py;
}

DERP_HD float texel(const ushort4* lvl, int W, int H, int i, int j, int c) {
  i %= W;
  if (i < 0) i += W;
  j %= H;
  if (j < 0) j += H;
  const ushort4 t = lvl[(size_t)j * W + i];
  const unsigned short v = c == 0 ? t.x : c == 1 ? t.y : c == 2 ? t.z : t.w;
  return (float)v / 65535.0f;
}

// GL_LINEAR on one level, channels [c0, c1)
DERP_HD void linear(const Canopy& cv, const ushort4* tex, int L, float s, float t, int c0, int c1, float* out) {
  const int W = cv.lw[L], H = cv.lh[L];
  const ushort4* lvl = tex + cv.lofs[L];
  const float uu = s * (float)W - 0.5f, vv = t * (float)H - 0.5f;
  const float fi = floorf(uu), fj = floorf(vv);
  const float a = uu - fi, b = vv - fj;
  const int i0 = (int)fi, j0 = (int)fj;
  for (int c = c0; c < c1; ++c) {
    out[c] = (((1.0f - a) * (1.0f - b)) * texel(lvl, W, H, i0, j0, c) + (a * (1.0f - b)) * texel(lvl, W, H, i0 + 1, j0, c)) +
             (((1.0f - a) * b) * texel(lvl, W, H, i0, j0 + 1, c) + (a * b) * texel(lvl, W, H, i0 + 1, j0 + 1, c));
  }
}

// GL_LINEAR_MIPMAP_LINEAR with MAG = LINEAR (c = 0), channels [c0, c1)
DERP_HD void sampleTex(const Canopy& cv, const ushort4* tex, float s, float t, float lambda, int c0, int c1, float* out) {
  if (!(lambda > 0)) {
    linear(cv, tex, 0, s, t, c0, c1, out);
    return;
  }
  const int q = cv.levels - 1;
  if (lambda >= (float)q) {
    linear(cv, tex, q, s, t, c0, c1, out);
    return;
  }
  const float d1 = floorf(lambda);
  const float tau = lambda - d1;
  float t1[4], t2[4];
  linear(cv, tex, (int)d1, s, t, c0, c1, t1);
  linear(cv, tex, (int)d1 + 1, s, t, c0, c1, t2);
  for (int c = c0; c < c1; ++c) out[c] = (1.0f - tau) * t1[c] + tau * t2[c];
}

struct Frag {
  float depth, u, v, lambda;
  float ax, ay, bx, by;  // dFdx(texVar), dFdy(texVar)
};

// The fragment of screen triangle t at window pixel (px, py); false where t does not cover the pixel centre.
DERP_HD bool fragment(const Canopy& cv, const Tri& t, int px, int py, Frag* f) {
  double l[3];
  if (!bary(t, px + 0.5, py + 0.5, l)) return false;
  f->depth = (float)((l[0] * t.z[0] + l[1] * t.z[1]) + l[2] * t.z[2]);
  f->depth = f->depth < 0 ? 0.0f : (f->depth > 1 ? 1.0f : f->depth);
  const int qx = px & ~1, qy = py & ~1;
  float U[2][2], V[2][2];
  for (int j = 0; j < 2; ++j)
    for (int i = 0; i < 2; ++i) {
      double m[3];
      bary(t, qx + i + 0.5, qy + j + 0.5, m);
      texVarAt(t, m, &U[j][i], &V[j][i]);
    }
  const int ox = px & 1, oy = py & 1;
  f->u = U[oy][ox];
  f->v = V[oy][ox];
  const float ax = U[oy][1] - U[oy][0], ay = V[oy][1] - V[oy][0];  // dFdx
  const float bx = U[1][ox] - U[0][ox], by = V[1][ox] - V[0][ox];  // dFdy
  const float tw = (float)cv.lw[0], th = (float)cv.lh[0];
  const float dux = ax * tw, dvx = ay * th, duy = bx * tw, dvy = by * th;
  const float rx = dux * dux + dvx * dvx, ry = duy * duy + dvy * dvy;
  const float rho2 = rx > ry ? rx : ry;
  f->lambda = rho2 > 0 ? (float)(0.5 * log2Series((double)rho2)) : -INFINITY;
  f->ax = ax;
  f->ay = ay;
  f->bx = bx;
  f->by = by;
  return true;
}

// canopyFS: the squared minor axis of the ellipse a = dFdx, b = dFdy describe
DERP_HD float minorAxis(const Frag& f) {
  const float aa = f.ax * f.ax + f.ay * f.ay, bb = f.bx * f.bx + f.by * f.by, ab = f.ax * f.bx + f.ay * f.by;
  const float h = (aa - bb) / 2;
  return (aa + bb) / 2 - sqrtf(h * h + ab * ab);
}

// canopyFS_SVD: sigma2 / sigma1 of the Jacobian with columns dFdx = (a, b), dFdy = (c, d), fp32 in the shader's order.
// Two cases the shader leaves undefined have a rule here:
//   - fp32 rounding can make s1 - s2 negative (a rank-1 Jacobian), where sqrt gives NaN: sigma2 is then 0, its exact
//     value, and the fragment's alpha is 0.
//   - a zero Jacobian (sigma1 = 0: texVar constant over the quad) stretches no direction more than another: the
//     ratio is 1.
DERP_HD float svdRatio(float a, float b, float c, float d) {
  const float s1 = ((a * a + b * b) + c * c) + d * d;
  const float sb = ((a * a + b * b) - c * c) - d * d;
  const float sc = a * c + b * d;
  const float s2 = sqrtf(sb * sb + (4 * sc) * sc);
  const float sigma1 = sqrtf((s1 + s2) / 2);
  const float m = s1 - s2;
  const float sigma2 = m > 0 ? sqrtf(m / 2) : 0.0f;
  return sigma1 > 0 ? sigma2 / sigma1 : 1.0f;
}

DERP_HD float coneAlpha(float u, float v) {
  const float du = u - 0.5f, dv = v - 0.5f;
  const float c = 1.0f - 2.0f * sqrtf(du * du + dv * dv);
  const float eps = 1.0f / 255.0f;
  return c > eps ? c : eps;
}

// createCubemapTexture's face table (= GL §8.13's): major axis, sc and tc axes of face f, each as +-(axis index + 1)
DERP_HD int faceAxis(int f, int which) {
  const int t[kFaces][3] = {{1, -3, -2}, {-1, 3, -2}, {2, 1, 3}, {-2, 1, -3}, {3, 1, -2}, {-3, -1, -2}};
  return t[f][which];
}

// Component of the integer vector d along the signed axis code
DERP_HD int alongAxis(const int* d, int code) { return code > 0 ? d[code - 1] : -d[-code - 1]; }

// The texel (i, j) of face f (GL rows: j = 0 at the bottom) lies one texel past one edge of the face: the texel of the
// adjacent face it continues to (seamless filtering, GL §8.13.1).  Exact in integers: the texel centre is
// e * MA + (2i + 1 - e) * SC + (2j + 1 - e) * TC in units of half a texel; the overflowing axis becomes the new major axis
// (magnitude e) and the old major axis the new face's edge row (magnitude e - 1).
DERP_HD void seamTexel(int f, int i, int j, int e, int* fo, int* io, int* jo) {
  int d[3] = {0, 0, 0};
  const int ma = faceAxis(f, 0), sc = faceAxis(f, 1), tc = faceAxis(f, 2);
  d[(ma > 0 ? ma : -ma) - 1] = ma > 0 ? e : -e;
  d[(sc > 0 ? sc : -sc) - 1] = (sc > 0 ? 1 : -1) * (2 * i + 1 - e);
  d[(tc > 0 ? tc : -tc) - 1] = (tc > 0 ? 1 : -1) * (2 * j + 1 - e);
  const int off = (i < 0 || i >= e) ? sc : tc;
  const int ax = (off > 0 ? off : -off) - 1, mx = (ma > 0 ? ma : -ma) - 1;
  const int sgn = d[ax] > 0 ? 1 : -1;
  d[ax] = sgn * e;
  d[mx] = (d[mx] > 0 ? 1 : -1) * (e - 1);
  int g = 0;
  while (faceAxis(g, 0) != sgn * (ax + 1)) ++g;
  *fo = g;
  *io = (alongAxis(d, faceAxis(g, 1)) + e - 1) / 2;
  *jo = (alongAxis(d, faceAxis(g, 2)) + e - 1) / 2;
}

// equirectFS' sample of the cubemap `cube` (the unpremultiplied output layout: faces +X .. -Z stacked, each top row
// first, B, G, R, A) in direction (x, y, z): face and (s, t) by GL §8.13 (ties of |x|, |y|, |z| go to x, then y),
// GL_LINEAR at level 0 in GL's bottom-up row order, seamless: a footprint texel past one face edge comes from the
// adjacent face, one past a corner is the mean of the footprint's three other texels, ((p + q) + r) / 3.  IEEE
// arithmetic: a NaN texel anywhere in the footprint makes the sample NaN.
DERP_HD void cubeSample(const float* cube, int e, float x, float y, float z, float* out) {
  const float axv = x < 0 ? -x : x, ayv = y < 0 ? -y : y, azv = z < 0 ? -z : z;
  const float d[3] = {x, y, z};
  int f;
  if (axv >= ayv && axv >= azv) f = x >= 0 ? 0 : 1;
  else if (ayv >= azv) f = y >= 0 ? 2 : 3;
  else f = z >= 0 ? 4 : 5;
  const int ma = faceAxis(f, 0), sc = faceAxis(f, 1), tc = faceAxis(f, 2);
  const float m = ma > 0 ? d[ma - 1] : -d[-ma - 1];
  const float scv = sc > 0 ? d[sc - 1] : -d[-sc - 1], tcv = tc > 0 ? d[tc - 1] : -d[-tc - 1];
  const float s = (scv / m + 1) * 0.5f, t = (tcv / m + 1) * 0.5f;
  const float uu = s * (float)e - 0.5f, vv = t * (float)e - 0.5f;
  const float fi = floorf(uu), fj = floorf(vv);
  const float a = uu - fi, b = vv - fj;
  const int i0 = (int)fi, j0 = (int)fj;
  float tx[4][4];
  int corner = -1;
  for (int k = 0; k < 4; ++k) {
    int fi2 = f, i = i0 + (k & 1), j = j0 + (k >> 1);
    const bool outI = i < 0 || i >= e, outJ = j < 0 || j >= e;
    if (outI && outJ) {
      corner = k;
      continue;
    }
    if (outI || outJ) seamTexel(f, i, j, e, &fi2, &i, &j);
    const float* p = cube + 4 * (((size_t)fi2 * e + (e - 1 - j)) * e + i);
    for (int c = 0; c < 4; ++c) tx[k][c] = p[c];
  }
  if (corner >= 0) {
    const int o0 = corner == 0 ? 1 : 0, o1 = corner <= 1 ? 2 : 1, o2 = corner == 3 ? 2 : 3;
    for (int c = 0; c < 4; ++c) tx[corner][c] = ((tx[o0][c] + tx[o1][c]) + tx[o2][c]) / 3.0f;
  }
  for (int c = 0; c < 4; ++c)
    out[c] = (((1.0f - a) * (1.0f - b)) * tx[0][c] + (a * (1.0f - b)) * tx[1][c]) +
             (((1.0f - a) * b) * tx[2][c] + (a * b) * tx[3][c]);
}

// Gaussian kernel of cv::getGaussianKernel(2r + 1, 1.5, CV_32F): fp64 weights, normalised, narrowed to float
inline void gaussianWeights(int r, float* w) {
  const int n = 2 * r + 1;
  double cd[64], sum = 0;
  const double scale2X = -0.5 / (1.5 * 1.5);
  for (int i = 0; i < n; ++i) {
    const double x = i - (n - 1) * 0.5;
    cd[i] = std::exp(scale2X * x * x);
    sum += cd[i];
  }
  sum = 1. / sum;
  for (int i = 0; i < n; ++i) w[i] = (float)(cd[i] * sum);
}

// createCubemapTexture (CanopyScene.cpp:340-379): per face, Eigen's fp32 projection * view
inline void faceMatrices(const float* center, FaceMats* out) {
  static const float table[kFaces][3][3] = {
      {{1, 0, 0}, {0, 0, -1}, {0, -1, 0}},  {{-1, 0, 0}, {0, 0, 1}, {0, -1, 0}}, {{0, 1, 0}, {1, 0, 0}, {0, 0, 1}},
      {{0, -1, 0}, {1, 0, 0}, {0, 0, -1}}, {{0, 0, 1}, {1, 0, 0}, {0, -1, 0}},  {{0, 0, -1}, {-1, 0, 0}, {0, -1, 0}}};
  const float kNearZ = 0.1f;
  const float P[16] = {2 * kNearZ / (kNearZ - -kNearZ), 0, (kNearZ + -kNearZ) / (kNearZ - -kNearZ), 0,
                       0, 2 * kNearZ / (kNearZ - -kNearZ), (kNearZ + -kNearZ) / (kNearZ - -kNearZ), 0,
                       0, 0, -1, -2 * kNearZ,
                       0, 0, -1, 0};
  for (int f = 0; f < kFaces; ++f) {
    float T[16] = {0};
    for (int c = 0; c < 3; ++c) {
      T[0 * 4 + c] = table[f][1][c];
      T[1 * 4 + c] = table[f][2][c];
      T[2 * 4 + c] = -table[f][0][c];
    }
    T[15] = 1;
    for (int r = 0; r < 3; ++r)  // translate(-position): t = linear * -position
      T[r * 4 + 3] = (T[r * 4 + 0] * -center[0] + T[r * 4 + 1] * -center[1]) + T[r * 4 + 2] * -center[2];
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c)
        out->m[f][r * 4 + c] = ((P[r * 4 + 0] * T[0 * 4 + c] + P[r * 4 + 1] * T[1 * 4 + c]) + P[r * 4 + 2] * T[2 * 4 + c]) +
                               P[r * 4 + 3] * T[3 * 4 + c];
  }
}

// SimpleMeshRenderer's snapshot matrix: frustum(-xMax, xMax, -xMax * H / W, xMax * H / W, 0.1) (GlUtil.h, far plane at
// infinity) times posForwardUp(position, forward, up), in fp32 in Eigen's order; xMax = 0.1 * tan(fov / 180 * pi / 2) in
// fp64 rounded to fp32.  Returns false when forward and up do not give a unitary basis (forwardUp's CHECK).
inline bool snapshotMatrix(const float* position, const float* forward, const float* up, double horizontalFovDeg,
                           int width, int height, float* out) {
  float R[3][3];
  if (!smr::forwardUp(forward, up, &R[0][0])) return false;
  float T[4][4] = {};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[r][c] = R[r][c];
    T[r][3] = (R[r][0] * -position[0] + R[r][1] * -position[1]) + R[r][2] * -position[2];  // result * -position
  }
  T[3][3] = 1;
  const float n = 0.1f;
  const float xMax = (float)((double)n * std::tan(horizontalFovDeg / 180 * 3.14159265358979323846 / 2));
  const float minX = -xMax, maxX = xMax, minY = (float)(-xMax * height) / width, maxY = (float)(xMax * height) / width;
  const float P[4][4] = {{2 * n / (maxX - minX), 0, (maxX + minX) / (maxX - minX), 0},
                         {0, 2 * n / (maxY - minY), (maxY + minY) / (maxY - minY), 0},
                         {0, 0, -1, -2 * n},
                         {0, 0, -1, 0}};
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[r * 4 + c] = ((P[r][0] * T[0][c] + P[r][1] * T[1][c]) + P[r][2] * T[2][c]) + P[r][3] * T[3][c];
  return true;
}

#if defined(__CUDACC__)
__device__ __forceinline__ uint16_t unorm16(float v) {
  if (!(v > 0)) return 0;  // NaN too
  if (v >= 1) return 65535;
  return (uint16_t)floorf(v * 65535.0f + 0.5f);
}

// disparityMesh (+ canopyVS' eye offset when ipd != 0), alphaFov and the GL_RGBA16 upload of one canopy over a
// w x h grid of camera `cam` (rescaled to that grid); disparityColor(metersToGrayscale) for the disparity texture
// (DisparityColor.h:18-57).  vtx and texD need disp; texC alone (a colour texture at its own size) does not.
__global__ void rephotoPrepKernel(DevCamera cam, const float* disp, const float* bgra, int w, int h, float cx, float cy,
                                  float cz, float ipd, float* vtx, ushort4* texC, ushort4* texD, int* anyZero) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const size_t i = (size_t)y * w + x;
  const float d = disp ? disp[i] : 0.0f;
  double dir[3];
  pixelRay(cam, x + 0.5, y + 0.5, dir);
  if (vtx) {
    const float distance = 1.0f / d;
    float p[3];
    for (int k = 0; k < 3; ++k) p[k] = (float)(cam.pos[k] + dir[k] * (double)distance);
    if (ipd != 0) {
      float ex, ey;
      eyeOffset(ipd, p[0], p[1], p[2], &ex, &ey);
      p[0] = p[0] - ex;
      p[1] = p[1] - ey;
    }
    for (int k = 0; k < 3; ++k) vtx[3 * i + k] = p[k];
  }
  if (!texC && !texD) return;
  const bool outside = outsideImageCircle(cam, x + 0.5, y + 0.5);
  if (outside) atomicOr(anyZero, 1);
  const uint16_t a = outside ? 0 : 65535;
  if (texC) {
    const float* c = bgra + 4 * i;
    texC[i] = make_ushort4(unorm16(c[0]), unorm16(c[1]), unorm16(c[2]), a);
  }
  if (texD) {
    const double dist2 = (float)(1.0 / (double)d);  // DisparityColor.h: float distance = 1.0 / disparity
    const float wx = (float)(cam.pos[0] + dir[0] * dist2), wy = (float)(cam.pos[1] + dir[1] * dist2),
                wz = (float)(cam.pos[2] + dir[2] * dist2);
    const float ex = wx - cx, ey = wy - cy, ez = wz - cz;
    const float meters = sqrtf(ex * ex + ey * ey + ez * ez);
    const uint16_t g = unorm16(1 / meters);
    texD[i] = make_ushort4(g, g, g, a);
  }
}

__global__ void rephotoMipKernel(const ushort4* src, int sw, int sh, ushort4* dst, int dw, int dh) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  const int x0 = min(2 * x, sw - 1), x1 = min(2 * x + 1, sw - 1), y0 = min(2 * y, sh - 1), y1 = min(2 * y + 1, sh - 1);
  const ushort4 a = src[(size_t)y0 * sw + x0], b = src[(size_t)y0 * sw + x1], c = src[(size_t)y1 * sw + x0],
                d = src[(size_t)y1 * sw + x1];
  dst[(size_t)y * dw + x] = make_ushort4((a.x + b.x + c.x + d.x + 2) >> 2, (a.y + b.y + c.y + d.y + 2) >> 2,
                                         (a.z + b.z + c.z + d.z + 2) >> 2, (a.w + b.w + c.w + d.w + 2) >> 2);
}

// One thread per (primitive, view): every covered pixel centre whose fragment survives the alpha test bids
// (depth bits, ~prim) with a 64-bit atomicMin; the least key is GL_LEQUAL's survivor in draw order.  mats: 16 floats
// per view; every view is W x H.
__global__ void __launch_bounds__(256) rephotoRasterKernel(Canopy cv, const float* __restrict__ mats, int W, int H,
                                                          int prims, unsigned long long* keys) {
  const int prim = blockIdx.x * blockDim.x + threadIdx.x, view = blockIdx.y;
  if (prim >= prims) return;
  float M[16];
  for (int i = 0; i < 16; ++i) M[i] = mats[16 * view + i];
  Tri tris[2];
  const int n = setupPrim(cv, M, W, H, prim, tris);
  unsigned long long* fk = keys + (size_t)view * W * H;
  for (int k = 0; k < n; ++k) {
    const Tri& t = tris[k];
    const float mnx = fminf(fminf(t.x[0], t.x[1]), t.x[2]), mxx = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]);
    const float mny = fminf(fminf(t.y[0], t.y[1]), t.y[2]), mxy = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]);
    const int x0 = (int)fmaxf(0.0f, ceilf(mnx - 0.5f)), x1 = (int)fminf((float)(W - 1), floorf(mxx - 0.5f));
    const int y0 = (int)fmaxf(0.0f, ceilf(mny - 0.5f)), y1 = (int)fminf((float)(H - 1), floorf(mxy - 0.5f));
    for (int py = y0; py <= y1; ++py)
      for (int px = x0; px <= x1; ++px) {
        Frag f;
        if (!fragment(cv, t, px, py, &f)) continue;
        if (cv.anyZeroAlpha) {
          float a[4];
          sampleTex(cv, cv.tex[0] ? cv.tex[0] : cv.tex[1], f.u, f.v, f.lambda, 3, 4, a);
          if (a[3] == 0) continue;
        }
        const unsigned long long key = ((unsigned long long)__float_as_uint(f.depth) << 32) | (unsigned)(~(unsigned)prim);
        atomicMin(fk + (size_t)py * W + px, key);
      }
  }
}

// The surviving fragment of each pixel, shaded by canopyFS or canopyFS_SVD and blended by accumulateFS into the fp32
// sums; optionally reports the winning primitive in the output layout (views stacked, e.g. cube faces +X, -X, +Y, -Y,
// +Z, -Z, each top row first).
__global__ void rephotoResolveKernel(Canopy cv, const float* __restrict__ mats, int W, int H, int views,
                                     const unsigned long long* keys, float4* accC, float4* accD, int32_t* winners) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = W * H;
  if (idx >= views * per) return;
  const int face = idx / per, px = (idx % per) % W, py = (idx % per) / W;
  const size_t o = (size_t)face * per + (size_t)(H - 1 - py) * W + px;
  const unsigned long long key = keys[idx];
  if (winners) winners[o] = key == ~0ull ? -1 : (int32_t)(~(unsigned)(key & 0xffffffffu));
  if (key == ~0ull) return;
  const int prim = (int)(~(unsigned)(key & 0xffffffffu));
  float M[16];
  for (int i = 0; i < 16; ++i) M[i] = mats[16 * face + i];
  Tri tris[2];
  const int n = setupPrim(cv, M, W, H, prim, tris);
  Frag f;
  bool hit = false;
  for (int k = 0; k < n && !hit; ++k) hit = fragment(cv, tris[k], px, py, &f);
  if (!hit) return;  // unreachable: the raster pass found this fragment
  const float mod = cv.svd ? svdRatio(f.ax, f.ay, f.bx, f.by) : minorAxis(f);
  const float cone = coneAlpha(f.u, f.v);
  float c[4];
  const ushort4* alphaTex = cv.tex[0] ? cv.tex[0] : cv.tex[1];
  sampleTex(cv, alphaTex, f.u, f.v, f.lambda, 3, 4, c);
  float a = c[3];
  a *= mod;
  a *= cone;
  const float w = cv.alphaBlend ? blendWeight(a) : a;
  for (int t = 0; t < 2; ++t) {
    if (!cv.tex[t]) continue;
    sampleTex(cv, cv.tex[t], f.u, f.v, f.lambda, 0, 3, c);
    float4* acc = t == 0 ? accC : accD;
    float4 s = acc[o];
    s.x = w * c[0] + s.x;
    s.y = w * c[1] + s.y;
    s.z = w * c[2] + s.z;
    s.w = w + s.w;
    acc[o] = s;
  }
}

// unpremulFS (rgba / a); zeroNan adds rephotography's zeroOutNans (ComputeRephotographyErrors.cpp:64-75), without it
// NaN (no canopy) stays
__global__ void rephotoUnpremulKernel(size_t n, const float4* acc, int zeroNan, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 s = acc[i];
  const float v[4] = {s.x / s.w, s.y / s.w, s.z / s.w, s.w / s.w};
  for (int c = 0; c < 4; ++c) out[4 * i + c] = zeroNan && v[c] != v[c] ? 0.0f : v[c];
}

// equirectFS: output pixel (x, y) of the 2e x e equirect, row y = 0 first as glReadPixels leaves it (lat = +pi/2 side).
// trig holds fp32 roundings of fp64 cos / sin: [cos lat (e) | sin lat (e) | cos lon (2e) | sin lon (2e)].
__global__ void canopyEquirectKernel(const float* __restrict__ cube, int e, const float* __restrict__ trig, float* out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= 2 * e) return;
  const float cl = trig[y], sl = trig[e + y], co = trig[2 * e + x], so = trig[4 * e + x];
  cubeSample(cube, e, cl * co, cl * so, sl, out + 4 * ((size_t)y * 2 * e + x));
}

__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// Separable Gaussian of `planes` interleaved 3-channel fp32 images (cv::GaussianBlur, BORDER_REFLECT_101): rows, then
// columns, each a left-to-right fp32 sum of weight * sample.
__global__ void rephotoBlurRowsKernel(const float* src, int w, int h, int r, const float* __restrict__ wt, float* dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
  if (x >= w) return;
  const float* s = src + (size_t)img * w * h * 3 + (size_t)y * w * 3;
  float acc[3] = {0, 0, 0};
  for (int k = -r; k <= r; ++k) {
    const int xx = reflect101(x + k, w);
    for (int c = 0; c < 3; ++c) acc[c] = acc[c] + wt[k + r] * s[3 * xx + c];
  }
  float* d = dst + (size_t)img * w * h * 3 + ((size_t)y * w + x) * 3;
  for (int c = 0; c < 3; ++c) d[c] = acc[c];
}

__global__ void rephotoBlurColsKernel(const float* src, int w, int h, int r, const float* __restrict__ wt, float* dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
  if (x >= w) return;
  const float* s = src + (size_t)img * w * h * 3;
  float acc[3] = {0, 0, 0};
  for (int k = -r; k <= r; ++k) {
    const int yy = reflect101(y + k, h);
    for (int c = 0; c < 3; ++c) acc[c] = acc[c] + wt[k + r] * s[((size_t)yy * w + x) * 3 + c];
  }
  float* d = dst + (size_t)img * w * h * 3 + ((size_t)y * w + x) * 3;
  for (int c = 0; c < 3; ++c) d[c] = acc[c];
}

// (x - muX)^2, (y - muY)^2, (x - muX)(y - muY) as three images; mu = [muX | muY]
__global__ void rephotoMomentsKernel(size_t n, const float* x, const float* y, const float* mu, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float dx = x[i] - mu[i], dy = y[i] - mu[n + i];
  out[i] = dx * dx;
  out[n + i] = dy * dy;
  out[2 * n + i] = dx * dy;
}

// computeSSIM's per-pixel tail (RephotographyUtil.h:65-84) and the masked, NaN-excluding sums of averageScore:
// one fp64 (sum, count) pair per channel and CTA.
__global__ void __launch_bounds__(256) rephotoScoreKernel(size_t pixels, const float* mu, const float* sig, const uint8_t* mask,
                                                          int ncc, float* score, double* partial) {
  __shared__ double ssum[3][256];
  __shared__ unsigned scnt[3][256];
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n = pixels * 3;
  const float c1 = 0.0001f, c2 = 0.0009f, c3 = (float)((double)0.0009f / 2.0f);
  for (int c = 0; c < 3; ++c) {
    ssum[c][threadIdx.x] = 0;
    scnt[c][threadIdx.x] = 0;
  }
  if (p < pixels) {
    for (int c = 0; c < 3; ++c) {
      const size_t i = p * 3 + c;
      const float muX = mu[i], muY = mu[n + i];
      const float sig2X = sig[i], sig2Y = sig[n + i], sigXY = sig[2 * n + i];
      const float sigX = sqrtf(sig2X), sigY = sqrtf(sig2Y);
      float lum = 1, con = 1;
      if (!ncc) {
        lum = (2 * (muX * muY) + c1) * (1.0f / ((muX * muX + muY * muY) + c1));
        con = (2 * (sigX * sigY) + c2) * (1.0f / ((sig2X + sig2Y) + c2));
      }
      const float str = (sigXY + c3) * (1.0f / (sigX * sigY + c3));
      const float v = (con * lum) * str;
      score[i] = v;
      if (mask[p] && v == v) {
        ssum[c][threadIdx.x] = v;
        scnt[c][threadIdx.x] = 1;
      }
    }
  }
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int c = 0; c < 3; ++c) {
        ssum[c][threadIdx.x] += ssum[c][threadIdx.x + s];
        scnt[c][threadIdx.x] += scnt[c][threadIdx.x + s];
      }
    __syncthreads();
  }
  if (threadIdx.x < 3) {
    partial[blockIdx.x * 6 + threadIdx.x] = ssum[threadIdx.x][0];
    partial[blockIdx.x * 6 + 3 + threadIdx.x] = (double)scnt[threadIdx.x][0];
  }
}
#endif

}  // namespace rephoto
}  // namespace derp
