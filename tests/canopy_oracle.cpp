// TEST INFRASTRUCTURE ONLY — the CPU checker of the canopy ABI (include/derp_canopy.h), the renderer SimpleMeshRenderer
// exports with.  Compiled by tests/canopy_oracle.py into a temporary directory and loaded by tests/test_smr.py and
// tests/test_gpu_smr.py; never linked into the product.
//
// It builds on the rephotography checker (tests/rephoto_oracle.cpp, included as it is: its RGBA16 textures and mips,
// trilinear sampling, log2 and blend-weight series, edge functions and cube-face matrices) and restates what the
// exporter adds, under the rules documented in facebook360_dep_b200/csrc/derp_rephoto.cuh, the way GL states them:
// views of any size with their own matrices, mesh size separate from texture size, canopyFS_SVD, blending off, canopyVS'
// stereo eye offset, unpremultiply keeping NaN and equirectFS' seamless resample.  Each canopy is drawn into each view
// with a depth buffer of its own, primitives in strip order with GL_LEQUAL.  It also exports the app-side host steps
// (facebook360_dep_b200/csrc/host/smr_host.h) for the numpy and cv2 pins.
//
// Build flags mirror oracle/Makefile (-O3 -funroll-loops -ffp-contract=off): no FMA contraction, so the fp32 / fp64
// sequences below are the device's bit for bit.
#include "rephoto_oracle.cpp"

#include "../include/derp_canopy.h"
#include "../facebook360_dep_b200/csrc/host/smr_host.h"

namespace oracle {
namespace rephoto {

// expm1 in fp64 by the device's fixed series (derp_rephoto.cuh): expm1(r) after reduction by ln 2, and k
static double expm1Reduced(double x, double* kOut) {
  const double k = std::floor(x * 1.4426950408889634 + 0.5);
  const double r = (x - k * 6.93147180369123816490e-01) - k * 1.90821492927058770002e-10;
  const double inv[13] = {1.0 / 6227020800.0, 1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0,
                          1.0 / 40320.0, 1.0 / 5040.0, 1.0 / 720.0, 1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0};
  double p = inv[0];
  for (int i = 1; i < 13; ++i) p = p * r + inv[i];
  *kOut = k;
  return p * r;
}

// canopyVS' exp and atan: the device's fixed series, fp64 rounded to fp32
static float expSeries(float xf) {
  if (std::isnan(xf)) return xf;
  double k;
  const double em1 = expm1Reduced(std::min(200.0, std::max(-200.0, (double)xf)), &k);
  return (float)std::ldexp(1.0 + em1, (int)k);
}

static float atanSeries(float xf) {
  if (std::isnan(xf)) return xf;
  double x = std::fabs((double)xf);
  const bool inv = x > 1, shift = (inv ? 1.0 / x : x) > 0.41421356237309503;
  if (inv) x = 1.0 / x;
  if (shift) x = (x - 1.0) / (x + 1.0);
  double s = -1.0 / 43.0;
  for (int n = 20; n >= 0; --n) s = s * (x * x) + (n % 2 ? -1.0 : 1.0) / (double)(2 * n + 1);
  double r = x * s;
  if (shift) r += 0.78539816339744830962;
  if (inv) r = 1.57079632679489661923 - r;
  return (float)(xf < 0 ? -r : r);
}

// canopyVS (CanopyScene.cpp): ipd(lat), error, solve (two secant steps), eye; fp32 in the shader's order
static float ipdAt(float ipdm, float lat) {
  const float kPi = 3.1415926535897932384626433832795f, kA = 25, kB = 0.17f;
  return ipdm * expSeries(-expSeries(kA * ((kB - 0.5f) - lat / kPi)) - expSeries(kA * ((kB - 0.5f) + lat / kPi)));
}

static void eye(float ipdm, const float* p, float* e) {
  auto error = [&](float dEst) {
    const float h = ipdAt(ipdm, atanSeries(p[2] / dEst)) / 2;
    return ((p[0] * p[0] + p[1] * p[1]) - h * h) - dEst * dEst;
  };
  const float xy2 = p[0] * p[0] + p[1] * p[1];
  const float i0 = ipdAt(ipdm, atanSeries(p[2] / std::sqrt(xy2)));
  float d0 = std::sqrt(xy2 - i0 * i0);
  for (int it = 0; it < 2; ++it) {
    const float d1 = (1 + 1e-3f) * d0;
    const float e0 = error(d0), e1 = error(d1);
    d0 = d0 - e0 / ((e1 - e0) / (d1 - d0));
  }
  const float k = -d0 / (ipdAt(ipdm, atanSeries(p[2] / d0)) / 2);
  const float idet = 1.0f / (1.0f + k * k);  // inverse(mat2(1, k, -k, 1)) = (1 / det) * adj
  e[0] = idet * p[0] + (idet * k) * p[1];
  e[1] = (idet * -k) * p[0] + idet * p[1];
}

// canopyFS_SVD's sigma2 / sigma1 with derp_rephoto.cuh's rule: s1 - s2 <= 0 gives sigma2 = 0, sigma1 = 0 gives 1
static float svdRatio(float a, float b, float c, float d) {
  const float s1 = ((a * a + b * b) + c * c) + d * d;
  const float sb = ((a * a + b * b) - c * c) - d * d;
  const float sc = a * c + b * d;
  const float s2 = std::sqrt(sb * sb + (4 * sc) * sc);
  const float sigma1 = std::sqrt((s1 + s2) / 2);
  const float sigma2 = s1 - s2 > 0 ? std::sqrt((s1 - s2) / 2) : 0.0f;
  return sigma1 > 0 ? sigma2 / sigma1 : 1.0f;
}

struct CanopySet {
  int w = 0, h = 0;  // mesh size
  std::vector<std::vector<float>> vtx;
  std::vector<Tex> color, disp;
  bool svd = false, alphaBlend = true;
};

// Canopy::render of one canopy into one W x H view: depth buffer cleared to 1, strip order, GL_LEQUAL
static void renderView(const CanopySet& sc, int ci, const float* M, int W, int H, bool wantColor, bool wantDisp,
                       std::vector<float>& canC, std::vector<float>& canD, std::vector<float>& alpha,
                       std::vector<int32_t>& prim) {
  const size_t P = (size_t)W * H;
  std::vector<float> depth(P, 1.0f);
  std::fill(alpha.begin(), alpha.end(), 0.0f);
  std::fill(prim.begin(), prim.end(), -1);
  const int w = sc.w, h = sc.h;
  const float* vt = sc.vtx[ci].data();
  const Tex& A = wantColor ? sc.color[ci] : sc.disp[ci];
  const float tw = (float)A.w[0], th = (float)A.h[0];  // the LOD's scale: the sampled texture's size
  const float sx = (float)(1.0 / w), sy = (float)(1.0 / h), halfW = 0.5f * (float)W, halfH = 0.5f * (float)H;
  for (int cy = 0; cy + 1 < h; ++cy)
    for (int cx = 0; cx + 1 < w; ++cx)
      for (int k = 0; k < 2; ++k) {
        const int pid = (cy * (w - 1) + cx) * 2 + k;
        const int ids[2][3] = {{cy * w + cx, (cy + 1) * w + cx, cy * w + cx + 1},
                               {(cy + 1) * w + cx, cy * w + cx + 1, (cy + 1) * w + cx + 1}};
        V v[3];
        bool ok = true;
        for (int i = 0; i < 3; ++i) {
          const int id = ids[k][i];
          const float* p = vt + 3 * (size_t)id;
          if (!(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]))) ok = false;
          v[i].x = ((M[0] * p[0] + M[1] * p[1]) + M[2] * p[2]) + M[3];
          v[i].y = ((M[4] * p[0] + M[5] * p[1]) + M[6] * p[2]) + M[7];
          v[i].z = ((M[8] * p[0] + M[9] * p[1]) + M[10] * p[2]) + M[11];
          v[i].w = ((M[12] * p[0] + M[13] * p[1]) + M[14] * p[2]) + M[15];
          v[i].u = sx * ((float)(id % w) + 0.5f);
          v[i].v = sy * ((float)(id / w) + 0.5f);
        }
        if (!ok) continue;
        // near-plane clipping z >= -w
        std::vector<V> poly;
        for (int i = 0; i < 3; ++i) {
          const V& a = v[i];
          const V& b = v[(i + 1) % 3];
          const float da = a.z + a.w, db = b.z + b.w;
          if (da >= 0) poly.push_back(a);
          if ((da >= 0) != (db >= 0)) {
            const V& from = da >= 0 ? a : b;
            const V& to = da >= 0 ? b : a;
            const float df = da >= 0 ? da : db, dt = da >= 0 ? db : da;
            const float t = df / (df - dt);
            poly.push_back({from.x + t * (to.x - from.x), from.y + t * (to.y - from.y), from.z + t * (to.z - from.z),
                            from.w + t * (to.w - from.w), from.u + t * (to.u - from.u), from.v + t * (to.v - from.v)});
          }
        }
        for (size_t f = 1; f + 1 < poly.size(); ++f) {
          const V* tv[3] = {&poly[0], &poly[f], &poly[f + 1]};
          Screen s;
          for (int j = 0; j < 3; ++j) {
            const float iw = 1.0f / tv[j]->w;
            s.x[j] = (tv[j]->x / tv[j]->w) * halfW + halfW;
            s.y[j] = (tv[j]->y / tv[j]->w) * halfH + halfH;
            s.z[j] = (tv[j]->z / tv[j]->w) * 0.5f + 0.5f;
            s.q[j] = iw;
            s.uq[j] = tv[j]->u * iw;
            s.vq[j] = tv[j]->v * iw;
          }
          s.area = ((double)s.x[1] - s.x[0]) * ((double)s.y[2] - s.y[0]) - ((double)s.x[2] - s.x[0]) * ((double)s.y[1] - s.y[0]);
          if (!(s.area != 0)) continue;
          // every pixel centre of the viewport the triangle could cover
          const double mnx = std::min({s.x[0], s.x[1], s.x[2]}), mxx = std::max({s.x[0], s.x[1], s.x[2]});
          const double mny = std::min({s.y[0], s.y[1], s.y[2]}), mxy = std::max({s.y[0], s.y[1], s.y[2]});
          const int x0 = (int)std::max(0.0, std::ceil(mnx - 0.5)), x1 = (int)std::min(W - 1.0, std::floor(mxx - 0.5));
          const int y0 = (int)std::max(0.0, std::ceil(mny - 0.5)), y1 = (int)std::min(H - 1.0, std::floor(mxy - 0.5));
          for (int py = y0; py <= y1; ++py)
            for (int px = x0; px <= x1; ++px) {
              double l[3];
              if (!edgeTest(s, px + 0.5, py + 0.5, l)) continue;
              float z = (float)((l[0] * s.z[0] + l[1] * s.z[1]) + l[2] * s.z[2]);
              z = z < 0 ? 0.0f : (z > 1 ? 1.0f : z);
              // helper invocations: the quad's four centres on this triangle's interpolant
              float U[2][2], Vv[2][2];
              const int qx = px & ~1, qy = py & ~1;
              for (int j = 0; j < 2; ++j)
                for (int i = 0; i < 2; ++i) {
                  double m[3];
                  edgeTest(s, qx + i + 0.5, qy + j + 0.5, m);
                  interpTex(s, m, &U[j][i], &Vv[j][i]);
                }
              const int ox = px & 1, oy = py & 1;
              const float u = U[oy][ox], vv = Vv[oy][ox];
              const float ax = U[oy][1] - U[oy][0], ay = Vv[oy][1] - Vv[oy][0];
              const float bx = U[1][ox] - U[0][ox], by = Vv[1][ox] - Vv[0][ox];
              const float dux = ax * tw, dvx = ay * th, duy = bx * tw, dvy = by * th;
              const float rx = dux * dux + dvx * dvx, ry = duy * duy + dvy * dvy;
              const float rho2 = std::max(rx, ry);
              const float lambda = rho2 > 0 ? (float)(0.5 * log2Series((double)rho2)) : -INFINITY;
              // canopyFS
              float a = trilinear(A, u, vv, lambda, 3);
              if (a == 0) continue;  // discard: no depth write
              const size_t o = (size_t)py * W + px;
              if (!(z <= depth[o])) continue;
              depth[o] = z;
              if (sc.svd) {
                a *= svdRatio(ax, ay, bx, by);
              } else {
                const float aa = ax * ax + ay * ay, bb = bx * bx + by * by, ab = ax * bx + ay * by;
                const float hh = (aa - bb) / 2;
                const float minor = (aa + bb) / 2 - std::sqrt(hh * hh + ab * ab);
                a *= minor;
              }
              const float du = u - 0.5f, dv = vv - 0.5f;
              a *= std::max(1.0f / 255.0f, 1.0f - 2.0f * std::sqrt(du * du + dv * dv));
              alpha[o] = a;
              prim[o] = pid;
              for (int c = 0; c < 3; ++c) {
                if (wantColor) canC[o * 3 + c] = trilinear(sc.color[ci], u, vv, lambda, c);
                if (wantDisp) canD[o * 3 + c] = trilinear(sc.disp[ci], u, vv, lambda, c);
              }
            }
        }
      }
}

static const int kAxes[6][3] = {{1, -3, -2}, {-1, 3, -2}, {2, 1, 3}, {-2, 1, -3}, {3, 1, -2}, {-3, -1, -2}};

static int along(const int* d, int code) { return code > 0 ? d[code - 1] : -d[-code - 1]; }

// GL §8.13.1 seamless filtering: the texel one past an edge of face f is the adjacent face's edge texel that continues
// the row or column (exact in half-texel integer coordinates)
static void seam(int f, int i, int j, int e, int* fo, int* io, int* jo) {
  int d[3] = {0, 0, 0};
  const int ma = kAxes[f][0], sc = kAxes[f][1], tc = kAxes[f][2];
  d[std::abs(ma) - 1] = ma > 0 ? e : -e;
  d[std::abs(sc) - 1] = (sc > 0 ? 1 : -1) * (2 * i + 1 - e);
  d[std::abs(tc) - 1] = (tc > 0 ? 1 : -1) * (2 * j + 1 - e);
  const int ax = std::abs((i < 0 || i >= e) ? sc : tc) - 1, mx = std::abs(ma) - 1;
  const int sgn = d[ax] > 0 ? 1 : -1;
  d[ax] = sgn * e;
  d[mx] = (d[mx] > 0 ? 1 : -1) * (e - 1);
  int g = 0;
  while (kAxes[g][0] != sgn * (ax + 1)) ++g;
  *fo = g;
  *io = (along(d, kAxes[g][1]) + e - 1) / 2;
  *jo = (along(d, kAxes[g][2]) + e - 1) / 2;
}

// equirectFS over the unpremultiplied cube (output layout), GL_LINEAR at level 0, seamless, corner = mean of three
static void equirect(const float* cube, int e, float* out) {
  const double kPi = 3.14159265358979323846;
  for (int y = 0; y < e; ++y)
    for (int x = 0; x < 2 * e; ++x) {
      const double lat = -(((y + 0.5) / e) - 0.5) * kPi, lon = (1 - (x + 0.5) / (2 * e)) * 2.0 * kPi;
      const float cl = (float)std::cos(lat), sl = (float)std::sin(lat), co = (float)std::cos(lon),
                  so = (float)std::sin(lon);
      const float d[3] = {cl * co, cl * so, sl};
      const float a0 = std::fabs(d[0]), a1 = std::fabs(d[1]), a2 = std::fabs(d[2]);
      const int f = (a0 >= a1 && a0 >= a2) ? (d[0] >= 0 ? 0 : 1) : (a1 >= a2 ? (d[1] >= 0 ? 2 : 3) : (d[2] >= 0 ? 4 : 5));
      auto comp = [&](int code) { return code > 0 ? d[code - 1] : -d[-code - 1]; };
      const float m = comp(kAxes[f][0]);
      const float s = (comp(kAxes[f][1]) / m + 1) * 0.5f, t = (comp(kAxes[f][2]) / m + 1) * 0.5f;
      const float uu = s * (float)e - 0.5f, vv = t * (float)e - 0.5f;
      const float fi = std::floor(uu), fj = std::floor(vv), a = uu - fi, b = vv - fj;
      float tx[4][4];
      int corner = -1;
      for (int k = 0; k < 4; ++k) {
        int g = f, i = (int)fi + (k & 1), j = (int)fj + (k >> 1);
        const bool oi = i < 0 || i >= e, oj = j < 0 || j >= e;
        if (oi && oj) {
          corner = k;
          continue;
        }
        if (oi || oj) seam(f, i, j, e, &g, &i, &j);
        for (int c = 0; c < 4; ++c) tx[k][c] = cube[(((size_t)g * e + (e - 1 - j)) * e + i) * 4 + c];
      }
      if (corner >= 0) {
        std::vector<int> o;
        for (int k = 0; k < 4; ++k)
          if (k != corner) o.push_back(k);
        for (int c = 0; c < 4; ++c) tx[corner][c] = ((tx[o[0]][c] + tx[o[1]][c]) + tx[o[2]][c]) / 3.0f;
      }
      for (int c = 0; c < 4; ++c)
        out[((size_t)y * 2 * e + x) * 4 + c] = (((1.0f - a) * (1.0f - b)) * tx[0][c] + (a * (1.0f - b)) * tx[1][c]) +
                                               (((1.0f - a) * b) * tx[2][c] + (a * b) * tx[3][c]);
    }
}

// CanopyScene::cubemap / equirect / render (include/derp_canopy.h): scenes with textures of one size share the raster
static int render(const char* who, const DerpCameraDesc* cams, int num_cams, const float* const* disparities, int width,
                  int height, const float* const* colors_bgra, int cw, int ch, int projection, const float* center,
                  const float* matrix, int outW, int outH, float ipd, bool alphaBlend, bool svd,
                  float* out_color, float* out_disparity, int32_t* winners) {
  const std::string name(who);
  if (!cams || num_cams < 0 || (num_cams > 0 && !disparities) || width < 2 || height < 2 || !center ||
      (!out_color && !out_disparity) || (out_color && num_cams > 0 && !colors_bgra) || (out_color && (cw < 1 || ch < 1)))
    return fail(DERP_EINVAL, name + ": bad arguments");
  int views, W, H;
  if (projection == DERP_CANOPY_CUBEMAP || projection == DERP_CANOPY_EQUIRECT) {
    if (!(projection == DERP_CANOPY_CUBEMAP ? outW == outH : outW == 2 * outH) || outH < 2)
      return fail(DERP_EINVAL, name + ": bad output size for the projection");
    views = 6;
    W = H = outH;
  } else if (projection == DERP_CANOPY_PERSPECTIVE) {
    if (!matrix || outW < 1 || outH < 1) return fail(DERP_EINVAL, name + ": perspective needs a matrix and a size");
    views = 1;
    W = outW;
    H = outH;
  } else {
    return fail(DERP_EINVAL, name + ": unknown projection");
  }
  CanopySet sc;
  sc.w = width;
  sc.h = height;
  sc.svd = svd;
  sc.alphaBlend = alphaBlend;
  const size_t n = (size_t)width * height, nc = (size_t)cw * ch;
  sc.vtx.resize(num_cams);
  sc.color.resize(num_cams);
  sc.disp.resize(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    Camera full;
    if (!full.init(cams[i])) return fail(DERP_EINVAL, name + ": invalid camera " + std::to_string(i));
    const Camera cam = full.rescale(width, height);
    std::vector<float>& vt = sc.vtx[i];
    vt.resize(n * 3);
    Tex& td = sc.disp[i];
    td.lv.assign(1, std::vector<uint16_t>(out_disparity ? n * 4 : 0));
    td.w = {width};
    td.h = {height};
    for (int y = 0; y < height; ++y)
      for (int x = 0; x < width; ++x) {
        const size_t o = (size_t)y * width + x;
        const double pix[2] = {x + 0.5, y + 0.5};
        const float d = disparities[i][o];
        double r[3];
        cam.rig(pix, (double)(1.0f / d), r);  // disparityMesh: float distance = 1.0f / disparity
        float p[3] = {(float)r[0], (float)r[1], (float)r[2]};
        if (ipd != 0) {  // canopyVS: pos -= eye(pos)
          float e[2];
          eye(ipd, p, e);
          p[0] = p[0] - e[0];
          p[1] = p[1] - e[1];
        }
        for (int k = 0; k < 3; ++k) vt[o * 3 + k] = p[k];
        if (out_disparity) {  // disparityColor(metersToGrayscale): float distance = 1.0 / disparity (double division)
          const uint16_t a = cam.isOutsideImageCircle(pix) ? 0 : 65535;  // alphaFov
          double q[3];
          cam.rig(pix, (double)(float)(1.0 / (double)d), q);
          const float ex = (float)q[0] - center[0], ey = (float)q[1] - center[1], ez = (float)q[2] - center[2];
          const float meters = std::sqrt(ex * ex + ey * ey + ez * ez);
          const uint16_t g = unorm16(1 / meters);
          for (int c = 0; c < 4; ++c) td.lv[0][o * 4 + c] = c == 3 ? a : g;
        }
      }
    if (out_disparity) buildMips(td);
    if (out_color) {  // alphaFov at the colour's own size
      const Camera ccam = full.rescale(cw, ch);
      Tex& tc = sc.color[i];
      tc.lv.assign(1, std::vector<uint16_t>(nc * 4));
      tc.w = {cw};
      tc.h = {ch};
      for (int y = 0; y < ch; ++y)
        for (int x = 0; x < cw; ++x) {
          const size_t o = (size_t)y * cw + x;
          const double pix[2] = {x + 0.5, y + 0.5};
          const uint16_t a = ccam.isOutsideImageCircle(pix) ? 0 : 65535;
          for (int c = 0; c < 4; ++c) tc.lv[0][o * 4 + c] = c == 3 ? a : unorm16(colors_bgra[i][o * 4 + c]);
        }
      buildMips(tc);
    }
  }
  std::vector<float> mats(16 * views);
  if (views == 6)
    for (int f = 0; f < 6; ++f) faceMatrix(f, center, &mats[16 * f]);
  else
    for (int i = 0; i < 16; ++i) mats[i] = matrix[i];
  const bool shared = out_color && out_disparity && cw == width && ch == height;
  const size_t P = (size_t)W * H;
  std::vector<float> accC(out_color ? views * P * 4 : 0, 0.0f), accD(out_disparity ? views * P * 4 : 0, 0.0f);
  std::vector<int32_t> win(winners ? views * P * num_cams : 0, -1);
  // passes: (colour, disparity) flags; the first pass reports the winners
  std::vector<std::pair<bool, bool>> passes;
  if (shared) passes.push_back({true, true});
  else {
    if (out_color) passes.push_back({true, false});
    if (out_disparity) passes.push_back({false, true});
  }
  for (size_t pi = 0; pi < passes.size(); ++pi) {
    const bool wc = passes[pi].first, wd = passes[pi].second;
    parallelFor(0, views, [&](int f0, int f1) {
      std::vector<float> canC(P * 3), canD(P * 3), alpha(P);
      std::vector<int32_t> prim(P);
      for (int face = f0; face < f1; ++face) {
        for (int ci = 0; ci < num_cams; ++ci) {  // accumulate (CanopyScene.cpp:306-310), camera order
          renderView(sc, ci, &mats[16 * face], W, H, wc, wd, canC, canD, alpha, prim);
          for (int py = 0; py < H; ++py)
            for (int px = 0; px < W; ++px) {
              const size_t o = (size_t)py * W + px;
              const size_t dst = (size_t)face * P + (size_t)(H - 1 - py) * W + px;  // views stacked, flipped
              if (winners && pi == 0) win[(size_t)ci * views * P + dst] = prim[o];
              if (prim[o] < 0) continue;  // cleared canopy pixel: alpha 0, weight 0
              const float wgt = sc.alphaBlend ? blendWeight(alpha[o]) : alpha[o];
              for (int t = 0; t < 2; ++t) {
                if (!(t == 0 ? wc : wd)) continue;
                std::vector<float>& acc = t == 0 ? accC : accD;
                const std::vector<float>& can = t == 0 ? canC : canD;
                for (int c = 0; c < 3; ++c) acc[dst * 4 + c] = wgt * can[o * 3 + c] + acc[dst * 4 + c];
                acc[dst * 4 + 3] = wgt + acc[dst * 4 + 3];
              }
            }
        }
      }
    });
  }
  std::vector<float> un(views * P * 4);
  for (int t = 0; t < 2; ++t) {  // unpremulFS: NaN (no canopy) stays
    float* out = t == 0 ? out_color : out_disparity;
    const std::vector<float>& acc = t == 0 ? accC : accD;
    if (!out) continue;
    for (size_t i = 0; i < views * P; ++i)
      for (int c = 0; c < 4; ++c) un[i * 4 + c] = acc[i * 4 + c] / acc[i * 4 + 3];
    if (projection == DERP_CANOPY_EQUIRECT) equirect(un.data(), outH, out);
    else std::memcpy(out, un.data(), un.size() * sizeof(float));
  }
  if (winners) std::memcpy(winners, win.data(), win.size() * sizeof(int32_t));
  return DERP_OK;
}

}  // namespace rephoto
}  // namespace oracle

extern "C" {

int derp_canopy_render(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                       int mesh_width, int mesh_height, const float* const* colors_bgra, int color_width,
                       int color_height, int projection, const float* position, const float* matrix, int out_width,
                       int out_height, float ipd, int alpha_blend, int shader, float* out_color, float* out_disparity,
                       int32_t* winners) {
  if (shader != DERP_CANOPY_ON_SCREEN && shader != DERP_CANOPY_SVD)
    return oracle::fail(DERP_EINVAL, "derp_canopy_render: bad shader");
  return oracle::rephoto::render("derp_canopy_render", cams, num_cams, disparities, mesh_width, mesh_height, colors_bgra,
                                 color_width, color_height, projection, position, matrix, out_width, out_height, ipd,
                                 alpha_blend != 0, shader == DERP_CANOPY_SVD, out_color, out_disparity, winners);
}

// canopyVS' eye offset of n rig-space points (the device's eyeOffset), for the fp64 comparison
void oracle_canopy_eye(const float* p, int n, float ipd, float* out) {
  for (int i = 0; i < n; ++i) oracle::rephoto::eye(ipd, p + 3 * i, out + 2 * i);
}

float oracle_canopy_svd_ratio(float a, float b, float c, float d) { return oracle::rephoto::svdRatio(a, b, c, d); }

// SimpleMeshRenderer's host steps (the app's own code, facebook360_dep_b200/csrc/host/smr_host.h and io.h)
void oracle_smr_png16(const float* bgra, int n, uint16_t* out) {
  const std::vector<uint16_t> v = smr::toPng16(bgra, (size_t)n);
  std::memcpy(out, v.data(), v.size() * sizeof(uint16_t));
}
void oracle_smr_alpha_blend(float* fore, const float* back, int n) { smr::alphaBlend(fore, back, (size_t)n); }
int oracle_smr_background_equirect(float* fore, int w, int h, const float* equi, int ew, int eh, const float* position,
                                   const float* forward, const float* up, double fov) {
  float R[9];
  if (!smr::forwardUp(forward, up, R)) return -1;
  smr::backgroundEquirect(fore, w, h, equi, ew, eh, R, position, fov);
  return 0;
}
void oracle_smr_lr180(const float* left, const float* right, int w, int h, float* out) {
  const std::vector<float> l(left, left + (size_t)w * h * 4), r(right, right + (size_t)w * h * 4);
  const std::vector<float> v = smr::lr180(l, r, w, h);
  std::memcpy(out, v.data(), v.size() * sizeof(float));
}
}  // extern "C"
