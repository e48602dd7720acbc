// TEST INFRASTRUCTURE ONLY — the CPU checker of the rephotography ABI (include/derp_rephoto.h).  Compiled by
// tests/rephoto_oracle.py into a temporary directory and loaded by tests/test_rephoto.py and tests/test_gpu_rephoto.py;
// never linked into the product.  It uses the depth oracle's camera model and OpenCV border helper (oracle/camera.h,
// oracle/cvprims.h) as they are, and exports derp_rephoto_cubemap / derp_rephoto_score with the CUDA library's
// signatures, plus the heat-map panel of the app's plot for the cv2 pin.
//
// Build flags mirror oracle/Makefile (-O3 -funroll-loops -ffp-contract=off): no FMA contraction, so the fp32 / fp64
// sequences below are the device's bit for bit.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

#include "../include/derp_rephoto.h"
#include "../oracle/camera.h"
#include "../oracle/cvprims.h"
#include "../facebook360_dep_b200/csrc/host/rephoto_plot.h"

namespace oracle {
namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
// one thread per item of [begin, end)
void parallelFor(int begin, int end, const std::function<void(int, int)>& fn) {
  std::vector<std::thread> ths;
  for (int i = begin; i < end; ++i) ths.emplace_back([&fn, i] { fn(i, i + 1); });
  for (auto& t : ths) t.join();
}
}  // namespace
}  // namespace oracle

// ---- rephotography: CPU restatement of derp_rephoto_cubemap / derp_rephoto_score --------------------------------------
// CanopyScene (CanopyScene.cpp) in the mode ComputeRephotographyErrors uses (cubemap, ipd 0, alphaBlend, canopyFS), under
// the rules documented in facebook360_dep_b200/csrc/derp_rephoto.cuh, written the way GL states them: a depth buffer
// per canopy and face, primitives drawn one after the other in strip order with GL_LEQUAL, each fragment shaded and
// alpha-tested before the depth test, then blended into the fp32 accumulation buffer.  The score follows
// RephotographyUtil.h with cv::GaussianBlur restated (pinned to cv2 by tests/golden/rephoto_vectors.npz).
namespace oracle {
namespace rephoto {

struct Tex {  // GL_RGBA16 mip chain, B, G, R, A
  std::vector<std::vector<uint16_t>> lv;
  std::vector<int> w, h;
};

static uint16_t unorm16(float v) {
  if (!(v > 0)) return 0;
  if (v >= 1) return 65535;
  return (uint16_t)std::floor(v * 65535.0f + 0.5f);
}

static void buildMips(Tex& t) {
  while (t.w.back() > 1 || t.h.back() > 1) {
    const int sw = t.w.back(), sh = t.h.back(), dw = std::max(1, sw / 2), dh = std::max(1, sh / 2);
    const std::vector<uint16_t>& s = t.lv.back();
    std::vector<uint16_t> d((size_t)dw * dh * 4);
    for (int y = 0; y < dh; ++y)
      for (int x = 0; x < dw; ++x) {
        const int xs[2] = {std::min(2 * x, sw - 1), std::min(2 * x + 1, sw - 1)};
        const int ys[2] = {std::min(2 * y, sh - 1), std::min(2 * y + 1, sh - 1)};
        for (int c = 0; c < 4; ++c) {
          int sum = 2;
          for (int j = 0; j < 2; ++j)
            for (int i = 0; i < 2; ++i) sum += s[((size_t)ys[j] * sw + xs[i]) * 4 + c];
          d[((size_t)y * dw + x) * 4 + c] = (uint16_t)(sum >> 2);
        }
      }
    t.lv.push_back(std::move(d));
    t.w.push_back(dw);
    t.h.push_back(dh);
  }
}

static float fetch(const Tex& t, int L, int i, int j, int c) {
  const int W = t.w[L], H = t.h[L];
  i = ((i % W) + W) % W;  // GL_REPEAT
  j = ((j % H) + H) % H;
  return (float)t.lv[L][((size_t)j * W + i) * 4 + c] / 65535.0f;
}

static float bilinear(const Tex& t, int L, float s, float tt, int c) {
  const float uu = s * (float)t.w[L] - 0.5f, vv = tt * (float)t.h[L] - 0.5f;
  const float fi = std::floor(uu), fj = std::floor(vv);
  const float a = uu - fi, b = vv - fj;
  const int i0 = (int)fi, j0 = (int)fj;
  return (((1.0f - a) * (1.0f - b)) * fetch(t, L, i0, j0, c) + (a * (1.0f - b)) * fetch(t, L, i0 + 1, j0, c)) +
         (((1.0f - a) * b) * fetch(t, L, i0, j0 + 1, c) + (a * b) * fetch(t, L, i0 + 1, j0 + 1, c));
}

static float trilinear(const Tex& t, float s, float tt, float lambda, int c) {
  const int q = (int)t.lv.size() - 1;
  if (!(lambda > 0)) return bilinear(t, 0, s, tt, c);
  if (lambda >= (float)q) return bilinear(t, q, s, tt, c);
  const float d1 = std::floor(lambda), tau = lambda - d1;
  return (1.0f - tau) * bilinear(t, (int)d1, s, tt, c) + tau * bilinear(t, (int)d1 + 1, s, tt, c);
}

static double log2Series(double x) {  // the device's fixed series (derp_rephoto.cuh)
  int e;
  const double m = std::frexp(x, &e);
  const double z = (m - 1.0) / (m + 1.0), z2 = z * z;
  double s = 1.0 / 15.0;
  const double k[7] = {1.0 / 13.0, 1.0 / 11.0, 1.0 / 9.0, 1.0 / 7.0, 1.0 / 5.0, 1.0 / 3.0, 1.0};
  for (double kk : k) s = s * z2 + kk;
  return (double)e + 2.0 * z * s * 1.4426950408889634;
}

// accumulateFS' weight exp(30 a) - 1: expm1 in fp64 by the device's fixed series (derp_rephoto.cuh), rounded to fp32
static float blendWeight(float a) {
  const double x = (double)(30.0f * a);
  const double k = std::floor(x * 1.4426950408889634 + 0.5);
  const double r = (x - k * 6.93147180369123816490e-01) - k * 1.90821492927058770002e-10;
  const double inv[13] = {1.0 / 6227020800.0, 1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0,
                          1.0 / 40320.0, 1.0 / 5040.0, 1.0 / 720.0, 1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0};
  double p = inv[0];
  for (int i = 1; i < 13; ++i) p = p * r + inv[i];
  const double em1 = p * r;
  if (k == 0) return (float)em1;
  return (float)(std::ldexp(1.0 + em1, (int)k) - 1.0);
}

struct V {
  float x, y, z, w, u, v;
};

struct Screen {
  float x[3], y[3], z[3], q[3], uq[3], vq[3];
  double area;
};

static bool edgeTest(const Screen& t, double px, double py, double* l) {
  const double s = t.area > 0 ? 1.0 : -1.0;
  bool in = true;
  for (int i = 0; i < 3; ++i) {
    const int a = (i + 1) % 3, b = (i + 2) % 3;
    const double dx = (double)t.x[b] - t.x[a], dy = (double)t.y[b] - t.y[a];
    const double e = (dx * (py - t.y[a]) - dy * (px - t.x[a])) * s;
    const bool topLeft = dy * s < 0 || (dy == 0 && dx * s < 0);
    if (!(e > 0 || (e == 0 && topLeft))) in = false;
    l[i] = e / (t.area * s);
  }
  return in;
}

static void interpTex(const Screen& t, const double* l, float* u, float* v) {
  const double iw = (l[0] * t.q[0] + l[1] * t.q[1]) + l[2] * t.q[2];
  *u = (float)(((l[0] * t.uq[0] + l[1] * t.uq[1]) + l[2] * t.uq[2]) / iw);
  *v = (float)(((l[0] * t.vq[0] + l[1] * t.vq[1]) + l[2] * t.vq[2]) / iw);
}

struct Scene {
  int w = 0, h = 0;
  std::vector<std::vector<float>> vtx;
  std::vector<Tex> color, disp;
  std::vector<bool> anyZero;
};

// Eigen: projection(frustum(-n, n, -n, n, n)) * view, fp32 (CanopyScene.cpp:340-378, GlUtil.h frustum)
static void faceMatrix(int face, const float* p, float* M) {
  static const float tab[6][3][3] = {
      {{1, 0, 0}, {0, 0, -1}, {0, -1, 0}},  {{-1, 0, 0}, {0, 0, 1}, {0, -1, 0}}, {{0, 1, 0}, {1, 0, 0}, {0, 0, 1}},
      {{0, -1, 0}, {1, 0, 0}, {0, 0, -1}}, {{0, 0, 1}, {1, 0, 0}, {0, -1, 0}},  {{0, 0, -1}, {-1, 0, 0}, {0, -1, 0}}};
  const float n = 0.1f;
  const float P[4][4] = {{2 * n / (n - -n), 0, (n + -n) / (n - -n), 0},
                         {0, 2 * n / (n - -n), (n + -n) / (n - -n), 0},
                         {0, 0, -1, -2 * n},
                         {0, 0, -1, 0}};
  float T[4][4] = {};
  for (int c = 0; c < 3; ++c) {
    T[0][c] = tab[face][1][c];
    T[1][c] = tab[face][2][c];
    T[2][c] = -tab[face][0][c];
  }
  T[3][3] = 1;
  for (int r = 0; r < 3; ++r) T[r][3] = (T[r][0] * -p[0] + T[r][1] * -p[1]) + T[r][2] * -p[2];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) M[r * 4 + c] = ((P[r][0] * T[0][c] + P[r][1] * T[1][c]) + P[r][2] * T[2][c]) + P[r][3] * T[3][c];
}

// Canopy::render of one canopy into one face: depth buffer cleared to 1, strip order, GL_LEQUAL
static void renderFace(const Scene& sc, int ci, const float* M, int edge, bool wantColor, bool wantDisp,
                       std::vector<float>& canC, std::vector<float>& canD, std::vector<float>& alpha,
                       std::vector<int32_t>& prim) {
  const size_t P = (size_t)edge * edge;
  std::vector<float> depth(P, 1.0f);
  std::fill(alpha.begin(), alpha.end(), 0.0f);
  std::fill(prim.begin(), prim.end(), -1);
  const int w = sc.w, h = sc.h;
  const float* vt = sc.vtx[ci].data();
  const Tex& A = wantColor ? sc.color[ci] : sc.disp[ci];
  const float sx = (float)(1.0 / w), sy = (float)(1.0 / h), half = 0.5f * (float)edge;
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
            s.x[j] = (tv[j]->x / tv[j]->w) * half + half;
            s.y[j] = (tv[j]->y / tv[j]->w) * half + half;
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
          const int x0 = (int)std::max(0.0, std::ceil(mnx - 0.5)), x1 = (int)std::min(edge - 1.0, std::floor(mxx - 0.5));
          const int y0 = (int)std::max(0.0, std::ceil(mny - 0.5)), y1 = (int)std::min(edge - 1.0, std::floor(mxy - 0.5));
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
              const float dux = ax * (float)w, dvx = ay * (float)h, duy = bx * (float)w, dvy = by * (float)h;
              const float rx = dux * dux + dvx * dvx, ry = duy * duy + dvy * dvy;
              const float rho2 = std::max(rx, ry);
              const float lambda = rho2 > 0 ? (float)(0.5 * log2Series((double)rho2)) : -INFINITY;
              // canopyFS
              float a = trilinear(A, u, vv, lambda, 3);
              if (a == 0) continue;  // discard: no depth write
              const size_t o = (size_t)py * edge + px;
              if (!(z <= depth[o])) continue;
              depth[o] = z;
              const float aa = ax * ax + ay * ay, bb = bx * bx + by * by, ab = ax * bx + ay * by;
              const float hh = (aa - bb) / 2;
              const float minor = (aa + bb) / 2 - std::sqrt(hh * hh + ab * ab);
              a *= minor;
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

static void blurC3(const float* src, int w, int h, const float* k, int r, float* dst) {
  std::vector<float> tmp((size_t)w * h * 3);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c) {
        float s = 0;
        for (int i = -r; i <= r; ++i) s = s + k[i + r] * src[((size_t)y * w + reflect101(x + i, w)) * 3 + c];
        tmp[((size_t)y * w + x) * 3 + c] = s;
      }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c) {
        float s = 0;
        for (int i = -r; i <= r; ++i) s = s + k[i + r] * tmp[((size_t)reflect101(y + i, h) * w + x) * 3 + c];
        dst[((size_t)y * w + x) * 3 + c] = s;
      }
}

}  // namespace rephoto
}  // namespace oracle

extern "C" {

int derp_rephoto_cubemap(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                         const float* const* colors_bgra, int width, int height, const float* center, int edge,
                         float* out_color, float* out_disparity, int32_t* winners) {
  using namespace oracle;
  using namespace oracle::rephoto;
  if (!cams || num_cams < 0 || (num_cams > 0 && !disparities) || width < 2 || height < 2 || !center || edge < 2 ||
      (!out_color && !out_disparity) || (out_color && num_cams > 0 && !colors_bgra))
    return fail(DERP_EINVAL, "derp_rephoto_cubemap: bad arguments");
  Scene sc;
  sc.w = width;
  sc.h = height;
  const size_t n = (size_t)width * height;
  sc.vtx.resize(num_cams);
  sc.color.resize(num_cams);
  sc.disp.resize(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    Camera full;
    if (!full.init(cams[i])) return fail(DERP_EINVAL, "derp_rephoto_cubemap: invalid camera " + std::to_string(i));
    const Camera cam = full.rescale(width, height);
    std::vector<float>& vt = sc.vtx[i];
    vt.resize(n * 3);
    Tex& tc = sc.color[i];
    Tex& td = sc.disp[i];
    tc.lv.assign(1, std::vector<uint16_t>(out_color ? n * 4 : 0));
    td.lv.assign(1, std::vector<uint16_t>(out_disparity ? n * 4 : 0));
    tc.w = td.w = {width};
    tc.h = td.h = {height};
    for (int y = 0; y < height; ++y)
      for (int x = 0; x < width; ++x) {
        const size_t o = (size_t)y * width + x;
        const double pix[2] = {x + 0.5, y + 0.5};
        const float d = disparities[i][o];
        double r[3];
        cam.rig(pix, (double)(1.0f / d), r);  // disparityMesh: float distance = 1.0f / disparity
        for (int k = 0; k < 3; ++k) vt[o * 3 + k] = (float)r[k];
        const uint16_t a = cam.isOutsideImageCircle(pix) ? 0 : 65535;  // alphaFov
        if (out_color)
          for (int c = 0; c < 4; ++c) tc.lv[0][o * 4 + c] = c == 3 ? a : unorm16(colors_bgra[i][o * 4 + c]);
        if (out_disparity) {  // disparityColor(metersToGrayscale): float distance = 1.0 / disparity (double division)
          double q[3];
          cam.rig(pix, (double)(float)(1.0 / (double)d), q);
          const float ex = (float)q[0] - center[0], ey = (float)q[1] - center[1], ez = (float)q[2] - center[2];
          const float meters = std::sqrt(ex * ex + ey * ey + ez * ez);
          const uint16_t g = unorm16(1 / meters);
          for (int c = 0; c < 4; ++c) td.lv[0][o * 4 + c] = c == 3 ? a : g;
        }
      }
    if (out_color) buildMips(tc);
    if (out_disparity) buildMips(td);
  }
  const size_t P = (size_t)edge * edge;
  std::vector<float> accC(out_color ? 6 * P * 4 : 0, 0.0f), accD(out_disparity ? 6 * P * 4 : 0, 0.0f);
  std::vector<int32_t> win(winners ? 6 * P * num_cams : 0, -1);
  parallelFor(0, 6, [&](int f0, int f1) {
    std::vector<float> canC(P * 3), canD(P * 3), alpha(P);
    std::vector<int32_t> prim(P);
    for (int face = f0; face < f1; ++face) {
      float M[16];
      faceMatrix(face, center, M);
      for (int ci = 0; ci < num_cams; ++ci) {  // accumulate (CanopyScene.cpp:306-310), camera order
        renderFace(sc, ci, M, edge, out_color != nullptr, out_disparity != nullptr, canC, canD, alpha, prim);
        for (int py = 0; py < edge; ++py)
          for (int px = 0; px < edge; ++px) {
            const size_t o = (size_t)py * edge + px;
            const size_t dst = (size_t)face * P + (size_t)(edge - 1 - py) * edge + px;  // faces stacked, flipped
            if (winners) win[(size_t)ci * 6 * P + dst] = prim[o];
            if (prim[o] < 0) continue;  // cleared canopy pixel: alpha 0, weight 0
            const float wgt = blendWeight(alpha[o]);
            for (int t = 0; t < 2; ++t) {
              std::vector<float>& acc = t == 0 ? accC : accD;
              const std::vector<float>& can = t == 0 ? canC : canD;
              if (acc.empty()) continue;
              for (int c = 0; c < 3; ++c) acc[dst * 4 + c] = wgt * can[o * 3 + c] + acc[dst * 4 + c];
              acc[dst * 4 + 3] = wgt + acc[dst * 4 + 3];
            }
          }
      }
    }
  });
  for (int t = 0; t < 2; ++t) {  // unpremulFS + zeroOutNans
    float* out = t == 0 ? out_color : out_disparity;
    const std::vector<float>& acc = t == 0 ? accC : accD;
    if (!out) continue;
    for (size_t i = 0; i < 6 * P; ++i)
      for (int c = 0; c < 4; ++c) {
        const float v = acc[i * 4 + c] / acc[i * 4 + 3];
        out[i * 4 + c] = v != v ? 0.0f : v;
      }
  }
  if (winners) std::memcpy(winners, win.data(), win.size() * sizeof(int32_t));
  return DERP_OK;
}

int derp_rephoto_score(int device, const float* ref_bgr, const float* ren_bgr, const uint8_t* mask, int width, int height,
                       int method, int stat_radius, float* score_map, double* avg) {
  using namespace oracle;
  if (!ref_bgr || !ren_bgr || !mask || width < 1 || height < 1 || !score_map || !avg)
    return fail(DERP_EINVAL, "derp_rephoto_score: bad arguments");
  if (method != DERP_REPHOTO_MSSIM && method != DERP_REPHOTO_NCC)
    return fail(DERP_EINVAL, "derp_rephoto_score: method must be DERP_REPHOTO_MSSIM or DERP_REPHOTO_NCC");
  if (stat_radius < 1 || stat_radius > 31) return fail(DERP_EINVAL, "derp_rephoto_score: stat_radius in [1, 31]");
  // cv::getGaussianKernel(2r + 1, 1.5, CV_32F)
  const int ks = 2 * stat_radius + 1;
  std::vector<double> cd(ks);
  double sum = 0;
  for (int i = 0; i < ks; ++i) {
    const double x = i - (ks - 1) * 0.5;
    cd[i] = std::exp((-0.5 / (1.5 * 1.5)) * x * x);
    sum += cd[i];
  }
  std::vector<float> k(ks);
  for (int i = 0; i < ks; ++i) k[i] = (float)(cd[i] * (1. / sum));
  const size_t n = (size_t)width * height * 3;
  std::vector<float> muX(n), muY(n), a(n), b(n), c(n), sig2X(n), sig2Y(n), sigXY(n);
  rephoto::blurC3(ref_bgr, width, height, k.data(), stat_radius, muX.data());
  rephoto::blurC3(ren_bgr, width, height, k.data(), stat_radius, muY.data());
  for (size_t i = 0; i < n; ++i) {
    const float dx = ref_bgr[i] - muX[i], dy = ren_bgr[i] - muY[i];
    a[i] = dx * dx;
    b[i] = dy * dy;
    c[i] = dx * dy;
  }
  rephoto::blurC3(a.data(), width, height, k.data(), stat_radius, sig2X.data());
  rephoto::blurC3(b.data(), width, height, k.data(), stat_radius, sig2Y.data());
  rephoto::blurC3(c.data(), width, height, k.data(), stat_radius, sigXY.data());
  const float c1 = 0.0001f, c2 = 0.0009f, c3 = (float)((double)0.0009f / 2.0f);
  double s[3] = {0, 0, 0}, cnt[3] = {0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const float sigX = std::sqrt(sig2X[i]), sigY = std::sqrt(sig2Y[i]);
    float lum = 1, con = 1;  // cv::pow(x, 0) = 1 everywhere (NCC)
    if (method == DERP_REPHOTO_MSSIM) {
      lum = (2 * (muX[i] * muY[i]) + c1) * (1.0f / ((muX[i] * muX[i] + muY[i] * muY[i]) + c1));
      con = (2 * (sigX * sigY) + c2) * (1.0f / ((sig2X[i] + sig2Y[i]) + c2));
    }
    const float str = (sigXY[i] + c3) * (1.0f / (sigX * sigY + c3));
    const float v = (con * lum) * str;
    score_map[i] = v;
    if (mask[i / 3] && v == v) {
      s[i % 3] += v;
      cnt[i % 3] += 1;
    }
  }
  for (int ch = 0; ch < 3; ++ch) avg[ch] = cnt[ch] > 0 ? s[ch] / cnt[ch] : 0.0;
  return DERP_OK;
}

const char* derp_backend(void) { return "rephoto-oracle-cpu"; }
const char* derp_last_error(void) { return oracle::g_err.c_str(); }

// stackResults' heat-map panel (the app's own code, facebook360_dep_b200/csrc/host/rephoto_plot.h), pinned to cv2
void oracle_rephoto_jet_panel(const float* score_bgr, const uint8_t* mask, int w, int h, uint8_t* out_bgr) {
  rephoto_plot::jetPanel(score_bgr, mask, w, h, out_bgr);
}
}  // extern "C"
