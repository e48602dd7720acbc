// include/derp_rephoto.h and include/derp_canopy.h: the canopy renderer and the rephotography score on sm_90a
// (derp_rephoto.cuh).
#include <cmath>
#include <cstring>

#include "derp_host.cuh"
#include "derp_rephoto.cuh"
#include "../../include/derp_rephoto.h"
#include "../../include/derp_canopy.h"

using namespace derp;

// ---- rephotography (derp_rephoto.cuh) ----------------------------------------------------------------
// Grow-only scratch per host thread, like the camera mesh: the app renders four cubemaps and one score per camera.
namespace {
struct RephotoScratch {
  DevBuf<float> disp, bgra, vtx, out, f32, mats, trig, eq;
  DevBuf<ushort4> texC, texD;
  DevBuf<unsigned long long> keys;
  DevBuf<float4> accC, accD;
  DevBuf<int> flags;
  DevBuf<int32_t> win;
  DevBuf<uint8_t> mask;
  DevBuf<double> partial;
};
thread_local RephotoScratch g_rephoto;

// CanopyScene::cubemap / equirect / render (derp_canopy.h) in every mode; rephotography is the cubemap, ipd 0,
// alpha-blended, on-screen case with NaN set to 0.  When the colour and the disparity colour are both wanted at one
// texture size, one raster serves both; otherwise each scene is a pass of its own (the alpha test and the LOD depend on
// the texture's size).
int canopyRender(const char* who, int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                 int mw, int mh, const float* const* colors_bgra, int cw, int ch, int projection, const float* position,
                 const float* matrix, int outW, int outH, float ipd, int alphaBlend, int shader, bool zeroNan,
                 float* out_color, float* out_disparity, int32_t* winners) {
  using namespace derp::rephoto;
  const std::string name(who);
  if (!cams || num_cams < 0 || (num_cams > 0 && !disparities) || mw < 2 || mh < 2 || !position ||
      (!out_color && !out_disparity) || (out_color && num_cams > 0 && !colors_bgra) || (out_color && (cw < 1 || ch < 1)))
    return fail(DERP_EINVAL, name + ": bad arguments");
  if (shader != DERP_CANOPY_ON_SCREEN && shader != DERP_CANOPY_SVD)
    return fail(DERP_EINVAL, name + ": shader must be DERP_CANOPY_ON_SCREEN or DERP_CANOPY_SVD");
  int views, W, H;  // the raster: `views` viewports of W x H
  if (projection == DERP_CANOPY_CUBEMAP || projection == DERP_CANOPY_EQUIRECT) {
    const bool ok = projection == DERP_CANOPY_CUBEMAP ? outW == outH : outW == 2 * outH;
    if (!ok || outH < 2) return fail(DERP_EINVAL, name + ": bad output size for the projection");
    views = kFaces;
    W = H = outH;
  } else if (projection == DERP_CANOPY_PERSPECTIVE) {
    if (!matrix || outW < 1 || outH < 1) return fail(DERP_EINVAL, name + ": perspective needs a matrix and a size");
    views = 1;
    W = outW;
    H = outH;
  } else {
    return fail(DERP_EINVAL, name + ": unknown projection");
  }
  if ((long long)mw * mh >= (1ll << 30) || (out_color && (long long)cw * ch >= (1ll << 30)) ||
      (long long)W * H * views >= (1ll << 31))
    return fail(DERP_EINVAL, name + ": image or output too large");
  std::vector<DevCamera> dcMesh(num_cams), dcTex(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    DevCamera c;
    if (!host::makeCamera(cams[i], &c)) return fail(DERP_EINVAL, name + ": invalid camera " + std::to_string(i));
    dcMesh[i] = host::rescaled(c, mw, mh);  // camera.rescale({disparity.cols, disparity.rows})
    if (out_color) dcTex[i] = host::rescaled(c, cw, ch);  // alphaFov: camera.rescale({color.cols, color.rows})
  }
  std::vector<float> mats(16 * views);
  if (views == kFaces) {
    FaceMats fm;
    faceMatrices(position, &fm);
    for (int f = 0; f < kFaces; ++f) std::memcpy(&mats[16 * f], fm.m[f], 16 * sizeof(float));
  } else {
    std::memcpy(mats.data(), matrix, 16 * sizeof(float));
  }
  struct Pass {
    bool color, disp;
  };
  std::vector<Pass> passes;
  if (out_color && out_disparity && cw == mw && ch == mh) {
    passes.push_back({true, true});
  } else {
    if (out_color) passes.push_back({true, false});
    if (out_disparity) passes.push_back({false, true});
  }
  CU(cudaSetDevice(device));
  RephotoScratch& s = g_rephoto;
  const size_t n = (size_t)mw * mh, nc = out_color ? (size_t)cw * ch : 0;
  const size_t pixels = (size_t)views * W * H;
  CU(s.disp.ensure(n));
  CU(s.vtx.ensure(n * 3));
  CU(s.keys.ensure(pixels));
  CU(s.flags.ensure(1));
  if (int rc = upload(s.mats, mats.data(), mats.size())) return rc;
  if (out_color) {
    CU(s.bgra.ensure(nc * 4));
    CU(s.accC.ensure(pixels));
    CU(cudaMemset(s.accC.p, 0, pixels * sizeof(float4)));
  }
  if (out_disparity) {
    CU(s.accD.ensure(pixels));
    CU(cudaMemset(s.accD.p, 0, pixels * sizeof(float4)));
  }
  if (winners) CU(s.win.ensure(pixels * std::max(num_cams, 1)));
  CU(s.out.ensure(pixels * 4));
  const int prims = (mw - 1) * (mh - 1) * 2;
  for (size_t pi = 0; pi < passes.size(); ++pi) {
    const Pass& ps = passes[pi];
    const int tw = ps.color ? cw : mw, th = ps.color ? ch : mh;
    int levels = 1;
    while ((tw >> levels) > 0 || (th >> levels) > 0) ++levels;
    if (levels > kMaxLevels) return fail(DERP_EINVAL, name + ": image too large");
    Canopy cv{};
    cv.mw = mw;
    cv.mh = mh;
    cv.levels = levels;
    cv.svd = shader == DERP_CANOPY_SVD;
    cv.alphaBlend = alphaBlend != 0;
    long long texels = 0;
    for (int l = 0; l < levels; ++l) {
      cv.lw[l] = std::max(1, tw >> l);
      cv.lh[l] = std::max(1, th >> l);
      cv.lofs[l] = texels;
      texels += (long long)cv.lw[l] * cv.lh[l];
    }
    if (ps.color) CU(s.texC.ensure(texels));
    if (ps.disp) CU(s.texD.ensure(texels));
    ushort4* texC = ps.color ? s.texC.p : nullptr;
    ushort4* texD = ps.disp ? s.texD.p : nullptr;
    cv.vtx = s.vtx.p;
    cv.tex[0] = texC;
    cv.tex[1] = texD;
    int32_t* win = winners && pi == 0 ? s.win.p : nullptr;
    const bool ownGrid = ps.color && (cw != mw || ch != mh);  // the colour texture on a grid of its own
    for (int i = 0; i < num_cams; ++i) {  // canopies in camera order: the blend sums are order-dependent
      CU(cudaMemcpy(s.disp.p, disparities[i], n * sizeof(float), cudaMemcpyDefault));
      if (ps.color) CU(cudaMemcpy(s.bgra.p, colors_bgra[i], nc * 4 * sizeof(float), cudaMemcpyDefault));
      CU(cudaMemset(s.flags.p, 0, sizeof(int)));
      if (ownGrid) {
        rephotoPrepKernel<<<dim3((cw + 127) / 128, ch), 128>>>(dcTex[i], nullptr, s.bgra.p, cw, ch, position[0], position[1],
                                                              position[2], 0.0f, nullptr, texC, nullptr, s.flags.p);
        rephotoPrepKernel<<<dim3((mw + 127) / 128, mh), 128>>>(dcMesh[i], s.disp.p, nullptr, mw, mh, position[0],
                                                              position[1], position[2], ipd, s.vtx.p, nullptr, nullptr,
                                                              s.flags.p);
      } else {
        rephotoPrepKernel<<<dim3((mw + 127) / 128, mh), 128>>>(dcMesh[i], s.disp.p, s.bgra.p, mw, mh, position[0],
                                                              position[1], position[2], ipd, s.vtx.p, texC, texD,
                                                              s.flags.p);
      }
      for (int l = 1; l < levels; ++l)
        for (int t = 0; t < 2; ++t) {
          ushort4* tex = t == 0 ? texC : texD;
          if (!tex) continue;
          rephotoMipKernel<<<dim3((cv.lw[l] + 127) / 128, cv.lh[l]), 128>>>(tex + cv.lofs[l - 1], cv.lw[l - 1],
                                                                            cv.lh[l - 1], tex + cv.lofs[l], cv.lw[l],
                                                                            cv.lh[l]);
        }
      CU(cudaMemcpy(&cv.anyZeroAlpha, s.flags.p, sizeof(int), cudaMemcpyDeviceToHost));
      CU(cudaMemset(s.keys.p, 0xff, pixels * sizeof(unsigned long long)));
      rephotoRasterKernel<<<dim3((prims + 255) / 256, views), 256>>>(cv, s.mats.p, W, H, prims, s.keys.p);
      rephotoResolveKernel<<<grid1(pixels), 256>>>(cv, s.mats.p, W, H, views, s.keys.p, ps.color ? s.accC.p : nullptr,
                                                   ps.disp ? s.accD.p : nullptr, win ? win + (size_t)i * pixels : nullptr);
      CU(cudaGetLastError());
    }
  }
  std::vector<float> trig;
  if (projection == DERP_CANOPY_EQUIRECT) {  // equirectFS' texel-centre directions, fp64 rounded to fp32
    const int e = outH;
    trig.resize((size_t)6 * e);
    const double kPi = 3.14159265358979323846;
    for (int y = 0; y < e; ++y) {
      const double lat = -(((y + 0.5) / e) - 0.5) * kPi;
      trig[y] = (float)std::cos(lat);
      trig[e + y] = (float)std::sin(lat);
    }
    for (int x = 0; x < 2 * e; ++x) {
      const double lon = (1 - (x + 0.5) / (2 * e)) * 2.0 * kPi;
      trig[2 * e + x] = (float)std::cos(lon);
      trig[4 * e + x] = (float)std::sin(lon);
    }
    if (int rc = upload(s.trig, trig.data(), trig.size())) return rc;
    CU(s.eq.ensure((size_t)2 * e * e * 4));
  }
  for (int t = 0; t < 2; ++t) {
    float* dst = t == 0 ? out_color : out_disparity;
    if (!dst) continue;
    rephotoUnpremulKernel<<<grid1(pixels), 256>>>(pixels, t == 0 ? s.accC.p : s.accD.p, zeroNan, s.out.p);
    CU(cudaGetLastError());
    if (projection == DERP_CANOPY_EQUIRECT) {
      const int e = outH;
      canopyEquirectKernel<<<dim3((2 * e + 127) / 128, e), 128>>>(s.out.p, e, s.trig.p, s.eq.p);
      CU(cudaGetLastError());
      CU(cudaMemcpy(dst, s.eq.p, (size_t)2 * e * e * 4 * sizeof(float), cudaMemcpyDefault));
    } else {
      CU(cudaMemcpy(dst, s.out.p, pixels * 4 * sizeof(float), cudaMemcpyDefault));
    }
  }
  if (winners && num_cams > 0)
    CU(cudaMemcpy(winners, s.win.p, pixels * num_cams * sizeof(int32_t), cudaMemcpyDefault));
  CU(cudaDeviceSynchronize());
  return DERP_OK;
}
}  // namespace

extern "C" {

int derp_rephoto_cubemap(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                         const float* const* colors_bgra, int width, int height, const float* center, int edge,
                         float* out_color, float* out_disparity, int32_t* winners) {
  return canopyRender("derp_rephoto_cubemap", device, cams, num_cams, disparities, width, height, colors_bgra, width, height,
                      DERP_CANOPY_CUBEMAP, center, nullptr, edge, edge, 0.0f, 1, DERP_CANOPY_ON_SCREEN, true, out_color,
                      out_disparity, winners);
}

int derp_canopy_render(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                       int mesh_width, int mesh_height, const float* const* colors_bgra, int color_width,
                       int color_height, int projection, const float* position, const float* matrix, int out_width,
                       int out_height, float ipd, int alpha_blend, int shader, float* out_color, float* out_disparity,
                       int32_t* winners) {
  return canopyRender("derp_canopy_render", device, cams, num_cams, disparities, mesh_width, mesh_height, colors_bgra,
                      color_width, color_height, projection, position, matrix, out_width, out_height, ipd, alpha_blend,
                      shader, false, out_color, out_disparity, winners);
}

int derp_canopy_snapshot_matrix(const float* position, const float* forward, const float* up, double horizontal_fov_deg,
                                int width, int height, float* matrix) {
  if (!position || !forward || !up || !matrix || width < 1 || height < 1)
    return fail(DERP_EINVAL, "derp_canopy_snapshot_matrix: bad arguments");
  if (!derp::rephoto::snapshotMatrix(position, forward, up, horizontal_fov_deg, width, height, matrix))
    return fail(DERP_EINVAL, "derp_canopy_snapshot_matrix: forward and up do not give a unitary basis");
  return DERP_OK;
}

int derp_rephoto_score(int device, const float* ref_bgr, const float* ren_bgr, const uint8_t* mask, int width, int height,
                       int method, int stat_radius, float* score_map, double* avg) {
  using namespace derp::rephoto;
  if (!ref_bgr || !ren_bgr || !mask || width < 1 || height < 1 || !score_map || !avg)
    return fail(DERP_EINVAL, "derp_rephoto_score: bad arguments");
  if (method != DERP_REPHOTO_MSSIM && method != DERP_REPHOTO_NCC)
    return fail(DERP_EINVAL, "derp_rephoto_score: method must be DERP_REPHOTO_MSSIM or DERP_REPHOTO_NCC");
  if (stat_radius < 1 || stat_radius > 31) return fail(DERP_EINVAL, "derp_rephoto_score: stat_radius in [1, 31]");
  CU(cudaSetDevice(device));
  RephotoScratch& s = g_rephoto;
  const size_t pixels = (size_t)width * height, n = pixels * 3;
  // f32 layout: [x | y | mu (2n) | moments (3n) | sig (3n) | tmp (3n) | weights (64)]
  CU(s.f32.ensure(13 * n + 64));
  float *x = s.f32.p, *y = x + n, *mu = y + n, *mom = mu + 2 * n, *sig = mom + 3 * n, *tmp = sig + 3 * n,
        *wt = tmp + 3 * n;
  float hw[64];
  gaussianWeights(stat_radius, hw);
  const unsigned blocks = grid1(pixels);
  CU(s.mask.ensure(pixels));
  CU(s.out.ensure(n));
  CU(s.partial.ensure((size_t)blocks * 6));
  CU(cudaMemcpy(x, ref_bgr, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(y, ren_bgr, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(s.mask.p, mask, pixels, cudaMemcpyDefault));
  CU(cudaMemcpy(wt, hw, (2 * stat_radius + 1) * sizeof(float), cudaMemcpyHostToDevice));
  const dim3 g2((width + 127) / 128, height, 2), g3((width + 127) / 128, height, 3);
  rephotoBlurRowsKernel<<<g2, 128>>>(x, width, height, stat_radius, wt, tmp);  // x, y are adjacent: two images
  rephotoBlurColsKernel<<<g2, 128>>>(tmp, width, height, stat_radius, wt, mu);
  rephotoMomentsKernel<<<grid1(n), 256>>>(n, x, y, mu, mom);
  rephotoBlurRowsKernel<<<g3, 128>>>(mom, width, height, stat_radius, wt, tmp);
  rephotoBlurColsKernel<<<g3, 128>>>(tmp, width, height, stat_radius, wt, sig);
  rephotoScoreKernel<<<blocks, 256>>>(pixels, mu, sig, s.mask.p, method == DERP_REPHOTO_NCC, s.out.p, s.partial.p);
  CU(cudaGetLastError());
  std::vector<double> part((size_t)blocks * 6);
  CU(cudaMemcpy(score_map, s.out.p, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(part.data(), s.partial.p, part.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (int c = 0; c < 3; ++c) {  // cv::mean(channel, mask without NaN): 0 for an empty mask
    double sum = 0, cnt = 0;
    for (unsigned b = 0; b < blocks; ++b) {
      sum += part[b * 6 + c];
      cnt += part[b * 6 + 3 + c];
    }
    avg[c] = cnt > 0 ? sum / cnt : 0.0;
  }
  return DERP_OK;
}

}  // extern "C"
