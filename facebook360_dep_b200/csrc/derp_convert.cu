// derp_camera_mesh* and derp_bc7_compress* (include/derp_b200.h): the geometry and the colour of ConvertToBinary on
// sm_90a (derp_mesh.cuh, derp_bc7.cuh); derp_equirect_mesh* (include/derp_eqrmesh.h): the mesh of
// CreateObjFromDisparityEquirect on the same mesh kernels; and the host hooks of the simplifier and the BC7 encoder.
#include <cfloat>
#include <cmath>
#include <cstring>

#include "derp_host.cuh"
#include "derp_mesh.cuh"
#include "derp_simplify.h"
#include "derp_bc7.cuh"
#include "../../include/derp_eqrmesh.h"

using namespace derp;

extern "C" {

// cv::resize(depth, depth, Size(), s, s, INTER_NEAREST) (ConvertToBinary.cpp:153-156): dsize = cvRound(size * s),
// source index = min(floor(d * (1 / s)), size - 1) (resize.cpp resizeNN with the caller's scale factors)
static void meshAxis(int sn, double scale, std::vector<int>& ofs) {
  if (!(scale < 1)) {
    ofs.resize(sn);
    for (int d = 0; d < sn; ++d) ofs[d] = d;
    return;
  }
  const int dn = (int)std::nearbyint(sn * scale);
  const double ifx = 1. / scale;
  ofs.resize(std::max(dn, 0));
  for (int d = 0; d < dn; ++d) ofs[d] = std::min(floorD(d * ifx), sn - 1);
}

int derp_camera_mesh_size(int width, int height, double depth_scale, int* mesh_width, int* mesh_height) {
  if (width < 1 || height < 1 || !(depth_scale > 0) || depth_scale > 1 || !mesh_width || !mesh_height)
    return fail(DERP_EINVAL, "derp_camera_mesh_size: bad arguments (depth_scale in (0, 1], ConvertToBinary.cpp:348)");
  *mesh_width = depth_scale < 1 ? (int)std::nearbyint(width * depth_scale) : width;
  *mesh_height = depth_scale < 1 ? (int)std::nearbyint(height * depth_scale) : height;
  return DERP_OK;
}

static int cameraMesh(int device, const float* disparity, int width, int height, double depth_scale, double resolution_x,
                      double resolution_y, double scalar_focal, float tear_ratio, const uint8_t* foreground_mask,
                      int mask_width, int mask_height, int triangles, float* vertexes, uint32_t* faces,
                      uint64_t* num_vertexes, uint64_t* num_faces) {
  int W = 0, H = 0;
  int rc = derp_camera_mesh_size(width, height, depth_scale, &W, &H);
  if (rc) return rc;
  if (!disparity || !vertexes || !faces || !num_vertexes || !num_faces || W < 1 || H < 1 ||
      (foreground_mask && (mask_width < 1 || mask_height < 1)))
    return fail(DERP_EINVAL, "derp_camera_mesh: bad arguments");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)W * H, nsrc = (size_t)width * height;
  if (n >= (1ull << 31)) return fail(DERP_EINVAL, "derp_camera_mesh: grid too large for 32-bit indexes");
  std::vector<int> ofs, tmp;
  meshAxis(width, depth_scale, ofs);
  meshAxis(height, depth_scale, tmp);
  ofs.insert(ofs.end(), tmp.begin(), tmp.end());
  if (foreground_mask) {  // cv::resize(mask, mask, depth.size(), 0, 0, INTER_NEAREST), ConvertToBinary.cpp:171-174
    nearestAxis(mask_width, W, tmp);
    ofs.insert(ofs.end(), tmp.begin(), tmp.end());
    nearestAxis(mask_height, H, tmp);
    ofs.insert(ofs.end(), tmp.begin(), tmp.end());
  }
  // grow-only scratch per host thread (the app converts one (frame, camera) after the other on each GPU worker thread)
  struct MeshScratch {
    DevBuf<float> dDisp, dVtx;
    DevBuf<double> dVtx64;
    DevBuf<int> dOfs;
    DevBuf<uint8_t> dFg, dQuad, dUsed;
    DevBuf<unsigned> dTiles, dIndex, dFaces;
    DevBuf<unsigned long long> dTotals;
  };
  static thread_local MeshScratch sc;
  DevBuf<float>&dDisp = sc.dDisp, &dVtx = sc.dVtx;
  DevBuf<int>& dOfs = sc.dOfs;
  DevBuf<uint8_t>&dFg = sc.dFg, &dQuad = sc.dQuad, &dUsed = sc.dUsed;
  DevBuf<unsigned>&dTiles = sc.dTiles, &dIndex = sc.dIndex, &dFaces = sc.dFaces;
  DevBuf<unsigned long long>& dTotals = sc.dTotals;
  const float* disp = disparity;
  const uint8_t* fg = foreground_mask;
  if ((rc = stageIn(disp, nsrc, dDisp))) return rc;
  if (fg && (rc = stageIn(fg, (size_t)mask_width * mask_height, dFg))) return rc;
  const int tiles = (int)((n + kScanTile - 1) / kScanTile);
  if ((rc = upload(dOfs, ofs.data(), ofs.size()))) return rc;
  CU(dQuad.ensure(n));
  CU(dUsed.ensure(n));
  CU(dTiles.ensure(2 * (size_t)tiles));
  CU(dIndex.ensure(n));
  CU(dTotals.ensure(2));
  CU(cudaMemset(dUsed.p, 0, n));
  MeshGrid g;
  g.W = W;
  g.H = H;
  g.srcW = width;
  g.disp = disp;
  g.xofs = dOfs.p;
  g.yofs = dOfs.p + W;
  g.fg = fg;
  g.fgW = mask_width;
  g.fgx = dOfs.p + W + H;
  g.fgy = dOfs.p + 2 * (size_t)W + H;
  g.stepX = resolution_x / W;
  g.stepY = resolution_y / H;
  g.scale = scalar_focal * 1.0;  // kRadius = 1 (MeshUtil.h:316)
  g.tearRatio = tear_ratio;
  g.floorZ = 0;
  meshQuadKernel<<<grid2(W, H), block2()>>>(g, dQuad.p, dUsed.p);
  meshTileCountKernel<true><<<tiles, kScanThreads>>>(n, dQuad.p, dUsed.p, dTiles.p, dTiles.p + tiles);
  meshTileScanKernel<<<1, kScanThreads>>>(tiles, dTiles.p, dTiles.p + tiles, dTotals.p);
  CU(cudaGetLastError());
  unsigned long long totals[2] = {0, 0};
  CU(cudaMemcpy(totals, dTotals.p, sizeof(totals), cudaMemcpyDeviceToHost));
  if (triangles > 0 && totals[0] > (unsigned long long)triangles) {
    // Simplification (ConvertToBinary.cpp:186-203): the mesh in double precision goes to the host, where the strictly
    // sequential edge-contraction sweeps run (derp_simplify.h), like MeshSimplifier with kThreads = 1 in the reference.
    DevBuf<double>& dVtx64 = sc.dVtx64;
    CU(dVtx64.ensure(std::max<size_t>(1, totals[1] * 3)));
    CU(dFaces.ensure(std::max<size_t>(1, totals[0] * 3)));
    g.floorZ = 0;  // the simplifier works on the raw values; the floor is applied to its output below
    meshEmitVertexesKernel<double><<<tiles, kScanThreads>>>(g, dUsed.p, dTiles.p + tiles, dIndex.p, dVtx64.p);
    meshEmitFacesKernel<true><<<tiles, kScanThreads>>>(W, n, dQuad.p, dTiles.p, dIndex.p, dFaces.p);
    CU(cudaGetLastError());
    std::vector<double> hv(totals[1] * 3);
    std::vector<uint32_t> hf(totals[0] * 3);
    CU(cudaMemcpy(hv.data(), dVtx64.p, hv.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(hf.data(), dFaces.p, hf.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    simplify::Mesh mesh(hv.data(), totals[1], hf.data(), totals[0]);
    mesh.run(triangles, 0.2f, false);  // kStrictness, kRemoveBoundaryEdges (ConvertToBinary.cpp:193-195)
    std::vector<float> ov(mesh.verts.size() * 3);
    std::vector<uint32_t> of(mesh.faces.size() * 3);
    for (size_t i = 0; i < mesh.verts.size(); ++i) {
      const simplify::V3& p = mesh.verts[i].p;
      ov[3 * i] = (float)p.x;
      ov[3 * i + 1] = (float)p.y;
      ov[3 * i + 2] = (float)(p.z < 0 ? (double)FLT_MIN : p.z);  // ConvertToBinary.cpp:199-203
    }
    for (size_t i = 0; i < mesh.faces.size(); ++i)
      for (int j = 0; j < 3; ++j) of[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
    CU(cudaMemcpy(vertexes, ov.data(), ov.size() * sizeof(float), cudaMemcpyDefault));
    CU(cudaMemcpy(faces, of.data(), of.size() * sizeof(uint32_t), cudaMemcpyDefault));
    *num_vertexes = mesh.verts.size();
    *num_faces = mesh.faces.size();
    return DERP_OK;
  }
  g.floorZ = triangles > 0;  // the reference applies it after the (here: no-op) simplification
  // outputs: written in place when the caller's buffers are device memory, else staged
  float* vtx = vertexes;
  uint32_t* fac = faces;
  if ((rc = outBuffer(vtx, totals[1] * 3, dVtx)) || (rc = outBuffer(fac, totals[0] * 3, dFaces))) return rc;
  meshEmitVertexesKernel<float><<<tiles, kScanThreads>>>(g, dUsed.p, dTiles.p + tiles, dIndex.p, vtx);
  meshEmitFacesKernel<true><<<tiles, kScanThreads>>>(W, n, dQuad.p, dTiles.p, dIndex.p, fac);
  CU(cudaGetLastError());
  if ((rc = stageOut(vertexes, vtx, totals[1] * 3)) || (rc = stageOut(faces, fac, totals[0] * 3))) return rc;
  CU(cudaDeviceSynchronize());
  *num_faces = totals[0];
  *num_vertexes = totals[1];
  return DERP_OK;
}

int derp_camera_mesh(int device, const float* disparity, int width, int height, double depth_scale, double resolution_x,
                     double resolution_y, double scalar_focal, float tear_ratio, const uint8_t* foreground_mask,
                     int mask_width, int mask_height, float* vertexes, uint32_t* faces, uint64_t* num_vertexes,
                     uint64_t* num_faces) {
  return cameraMesh(device, disparity, width, height, depth_scale, resolution_x, resolution_y, scalar_focal, tear_ratio,
                    foreground_mask, mask_width, mask_height, 0, vertexes, faces, num_vertexes, num_faces);
}

int derp_camera_mesh_simplified(int device, const float* disparity, int width, int height, double depth_scale,
                                double resolution_x, double resolution_y, double scalar_focal, float tear_ratio,
                                const uint8_t* foreground_mask, int mask_width, int mask_height, int triangles,
                                float* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces) {
  return cameraMesh(device, disparity, width, height, depth_scale, resolution_x, resolution_y, scalar_focal, tear_ratio,
                    foreground_mask, mask_width, mask_height, triangles, vertexes, faces, num_vertexes, num_faces);
}

// ---- equirect mesh (CreateObjFromDisparityEquirect) ----
// cv::resize(disp, disp, Size(), scale, scale) (INTER_LINEAR), CreateObjFromDisparityEquirect.cpp:59-62: the grid is
// cvRound(size * scale) when scale < 1, the input size otherwise.  scale <= 0 (or NaN) is refused: OpenCV throws on the
// empty size; so is a grid narrower or lower than 2 (a row has no quads and getFaces' wrap joins a column to itself).
int derp_equirect_mesh_size(int width, int height, double scale, int* mesh_width, int* mesh_height) {
  if (width < 1 || height < 1 || !(scale > 0) || !mesh_width || !mesh_height)
    return fail(DERP_EINVAL, "derp_equirect_mesh_size: bad arguments (scale > 0)");
  const int w = scale < 1 ? (int)std::nearbyint(width * scale) : width;
  const int h = scale < 1 ? (int)std::nearbyint(height * scale) : height;
  if (w < 2 || h < 2) return fail(DERP_EINVAL, "derp_equirect_mesh_size: the mesh grid must be at least 2 x 2");
  if ((size_t)w * h * 2 >= (1ull << 31)) return fail(DERP_EINVAL, "derp_equirect_mesh_size: grid too large for 32-bit indexes");
  *mesh_width = w;
  *mesh_height = h;
  return DERP_OK;
}

// INTER_LINEAR taps of one axis for the scale factor f (see LinearTaps in derp_mesh.cuh): position (d + 0.5) / f - 0.5 in
// double, weight float(position - floor); columns clamp the left edge and copy at the right edge, rows clamp the index only
static void linearAxis(int sn, int dn, double f, bool column, std::vector<int>& ofs, std::vector<uint8_t>& copy,
                       std::vector<float>& w) {
  const double inv = 1. / f;
  ofs.clear(), copy.clear(), w.clear();
  for (int d = 0; d < dn; ++d) {
    const double p = (d + 0.5) * inv - 0.5;
    int s = floorD(p);
    float a = (float)(p - s);
    if (column) {
      if (s < 0) s = 0, a = 0.f;
      copy.push_back(s + 1 >= sn);
      ofs.push_back(s + 1 >= sn ? sn - 1 : s);
    } else {
      ofs.push_back(std::min(std::max(s, 0), sn - 1));
      ofs.push_back(std::min(std::max(s + 1, 0), sn - 1));
    }
    w.push_back(1.f - a);
    w.push_back(a);
  }
}

// sin / cos of getVertexesEquirect's angles (MeshUtil.h:304-307) with the host's C library: theta of every column
// (u = float(x + 0.5) / float(W), theta = float(u * 2.0f * M_PI)), phi of every row
static void eqrAngles(int W, int H, std::vector<float>& t) {
  t.resize(2 * (size_t)W + 2 * (size_t)H);
  for (int x = 0; x < W; ++x) {
    const float u = float(x + 0.5) / float(W);
    const float theta = u * 2.0f * M_PI;
    t[x] = sinf(theta);
    t[W + x] = cosf(theta);
  }
  for (int y = 0; y < H; ++y) {
    const float v = float(y + 0.5) / float(H);
    const float phi = v * M_PI;
    t[2 * W + y] = sinf(phi);
    t[2 * W + H + y] = cosf(phi);
  }
}

static int equirectMesh(int device, const float* disparity, int width, int height, double scale, double max_depth,
                        float tear_ratio, int num_faces, float strictness, double* vertexes, uint32_t* faces,
                        uint64_t* num_vertexes, uint64_t* num_faces_out) {
  int W = 0, H = 0;
  int rc = derp_equirect_mesh_size(width, height, scale, &W, &H);
  if (rc) return rc;
  if (!disparity || !vertexes || !faces || !num_vertexes || !num_faces_out || !(strictness >= 0 && strictness <= 1))
    return fail(DERP_EINVAL, "derp_equirect_mesh: bad arguments (strictness in [0, 1])");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)W * H, nsrc = (size_t)width * height;
  const size_t maxFaces = 2 * (size_t)W * (H - 1);  // getFaces' allocation (MeshUtil.h:271)
  struct EqrScratch {
    DevBuf<float> dDisp, dSmall, dTables, dAngles;
    DevBuf<double> dVtx;
    DevBuf<int> dOfs;
    DevBuf<uint8_t> dCopy, dQuad;
    DevBuf<unsigned> dTiles, dFaces;
    DevBuf<unsigned long long> dTotals;
  };
  static thread_local EqrScratch sc;
  const float* disp = disparity;
  if ((rc = stageIn(disp, nsrc, sc.dDisp))) return rc;
  if (W != width || H != height) {  // --scale < 1
    std::vector<int> xo, yo;
    std::vector<uint8_t> xc, unused;
    std::vector<float> xw, yw;
    linearAxis(width, W, scale, true, xo, xc, xw);
    linearAxis(height, H, scale, false, yo, unused, yw);
    xo.insert(xo.end(), yo.begin(), yo.end());
    xw.insert(xw.end(), yw.begin(), yw.end());
    if ((rc = upload(sc.dOfs, xo.data(), xo.size())) || (rc = upload(sc.dCopy, xc.data(), xc.size())) ||
        (rc = upload(sc.dTables, xw.data(), xw.size())))
      return rc;
    CU(sc.dSmall.ensure(n));
    const LinearTaps t{sc.dOfs.p, sc.dCopy.p, sc.dTables.p, sc.dOfs.p + W, sc.dTables.p + 2 * (size_t)W};
    resizeLinearKernel<<<grid2(W, H), block2()>>>(disp, width, t, W, H, sc.dSmall.p);
    CU(cudaGetLastError());
    disp = sc.dSmall.p;
  }
  std::vector<float> angles;
  eqrAngles(W, H, angles);
  const bool simplify = strictness > 0;
  // the vertexes go straight to the caller's buffer when it is device memory and nothing is simplified
  double* vtx = vertexes;
  if (simplify) {
    CU(sc.dVtx.ensure(n * 3));
    vtx = sc.dVtx.p;
  } else if ((rc = outBuffer(vtx, n * 3, sc.dVtx))) {
    return rc;
  }
  DevBuf<float>& dAngles = sc.dAngles;
  if ((rc = upload(dAngles, angles.data(), angles.size()))) return rc;
  eqrVertexKernel<<<grid2(W, H), block2()>>>(W, H, disp, (float)max_depth, dAngles.p, dAngles.p + W,
                                             dAngles.p + 2 * W, dAngles.p + 2 * W + H, vtx);
  const int tiles = (int)((n + kScanTile - 1) / kScanTile);
  CU(sc.dQuad.ensure(n));
  CU(sc.dTiles.ensure(2 * (size_t)tiles));
  CU(sc.dTotals.ensure(2));
  EqrGrid g{W, H, vtx, tear_ratio};
  meshQuadKernel<<<grid2(W, H), block2()>>>(g, sc.dQuad.p, nullptr);
  meshTileCountKernel<false><<<tiles, kScanThreads>>>(n, sc.dQuad.p, nullptr, sc.dTiles.p, sc.dTiles.p + tiles);
  meshTileScanKernel<<<1, kScanThreads>>>(tiles, sc.dTiles.p, sc.dTiles.p + tiles, sc.dTotals.p);
  CU(cudaGetLastError());
  unsigned long long totals[2] = {0, 0};
  CU(cudaMemcpy(totals, sc.dTotals.p, sizeof(totals), cudaMemcpyDeviceToHost));
  const size_t nf = totals[0] + 2 * (size_t)(H - 1);
  uint32_t* fac = faces;
  if (simplify) {
    CU(sc.dFaces.ensure(nf * 3));
    fac = sc.dFaces.p;
  } else if ((rc = outBuffer(fac, maxFaces * 3, sc.dFaces))) {
    return rc;
  }
  meshEmitFacesKernel<false><<<tiles, kScanThreads>>>(W, n, sc.dQuad.p, sc.dTiles.p, nullptr, fac);
  eqrWrapFacesKernel<<<(H - 1 + 255) / 256, 256>>>(W, H, totals[0], fac);
  CU(cudaGetLastError());
  if (simplify) {
    // MeshSimplifier(vertexes, faces, kIsEquiError = false, threads).simplify(num_faces, strictness), on the host
    // (derp_simplify.h); the reference's thread count only splits per-face work and does not change the result
    std::vector<double> hv(n * 3);
    std::vector<uint32_t> hf(nf * 3);
    CU(cudaMemcpy(hv.data(), vtx, hv.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(hf.data(), fac, hf.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    simplify::Mesh mesh(hv.data(), n, hf.data(), nf, false);
    mesh.run(num_faces, strictness, false);
    hv.resize(mesh.verts.size() * 3);
    hf.resize(mesh.faces.size() * 3);
    for (size_t i = 0; i < mesh.verts.size(); ++i) {
      hv[3 * i] = mesh.verts[i].p.x;
      hv[3 * i + 1] = mesh.verts[i].p.y;
      hv[3 * i + 2] = mesh.verts[i].p.z;
    }
    for (size_t i = 0; i < mesh.faces.size(); ++i)
      for (int j = 0; j < 3; ++j) hf[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
    CU(cudaMemcpy(vertexes, hv.data(), hv.size() * sizeof(double), cudaMemcpyDefault));
    CU(cudaMemcpy(faces, hf.data(), hf.size() * sizeof(uint32_t), cudaMemcpyDefault));
    *num_vertexes = mesh.verts.size();
    *num_faces_out = mesh.faces.size();
    return DERP_OK;
  }
  if ((rc = stageOut(vertexes, vtx, n * 3)) || (rc = stageOut(faces, fac, nf * 3))) return rc;
  CU(cudaDeviceSynchronize());
  *num_vertexes = n;
  *num_faces_out = nf;
  return DERP_OK;
}

int derp_equirect_mesh(int device, const float* disparity, int width, int height, double scale, double max_depth,
                       float tear_ratio, double* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces) {
  return equirectMesh(device, disparity, width, height, scale, max_depth, tear_ratio, 0, 0.f, vertexes, faces,
                      num_vertexes, num_faces);
}

int derp_equirect_mesh_simplified(int device, const float* disparity, int width, int height, double scale,
                                  double max_depth, float tear_ratio, int num_faces, float strictness, double* vertexes,
                                  uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces_out) {
  return equirectMesh(device, disparity, width, height, scale, max_depth, tear_ratio, num_faces, strictness, vertexes,
                      faces, num_vertexes, num_faces_out);
}

// ---- BC7 colour (ConvertToBinary's default colour format) ----
static int bc7Launch(int device, const void* src, size_t srcBytes, int mode, int channels, int width, int height,
                     const uint8_t* lutHost, size_t lutBytes, uint8_t* blocks) {
  CU(cudaSetDevice(device));
  const size_t outBytes = (size_t)width * height;
  // grow-only scratch per host thread (the app converts one (frame, camera) after the other on each GPU worker thread)
  static thread_local struct {
    DevBuf<uint8_t> dSrc, dOut, dLut;
  } sc;
  // 16-byte alignment: the RGBA source is read and the blocks are written as uint4
  const uint8_t* s = static_cast<const uint8_t*>(src);
  uint8_t* o = blocks;
  int rc = stageIn(s, srcBytes, sc.dSrc, 16);
  if (rc || (rc = outBuffer(o, outBytes, sc.dOut, 16))) return rc;
  CU(cudaMemset(o, 0, outBytes));  // the reference's output vector starts zeroed; partial edge blocks are never written
  const int bx = width / 4, by = height / 4;
  if (bx > 0 && by > 0) {
    const unsigned grid = (unsigned)(((size_t)bx * by + derp::bc7::kBc7Threads - 1) / derp::bc7::kBc7Threads);
    if (mode == 0) {
      derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(derp::bc7::Rgba8Source{(const uint8_t*)s, width}, width, bx, by, o);
    } else {
      if ((rc = upload(sc.dLut, lutHost, lutBytes))) return rc;
      if (mode == 8)
        derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(
            derp::bc7::BgrSource<uint8_t>{(const uint8_t*)s, width, channels, sc.dLut.p}, width, bx, by, o);
      else
        derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(
            derp::bc7::BgrSource<uint16_t>{(const uint16_t*)s, width, channels, sc.dLut.p}, width, bx, by, o);
    }
    CU(cudaGetLastError());
  }
  if ((rc = stageOut(blocks, o, outBytes))) return rc;
  CU(cudaDeviceSynchronize());  // return with blocks written, also when a staged copy goes to another GPU
  return DERP_OK;
}

int derp_bc7_compress(int device, const uint8_t* rgba, int width, int height, uint8_t* blocks) {
  if (!rgba || !blocks || width < 1 || height < 1) return fail(DERP_EINVAL, "derp_bc7_compress: bad arguments");
  return bc7Launch(device, rgba, (size_t)width * height * 4, 0, 4, width, height, nullptr, 0, blocks);
}

int derp_bc7_compress_image(int device, const void* pixels, int bits_per_channel, int channels, int width, int height,
                            float gamma, uint8_t* blocks) {
  if (!pixels || !blocks || width < 1 || height < 1 || (bits_per_channel != 8 && bits_per_channel != 16) ||
      (channels != 3 && channels != 4))
    return fail(DERP_EINVAL, "derp_bc7_compress_image: 8 or 16 bits per channel, 3 (BGR) or 4 (BGRA) channels");
  std::vector<uint8_t> lut((size_t)1 << bits_per_channel);
  derp::bc7::gammaTable(bits_per_channel, gamma, lut.data());
  return bc7Launch(device, pixels, (size_t)width * height * channels * (bits_per_channel / 8), bits_per_channel, channels,
                   width, height, lut.data(), lut.size(), blocks);
}

// host-only hook for tests/test_mesh.py: the simplifier on an arbitrary mesh (double xyz, uint32 indices); outputs sized
// like the inputs
int derp_test_simplify(const double* xyz, uint64_t nv, const uint32_t* idx, uint64_t nf, int triangles, float strictness,
                       int remove_boundary_edges, double* out_xyz, uint32_t* out_idx, uint64_t* out_nv, uint64_t* out_nf) {
  derp::simplify::Mesh mesh(xyz, nv, idx, nf);
  mesh.run(triangles, strictness, remove_boundary_edges != 0);
  for (size_t i = 0; i < mesh.verts.size(); ++i) {
    out_xyz[3 * i] = mesh.verts[i].p.x;
    out_xyz[3 * i + 1] = mesh.verts[i].p.y;
    out_xyz[3 * i + 2] = mesh.verts[i].p.z;
  }
  for (size_t i = 0; i < mesh.faces.size(); ++i)
    for (int j = 0; j < 3; ++j) out_idx[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
  *out_nv = mesh.verts.size();
  *out_nf = mesh.faces.size();
  return 0;
}

// host-only hook for tests/test_eqr_obj.py: the simplifier with MeshSimplifier's relative cost (isEquiError = false)
int derp_test_simplify_relative(const double* xyz, uint64_t nv, const uint32_t* idx, uint64_t nf, int triangles,
                                float strictness, double* out_xyz, uint32_t* out_idx, uint64_t* out_nv,
                                uint64_t* out_nf) {
  derp::simplify::Mesh mesh(xyz, nv, idx, nf, false);
  mesh.run(triangles, strictness, false);
  for (size_t i = 0; i < mesh.verts.size(); ++i) {
    out_xyz[3 * i] = mesh.verts[i].p.x;
    out_xyz[3 * i + 1] = mesh.verts[i].p.y;
    out_xyz[3 * i + 2] = mesh.verts[i].p.z;
  }
  for (size_t i = 0; i < mesh.faces.size(); ++i)
    for (int j = 0; j < 3; ++j) out_idx[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
  *out_nv = mesh.verts.size();
  *out_nf = mesh.faces.size();
  return 0;
}

// HOST instantiation of resizeLinearKernel's per-pixel function (derp_mesh.cuh) for tests/test_eqr_obj.py -m "not gpu":
// cv::resize(src, dst, Size(), scale, scale) with INTER_LINEAR; dst holds the derp_equirect_mesh_size grid
int derp_test_resize_linear_host(const float* src, int width, int height, double scale, float* dst) {
  int W = 0, H = 0;
  if (!src || !dst || derp_equirect_mesh_size(width, height, scale, &W, &H)) return DERP_EINVAL;
  if (W == width && H == height) {
    std::memcpy(dst, src, (size_t)W * H * sizeof(float));
    return DERP_OK;
  }
  std::vector<int> xo, yo;
  std::vector<uint8_t> xc, unused;
  std::vector<float> xw, yw;
  linearAxis(width, W, scale, true, xo, xc, xw);
  linearAxis(height, H, scale, false, yo, unused, yw);
  const LinearTaps t{xo.data(), xc.data(), xw.data(), yo.data(), yw.data()};
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) dst[(size_t)y * W + x] = linearPixel(src, width, t, x, y);
  return DERP_OK;
}

// HOST instantiation of the BC7 block encoder (derp_bc7.cuh) for tests/test_bc7.py -m "not gpu"; the apps call
// derp_bc7_compress* (CUDA) only.
int derp_test_bc7_blocks_host(const uint8_t* rgba, int width, int height, uint8_t* blocks) {
  if (!rgba || !blocks || width < 1 || height < 1) return DERP_EINVAL;
  std::memset(blocks, 0, (size_t)width * height);
  derp::bc7::encodeSurfaceOnHost(rgba, width, height, blocks);
  return DERP_OK;
}
int derp_test_bc7_gamma_table(int bits_per_channel, float gamma, uint8_t* lut) {
  if ((bits_per_channel != 8 && bits_per_channel != 16) || !lut) return DERP_EINVAL;
  derp::bc7::gammaTable(bits_per_channel, gamma, lut);
  return DERP_OK;
}

}  // extern "C"
