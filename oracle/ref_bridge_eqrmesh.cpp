// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// oracle/_ref/libeqrmesh_ref.so: include/derp_eqrmesh.h over the REFERENCE'S OWN source/render/MeshUtil.h and
// MeshSimplifier.cpp (compiled where they lie under /root/reference, against the stand-ins of refshim/), called in the
// order of CreateObjFromDisparityEquirect.cpp:56-93.  That file is an executable; its dozen lines of glue are restated
// here.  The one step the stand-ins cannot run is the app's cv::resize(disp, disp, Size(), scale, scale) (default
// INTER_LINEAR): cvprims_linear.h, pinned to cv2 4.13, answers for it.  Recipe: eqrmesh.mk.
#include <cstring>
#include <exception>
#include <string>

#include "source/render/MeshSimplifier.h"
#include "source/render/MeshUtil.h"

#include "../include/derp_eqrmesh.h"
#include "cvprims_linear.h"

using namespace fb360_dep;

namespace {

thread_local std::string g_err;

int fail(const std::string& msg) {
  g_err = msg;
  return DERP_EINVAL;
}

template <typename F>
int guarded(F&& f) {
  try {
    return f();
  } catch (const std::exception& e) {
    return fail(e.what());
  }
}

Eigen::MatrixXd toVertexes(const double* xyz, uint64_t nv) {
  Eigen::MatrixXd vertexes((Eigen::Index)nv, 3);
  for (uint64_t i = 0; i < nv; ++i)
    for (int j = 0; j < 3; ++j) vertexes((Eigen::Index)i, j) = xyz[3 * i + j];
  return vertexes;
}
Eigen::MatrixXi toFaces(const uint32_t* idx, uint64_t nf) {
  Eigen::MatrixXi faces((Eigen::Index)nf, 3);
  for (uint64_t i = 0; i < nf; ++i)
    for (int j = 0; j < 3; ++j) faces((Eigen::Index)i, j) = (int)idx[3 * i + j];
  return faces;
}
void fromMesh(const Eigen::MatrixXd& vertexes, const Eigen::MatrixXi& faces, double* xyz, uint32_t* idx, uint64_t* nv,
              uint64_t* nf) {
  for (Eigen::Index i = 0; i < vertexes.rows(); ++i)
    for (int j = 0; j < 3; ++j) xyz[3 * i + j] = vertexes(i, j);
  for (Eigen::Index i = 0; i < faces.rows(); ++i)
    for (int j = 0; j < 3; ++j) idx[3 * i + j] = (uint32_t)faces(i, j);
  *nv = (uint64_t)vertexes.rows();
  *nf = (uint64_t)faces.rows();
}

int equirectMeshRef(const float* disparity, int width, int height, double scale, double max_depth, float tear_ratio,
                    int num_faces, float strictness, double* vertexesOut, uint32_t* facesOut, uint64_t* nvOut,
                    uint64_t* nfOut) {
  int W = 0, H = 0;
  if (!oracle::equirectGrid(width, height, scale, &W, &H) || !disparity || !vertexesOut || !facesOut || !nvOut || !nfOut ||
      !(0 <= strictness && strictness <= 1))
    return fail("bad arguments");
  return guarded([&] {
    cv::Mat_<float> disp(height, width);
    std::memcpy(disp.data, disparity, (size_t)width * height * sizeof(float));
    if (scale < 1) {  // cv::resize(disp, disp, cv::Size(), scale, scale)
      std::vector<float> small;
      oracle::resizeLinearScaledF32(disparity, width, height, scale, small, &W, &H);
      disp = cv::Mat_<float>(H, W);
      std::memcpy(disp.data, small.data(), small.size() * sizeof(float));
    }
    Eigen::MatrixXd vertexes = mesh_util::getVertexesEquirect(disp, max_depth);
    Eigen::MatrixXi faces = mesh_util::getFaces(vertexes, disp.cols, disp.rows, true, true, tear_ratio);
    if (strictness > 0) {
      render::MeshSimplifier ms(vertexes, faces, false, 1);
      ms.simplify(num_faces, strictness);
      vertexes = ms.getVertexes();
      faces = ms.getFaces();
    }
    fromMesh(vertexes, faces, vertexesOut, facesOut, nvOut, nfOut);
    return (int)DERP_OK;
  });
}

}  // namespace

extern "C" {

const char* derp_last_error(void) { return g_err.c_str(); }

int derp_equirect_mesh_size(int width, int height, double scale, int* mesh_width, int* mesh_height) {
  if (!mesh_width || !mesh_height || !oracle::equirectGrid(width, height, scale, mesh_width, mesh_height))
    return fail("bad arguments");
  return DERP_OK;
}

int derp_equirect_mesh(int /*device*/, const float* disparity, int width, int height, double scale, double max_depth,
                       float tear_ratio, double* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces) {
  return equirectMeshRef(disparity, width, height, scale, max_depth, tear_ratio, 0, 0.f, vertexes, faces, num_vertexes,
                         num_faces);
}

int derp_equirect_mesh_simplified(int /*device*/, const float* disparity, int width, int height, double scale,
                                  double max_depth, float tear_ratio, int num_faces, float strictness, double* vertexes,
                                  uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces_out) {
  return equirectMeshRef(disparity, width, height, scale, max_depth, tear_ratio, num_faces, strictness, vertexes, faces,
                         num_vertexes, num_faces_out);
}

/* test hook: MeshSimplifier(v, f, isEquiError = false, 1).simplify(triangles, strictness) on an arbitrary mesh */
int derp_ref_simplify_relative(const double* xyz, uint64_t nv, const uint32_t* idx, uint64_t nf, int triangles,
                               float strictness, double* out_xyz, uint32_t* out_idx, uint64_t* out_nv, uint64_t* out_nf) {
  return guarded([&] {
    render::MeshSimplifier ms(toVertexes(xyz, nv), toFaces(idx, nf), false, 1);
    ms.simplify(triangles, strictness);
    fromMesh(ms.getVertexes(), ms.getFaces(), out_xyz, out_idx, out_nv, out_nf);
    return (int)DERP_OK;
  });
}

/* test hook: mesh_util::addTextureCoordinatesEquirect + writeObj(vertexes, faces, obj, mtl) (MeshUtil.h:91-129, 408-418)
 * with writeMtl(obj, color) (MeshUtil.h:131-144) when color is not null: the files the app means to write */
int derp_ref_write_obj(const double* xyz, uint64_t nv, const uint32_t* idx, uint64_t nf, const char* obj,
                       const char* color) {
  return guarded([&] {
    Eigen::MatrixXd vertexes = toVertexes(xyz, nv);
    std::string fnMtl;
    if (color) {
      mesh_util::addTextureCoordinatesEquirect(vertexes);
      fnMtl = mesh_util::writeMtl(obj, color);
    }
    mesh_util::writeObj(vertexes, toFaces(idx, nf), obj, fnMtl);
    return (int)DERP_OK;
  });
}

}  // extern "C"
