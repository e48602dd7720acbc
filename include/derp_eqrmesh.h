/*
 * derp_eqrmesh.h — C ABI of the equirect mesh of CreateObjFromDisparityEquirect
 * (source/conversion/CreateObjFromDisparityEquirect.cpp) on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every pointer may be host or device memory.  The camera mesh of ConvertToBinary
 * (derp_camera_mesh*) is in derp_b200.h; both meshes run on the same kernels (csrc/derp_mesh.cuh).
 *
 * derp_equirect_mesh: the app's mesh of a disparity equirect (CreateObjFromDisparityEquirect.cpp:56-71).  For
 * scale < 1, cv::resize(disp, disp, Size(), scale, scale) with INTER_LINEAR (grid cvRound(size * scale);
 * derp_equirect_mesh_size gives it); then mesh_util::getVertexesEquirect(disp, (float)max_depth)
 * (source/render/MeshUtil.h:298-313: depth = fmin(max_depth, 1 / disparity), so NaN and 0 disparities sit at max_depth)
 * and mesh_util::getFaces(wrapHorizontally = true, isRigCoordinates = true, tear_ratio) (MeshUtil.h:264-296: the corner
 * distance is the vertex's norm; two faces per row pair join the last and the first column after all quad faces).
 * Outputs in the reference's order: fp64 x, y, z per vertex (what mesh_util::writeObj prints) and uint32 x 3 per face.
 * `vertexes` needs room for 3 doubles per grid cell, `faces` for 6 uint32 per grid cell.
 *
 * derp_equirect_mesh_simplified: the same, then the app's simplification when strictness > 0:
 * render::MeshSimplifier(vertexes, faces, isEquiError = false, threads).simplify(num_faces, strictness)
 * (source/render/MeshSimplifier.cpp; costs divided by the squared norm of the contraction target), on the host inside
 * the library like derp_camera_mesh_simplified.  The reference's thread count only splits per-face work and does not
 * change the result.  strictness 0 gives the plain mesh.
 *
 * Refused with DERP_EINVAL: scale <= 0 or NaN (OpenCV throws on the empty size), a grid narrower or lower than 2 cells
 * (no quads, and the wrap would join a column to itself), strictness outside [0, 1] (the app's CHECK), 2^31 faces or
 * more.
 */
#ifndef DERP_EQRMESH_H_
#define DERP_EQRMESH_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int derp_equirect_mesh_size(int width, int height, double scale, int* mesh_width, int* mesh_height);
int derp_equirect_mesh(int device, const float* disparity, int width, int height, double scale, double max_depth,
                       float tear_ratio, double* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces);
int derp_equirect_mesh_simplified(int device, const float* disparity, int width, int height, double scale,
                                  double max_depth, float tear_ratio, int num_faces, float strictness, double* vertexes,
                                  uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces_out);

#ifdef __cplusplus
}
#endif
#endif /* DERP_EQRMESH_H_ */
