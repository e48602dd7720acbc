/*
 * derp_canopy.h — C ABI of CanopyScene (source/render/CanopyScene.cpp) on the H100: the renderer SimpleMeshRenderer
 * exports with, in all its modes.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every image pointer may be host or device memory.
 *
 * derp_canopy_render renders CanopyScene(cams, disparities, colors, onScreen = shader == DERP_CANOPY_ON_SCREEN) from
 * `position`.  One canopy per camera, in the order given:
 *   - mesh: vertices camera.rig({x + .5, y + .5}, 1 / disparity) of the camera rescaled to mesh_width x mesh_height
 *     (disparities[i], float [mesh_height][mesh_width]); with ipd != 0, canopyVS' stereo eye offset (positive ipd =
 *     left eye, in metres), computed per vertex about the rig origin.
 *   - colour texture: colors_bgra[i], float B, G, R, A [color_height][color_width] at any size (its alpha is replaced
 *     by the image circle mask at that size, alphaFov).
 *   - disparity-colour texture: disparityColors(metersToGrayscale) about `position` (DisparityColor.h), at the mesh's
 *     size.
 * projection:
 *   - DERP_CANOPY_CUBEMAP: cubemap(out_height, position): faces +X, -X, +Y, -Y, +Z, -Z stacked, out_width = out_height
 *     = edge, output [6 * edge][edge];
 *   - DERP_CANOPY_EQUIRECT: equirect(out_height, position): the cube of edge out_height resampled by equirectFS,
 *     out_width = 2 * out_height, output [out_height][2 * out_height], the +Z row first (no flip, as glReadPixels
 *     leaves it);
 *   - DERP_CANOPY_PERSPECTIVE: one view with the caller's row-major clip matrix (clip = M * (x, y, z, 1); see
 *     derp_canopy_snapshot_matrix), output [out_height][out_width], flipped top row first like the snapshot's cv::flip.
 * alpha_blend: accumulateFS' soft-max weight exp(30 a) - 1 when non-zero, the fragment alpha otherwise.  Outputs are
 * float B, G, R, A, unpremultiplied (rgba / a) with NaN kept where no canopy covers (alpha NaN).  out_color and / or
 * out_disparity may be NULL, not both; colors_bgra may be NULL without out_color.  winners (optional, int32
 * [num_cams][raster rows][raster width]) receives each canopy's surviving primitive per raster pixel, -1 where none, of
 * the colour scene when out_color is given, else of the disparity-colour scene; the raster is the cube (cubemap and
 * equirect, [6 * edge][edge]) or the perspective view.
 * The rasterisation, derivative, filtering and resampling rules are documented in
 * facebook360_dep_b200/csrc/derp_rephoto.cuh.
 *
 * derp_canopy_snapshot_matrix forms SimpleMeshRenderer's snapshot matrix, frustum(-xMax, xMax, -xMax * H / W,
 * xMax * H / W, 0.1) * posForwardUp(position, forward, up), in fp32 as Eigen forms it (row-major, 16 floats); it runs
 * on the host and fails with DERP_EINVAL when forward and up do not give a unitary basis.
 */
#ifndef DERP_CANOPY_H_
#define DERP_CANOPY_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define DERP_CANOPY_CUBEMAP 0
#define DERP_CANOPY_EQUIRECT 1
#define DERP_CANOPY_PERSPECTIVE 2

#define DERP_CANOPY_ON_SCREEN 0 /* canopyFS */
#define DERP_CANOPY_SVD 1       /* canopyFS_SVD, the exporter's */

int derp_canopy_render(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                       int mesh_width, int mesh_height, const float* const* colors_bgra, int color_width,
                       int color_height, int projection, const float* position, const float* matrix, int out_width,
                       int out_height, float ipd, int alpha_blend, int shader, float* out_color, float* out_disparity,
                       int32_t* winners);
int derp_canopy_snapshot_matrix(const float* position, const float* forward, const float* up, double horizontal_fov_deg,
                                int width, int height, float* matrix);

#ifdef __cplusplus
}
#endif
#endif /* DERP_CANOPY_H_ */
