/*
 * derp_rephoto.h — C ABI of rephotography (source/render/ComputeRephotographyErrors.cpp) on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every image pointer may be host or device memory.
 *
 * derp_rephoto_cubemap renders CanopyScene(cams, disparities, colors).cubemap(edge, center) (CanopyScene.cpp:329-413) in
 * the one mode the app uses: ipd = 0, alphaBlend = true, fragment shader canopyFS.  One canopy per camera, in the order
 * given: mesh vertices camera.rig({x + .5, y + .5}, 1 / disparity) of the camera rescaled to width x height, the texture
 * colors_bgra[i] (float B, G, R, A [height][width], already at the disparity's size; its alpha is replaced by the image
 * circle mask, alphaFov).  Cubemap faces +X, -X, +Y, -Y, +Z, -Z stacked vertically, each edge x edge, top row first:
 * float B, G, R, A [6 * edge][edge], NaN set to 0 (zeroOutNans).  out_color receives the colour cubemap; out_disparity the
 * cubemap of disparityColors(metersToGrayscale) about `center` (DisparityColor.h), which shares the colour cubemap's
 * geometry, so one raster serves both (either may be NULL, colors_bgra may be NULL without out_color).  winners
 * (optional, int32 [num_cams][6 * edge][edge]) receives each canopy's surviving primitive per pixel, -1 where none.
 * The rasterisation, derivative and filtering rules are documented in facebook360_dep_b200/csrc/derp_rephoto.cuh.
 *
 * derp_rephoto_score is computeScoreMap + averageScore (RephotographyUtil.h:39-120): ref / ren are float B, G, R
 * [height][width] images, mask uint8 [height][width] (non-zero = scored), method DERP_REPHOTO_MSSIM or _NCC, stat_radius
 * the Gaussian's radius (window 2r + 1, sigma 1.5, 1..31).  score_map float B, G, R [height][width]; avg[3] the
 * per-channel mean over the mask without NaN scores (B, G, R; 0 for an empty mask).
 */
#ifndef DERP_REPHOTO_H_
#define DERP_REPHOTO_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define DERP_REPHOTO_MSSIM 0
#define DERP_REPHOTO_NCC 1

int derp_rephoto_cubemap(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                         const float* const* colors_bgra, int width, int height, const float* center, int edge,
                         float* out_color, float* out_disparity, int32_t* winners);
int derp_rephoto_score(int device, const float* ref_bgr, const float* ren_bgr, const uint8_t* mask, int width, int height,
                       int method, int stat_radius, float* score_map, double* avg);

#ifdef __cplusplus
}
#endif
#endif /* DERP_REPHOTO_H_ */
