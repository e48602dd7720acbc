/*
 * derp_sweepview.h — C ABI of the constant-depth sweep slices of GenerateCameraOverlaps
 * (source/render/GenerateCameraOverlaps.cpp) and GenerateEquirect (source/render/GenerateEquirect.cpp), and of the
 * constant-depth equirect mask projection of ProjectEquirectsToCameras (source/conversion), on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every image pointer may be host or device memory, so a caller can upload the source images
 * once (derp_device_alloc / derp_device_copy) and pass the same device pointers for every destination and slice.
 *
 * Cameras are passed as the apps hold them after Camera::rescale(resolution * scale): resolution, principal
 * (has_principal = 1) and focal already rescaled; the resolution may be fractional.  images_bgra[i] is camera i's float
 * B, G, R, A image of image_sizes[2 i] x image_sizes[2 i + 1] pixels (width, height).  Outputs are float B, G, R, A.
 *
 * derp_sweep_overlaps: projectSrcsToDst(cams[dst], cams, images, disparities[k]) for k < num_slices
 * (GenerateCameraOverlaps.cpp:54-83): out[k][int(res.y)][int(res.x)].  Per pixel outside the image circle (0, 0, 0, 0);
 * otherwise world = rig({x + .5, y + .5}, 1.0f / disparity), the fp32 sum in camera order of getPixelBilinear over every
 * camera (the destination included) that sees it, times the fp32 1.0f / count (NaN where no camera sees it).
 *
 * derp_sweep_crop_bounds: createCroppedEquirect's bounding box (GenerateEquirect.cpp:139-156) of the equirect pixels of
 * a height x 2 height equirect at depths[k] that any camera sees, as bounds[k] = {minX, maxX, minY, maxY}; with nothing
 * visible the initial values {2 height, 0, height, 0}.
 * derp_sweep_crop_width: size_t(double(height) / (maxY - minY) * (maxX - minX)); DERP_EINVAL for an empty box or one of
 * zero width or height (the reference divides by zero or writes an empty image there).
 *
 * derp_sweep_equirect: createEquirect (bounds == NULL) or createCroppedEquirect with bounds[k] (GenerateEquirect.cpp:
 * 79-175) at depths[k]: out[k][height][width_k], width_k = 2 height or derp_sweep_crop_width(bounds[k]).  The sample
 * direction's sin / cos come from the host's C library; a pixel averages images[c](int(py), int(px)) over the cameras
 * that see its point (fp32 sum, then fp64 1. / n per channel as OpenCV's Vec / int), else the background (0, 0, 1, 1),
 * or (0, 0, 0, 1) with black_bg.  center >= 0 first rotates the rig so that camera `center` faces the equirect's centre
 * (centerRig, GenerateEquirect.cpp:186-231).  Every camera's resolution must fit its image (the texel read is not
 * clamped); DERP_EINVAL otherwise.
 *
 * derp_sweep_center_rig: centerRig(cams, cams[center].id) on the host: out[i] receives camera i with the rotation and
 * origin of the centred rig (forward / up / right as the last transformRig passed them to setRotation), rotation9
 * (optional) the re-unitarised rotation matrix of each camera, row-major, rows right, up, backward.
 *
 * derp_sweep_last_hits: the number of (sample, camera) pairs in which the camera saw the sample's point, summed over the
 * calling thread's last derp_sweep_overlaps or derp_sweep_equirect (the work measure v-bar = hits / samples that
 * tools/sweep_views_bench.py reports).
 *
 * derp_test_sweep_overlaps_host / derp_test_sweep_equirect_host: the same per-pixel functions (DERP_HD), run on the host
 * with host pointers, for tests without a GPU.
 *
 * derp_project_equirect_masks: ProjectEquirectsToCameras' projection (ProjectEquirectsToCameras.cpp:94-125) of one
 * frame for the whole rig.  eqr_masks[i] is camera i's equirect mask, bytes 0 / non-zero, of mask_sizes[2 i] x
 * mask_sizes[2 i + 1] pixels (width, height; any size per camera); out[i] receives [int(res.y)][int(res.x)] bytes, 255
 * where the reference sets the camera mask and 0 elsewhere.  Per pixel: world = rig({x + .5, y + .5}, depth) in fp64,
 * worldToEquirect (ImageUtil.cpp:127-140, float acosf / atan2f), the range test and mask(int(v H), int(u W)).  A NaN
 * equirect coordinate (near a pole, where float(norm) < |z| makes acos NaN and the reference indexes the mask with
 * int(NaN)) leaves the pixel 0; no mask byte outside the image is read for any input.  The device decides a pixel only
 * when an interval evaluation of the chain proves the reference's decision; the other pixels are recomputed on the
 * host with the same code and the C library (derp_sweepview.cuh documents the bound).
 * derp_project_last_host_pixels: the number of pixels the calling thread's last derp_project_equirect_masks resolved on
 * the host.
 * derp_test_project_equirect_masks_host: the same per-pixel function on the host, with host pointers, for tests without a
 * GPU.
 * derp_test_eqr_index_proven: a probe of the device's proof, for tests: the mask index (>= 0), -1 (nothing read) or -2
 *   (undecided) that eqrIndexProven gives for the boxes boxes[6 i .. 6 i + 5] = (x lo, x hi, y lo, y hi, z lo, z hi) of
 *   a width x height mask, on `device` with host pointers.
 * derp_test_eqr_index_host: its host twin, eqrIndex of the points pts[3 i .. 3 i + 2]: the index or -1.
 */
#ifndef DERP_SWEEPVIEW_H_
#define DERP_SWEEPVIEW_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int derp_sweep_overlaps(int device, const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                        const int32_t* image_sizes, int dst, const float* disparities, int num_slices, float* out);
int derp_sweep_crop_bounds(int device, const DerpCameraDesc* cams, int num_cams, int center, uint64_t height,
                           const float* depths, int num_depths, double* bounds);
int derp_sweep_crop_width(uint64_t height, const double* bounds, uint64_t* width);
int derp_sweep_equirect(int device, const DerpCameraDesc* cams, int num_cams, int center, const float* const* images_bgra,
                        const int32_t* image_sizes, uint64_t height, const float* depths, int num_depths,
                        const double* bounds, int black_bg, float* const* out);
int derp_sweep_center_rig(const DerpCameraDesc* cams, int num_cams, int center, DerpCameraDesc* out, double* rotation9);
uint64_t derp_sweep_last_hits(void);

int derp_test_sweep_overlaps_host(const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                                  const int32_t* image_sizes, int dst, const float* disparities, int num_slices,
                                  float* out);
int derp_test_sweep_equirect_host(const DerpCameraDesc* cams, int num_cams, int center,
                                  const float* const* images_bgra, const int32_t* image_sizes, uint64_t height,
                                  const float* depths, int num_depths, const double* bounds, int black_bg,
                                  float* const* out);

int derp_project_equirect_masks(int device, const DerpCameraDesc* cams, int num_cams, double depth,
                                const uint8_t* const* eqr_masks, const int32_t* mask_sizes, uint8_t* const* out);
uint64_t derp_project_last_host_pixels(void);
int derp_test_project_equirect_masks_host(const DerpCameraDesc* cams, int num_cams, double depth,
                                          const uint8_t* const* eqr_masks, const int32_t* mask_sizes,
                                          uint8_t* const* out);
int derp_test_eqr_index_proven(int device, const double* boxes, int n, int width, int height, int64_t* out);
int derp_test_eqr_index_host(const double* pts, int n, int width, int height, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* DERP_SWEEPVIEW_H_ */
