/*
 * derp_riganalysis.h — C ABI of RigAnalyzer's coverage analysis (source/rig/RigAnalyzer.cpp) on the H100: how many
 * cameras of a rig see each direction, at each distance.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every output pointer may be host or device memory (device memory of the current device is
 * written in place).  The rig may have any number of cameras.
 *
 * Cameras: cams[i] as the app holds them (resolution, principal and focal already rescaled), and optionally
 * rotation9[9 i .. 9 i + 8], camera i's rotation matrix row-major with rows right, up, backward, used exactly as given.
 * This is the rotation Camera::perturbCameras leaves (setRotation(angleAxis) does not re-unitarise).  rotation9 = NULL:
 * the rotation setRotation(forward, up, right) builds from cams[i].  Camera i "sees" a point as Camera::sees
 * (Camera.h:154-190) decides it; a NaN pixel (a point on the camera's optical axis) is seen, as isOutsideSensor is false
 * for NaN.
 *
 * derp_rig_coverage: main's coverage loop (RigAnalyzer.cpp:557-589).  samples: num_samples unit vectors (x, y, z),
 *   host memory; distances: num_distances values, host memory.  hist[k (num_cams + 1) + c] receives the number of
 *   samples s for which exactly c cameras see distances[k] * s.
 * derp_rig_equirect_coverage: saveEquirect's loop (RigAnalyzer.cpp:376-438) on a width x height equirect: pixel (x, y)
 *   has lat = M_PI / 2 - (y + 0.5) / height * M_PI, lon = -M_PI + (x + 0.5) / width * 2 * M_PI (sin / cos from the
 *   host's C library) and the point (cos(lat) cos(lon), cos(lat) sin(lon), sin(lat)) * distance.  counts[y][x] receives
 *   the number of cameras that see it; min_timing[y][x] (optional) minTimingDiff: 1.0, or the least
 *   |t_i - t_j| in float over pairs of those cameras, t = float(pixel.y / resolution.y).
 * derp_rig_camera_coverage: saveCamera (RigAnalyzer.cpp:346-374) for camera cam: counts[int(res.y)][int(res.x)] is 0
 *   outside cam's image circle, else the number of cameras (cam included) that see cam.rig({x + .5, y + .5},
 *   distance).
 * derp_rig_cross_section: saveCrossSection (RigAnalyzer.cpp:440-460) on a dim x dim grid: counts[y][x] is the number
 *   of cameras that see (x + .5 - .5 dim, y + .5 - .5 dim, 0).
 *
 * The device decides a camera only where the decision is the reference's: with -fmad=false, Camera::sees on a point
 * is IEEE arithmetic for RECTILINEAR, EQUISOLID and ORTHOGRAPHIC cameras; FTHETA's atan2 and the camera mode's rig
 * point (sin / cos / atan / asin) are bounded by an interval evaluation (derp_riganalysis.cuh documents the bound).
 * Any other point is recomputed on the host with the same code and the C library.
 * derp_rig_analysis_last_host_points: the number of points the calling thread's last call resolved on the host.
 *
 * derp_test_rig_*_host: the same computations on the host (DERP_HD code, the reference's loops), with host pointers,
 * for tests without a GPU.
 *
 * Probes of the device's interval proofs, for tests: each runs the device function the kernels run on the given inputs
 * (host pointers in and out, on `device`).
 * derp_test_math: the device's function fn (DERP_MATH_*) of a[i] (and b[i]; acosf and atan2f take them narrowed to
 *   float): out[3 i] the value, out[3 i + 1 .. 3 i + 2] the interval the proofs widen it to (derp_interval.cuh's widenD
 *   / widenF; the value itself for DERP_MATH_ATAN2POS, the sweep's FTHETA atan2).
 * derp_test_acosf_exhaustive: every float x in [-1, 1], the device's acosf against the host's acosf and acos(double(x));
 *   stats[0] and stats[1] the greatest device and host errors in ulps of acos(double(x)) times 2^20, stats[2] the
 *   greatest distance between the two in float steps, stats[3] the host values outside the device value's widenF.
 * derp_test_rig_point_iv: rigPointIv of cam's pixels (pix[2 i], pix[2 i + 1]) at depth: out[7 i .. 7 i + 5] the
 *   intervals (lo, hi) of x, y and z, out[7 i + 6] undistort's result for the pixel.  Host twin: derp_test_camera_rig
 *   at the pixel's centre.
 * derp_test_sees_iv: seesIv of cam on the boxes boxes[6 i .. 6 i + 5] = (x lo, x hi, y lo, y hi, z lo, z hi):
 *   decision[i] 1 (seen), 0 (not seen) or -1 (undecided), py[2 i .. 2 i + 1] the pixel row's interval when seen.  Host
 *   twin: derp_test_camera_sees.
 * derp_test_sees_device: the device's Camera::sees of exact points, as derp_test_camera_sees on the host.
 * derp_test_proven_count: provenCount with timing of exact points: counts[i] the cameras that see point i and
 *   timing[i] its minTimingDiff, or counts[i] = -1 where the device leaves the point to the host.
 * derp_test_count_timing_host: the host twin (saveEquirect's per-point loop): counts[i] and timing[i] always.
 */
#ifndef DERP_RIGANALYSIS_H_
#define DERP_RIGANALYSIS_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int derp_rig_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                      const double* samples, int num_samples, const double* distances, int num_distances,
                      uint64_t* hist);
int derp_rig_equirect_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int width,
                               int height, double distance, int32_t* counts, float* min_timing);
int derp_rig_camera_coverage(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int cam,
                             double distance, int32_t* counts);
int derp_rig_cross_section(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams, int dim,
                           int32_t* counts);
uint64_t derp_rig_analysis_last_host_points(void);

int derp_test_rig_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                                const double* samples, int num_samples, const double* distances, int num_distances,
                                uint64_t* hist);
int derp_test_rig_equirect_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int width,
                                         int height, double distance, int32_t* counts, float* min_timing);
int derp_test_rig_camera_coverage_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int cam,
                                       double distance, int32_t* counts);
int derp_test_rig_cross_section_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, int dim,
                                     int32_t* counts);

enum {
  DERP_MATH_SIN = 0,
  DERP_MATH_COS = 1,
  DERP_MATH_ATAN = 2,
  DERP_MATH_ASIN = 3,
  DERP_MATH_ATAN2 = 4,
  DERP_MATH_ACOSF = 5,
  DERP_MATH_ATAN2F = 6,
  DERP_MATH_ATAN2POS = 7
};
int derp_test_math(int device, int fn, const double* a, const double* b, int n, double* out);
int derp_test_acosf_exhaustive(int device, uint32_t* stats);
int derp_test_rig_point_iv(int device, const DerpCameraDesc* cam, const int32_t* pix, int n, double depth, double* out);
int derp_test_sees_iv(int device, const DerpCameraDesc* cam, const double* boxes, int n, int32_t* decision,
                      double* py);
int derp_test_sees_device(int device, const DerpCameraDesc* cam, const double* pts, int n, double* pix, uint8_t* seen);
int derp_test_proven_count(int device, const DerpCameraDesc* cams, const double* rotation9, int num_cams,
                           const double* pts, int n, int32_t* counts, float* timing);
int derp_test_count_timing_host(const DerpCameraDesc* cams, const double* rotation9, int num_cams, const double* pts,
                                int n, int32_t* counts, float* timing);

#ifdef __cplusplus
}
#endif
#endif /* DERP_RIGANALYSIS_H_ */
