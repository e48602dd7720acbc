/*
 * derp_blur.h — C ABI of the Gaussian blur GenerateForegroundMasks applies at --blur_radius, on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every image pointer may be host, pinned, managed, device or another GPU's memory, at any
 * alignment (derp_b200.h's caller-pointer rule).
 *
 * derp_gaussian_blur is cv_util::gaussianBlur(image, radius) = cv::GaussianBlur(image, (2 radius + 1)^2, sigma 0)
 * (CvUtil.h:302-312) of a 3-channel 16-bit image, the blur GenerateForegroundMasks applies to background and frame
 * (BackgroundSubtractionUtil.h:30-33).  Bit-identical to OpenCV's fixed-point path (16-bit taps, BORDER_REFLECT_101)
 * for radius 0 (a copy) to 64, also on images smaller than the kernel; a larger radius is DERP_EINVAL.  src and dst are
 * u16 [height][width][3] and may be the same buffer.  The call returns with dst written.
 */
#ifndef DERP_BLUR_H_
#define DERP_BLUR_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int derp_gaussian_blur(int device, const uint16_t* src, int width, int height, int radius, uint16_t* dst);

#ifdef __cplusplus
}
#endif
#endif /* DERP_BLUR_H_ */
