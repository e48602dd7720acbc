/*
 * derp_resize.h — C ABI of the pyramid resize of the render pipeline (scripts/render/resize.py), on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every image pointer may be host, pinned, managed, device or another GPU's memory, at any
 * alignment (derp_b200.h's caller-pointer rule).
 *
 * derp_resize_area is cv2.resize(src, (dst_w, dst_h), interpolation=INTER_AREA), followed, when threshold >= 0, by
 * cv2.threshold(., threshold, 255, THRESH_BINARY) (v > threshold ? 255 : 0, in the sample type), of a
 * [src_h][src_w][channels] image of 8-bit (sample_bits 8, uint8_t), 16-bit (16, uint16_t) or float (32) samples with 1, 3
 * or 4 channels, in either direction.  dst is [dst_h][dst_w][channels] of the same type.  Every value equals OpenCV 4.13's
 * (x86, SSE baseline) on one OpenCV thread: the same size is a copy, integer ratios follow resizeAreaFast_, other
 * shrinking ratios ResizeArea_Invoker, and a growing axis the bilinear variant, in fixed point for 8-bit samples.  (With
 * several OpenCV threads, a float row that starts one of OpenCV's stripes may hold +0 where this holds -0.)
 * src and dst must not overlap.  DERP_EINVAL for other bit depths or channel counts, non-positive sizes, and images whose
 * byte counts overflow.  The call returns with dst written.
 */
#ifndef DERP_RESIZE_H_
#define DERP_RESIZE_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int derp_resize_area(int device, const void* src, int sample_bits, int channels, int src_w, int src_h, void* dst, int dst_w,
                     int dst_h, int threshold);

#ifdef __cplusplus
}
#endif
#endif /* DERP_RESIZE_H_ */
