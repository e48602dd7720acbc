"""Generates tests/golden/resize_vectors.npz: cv2.resize(INTER_AREA) [+ cv2.threshold(., t, 255, THRESH_BINARY)] with
cv2 4.13 on one OpenCV thread, for every sample type (u8, u16, f32) and channel count (1, 3, 4) on each path of
resize.cpp: same size, 2 x 2, 3 x 3, 2 x 3, general ratios (3360 -> 2048 and 2160 -> 1318 on thin images), both axes
growing, one axis growing while the other shrinks, 1 x N, N x 1 and 1 x 1 destinations; float content with NaN, +-inf,
denormals and -0; and the threshold at 127 on 8-bit values around it.  The inputs are regenerated from their seeds by
source() (numpy's RandomState streams are fixed), so the file holds the outputs only.

    python tests/golden/gen_resize_vectors.py   (writes the .npz next to this file)
"""
import os

import numpy as np

TYPES = {8: np.uint8, 16: np.uint16, 32: np.float32}
CHANNELS = (1, 3, 4)
# (name, (src_w, src_h), (dst_w, dst_h))
SHAPES = [
    ("same", (13, 7), (13, 7)),
    ("2x2", (26, 14), (13, 7)),
    ("2x2_odd_row", (22, 6), (11, 3)),  # 11 float lanes: a 1-channel row ends in OpenCV's scalar tail
    ("3x3", (21, 15), (7, 5)),
    ("2x3", (26, 15), (13, 5)),
    ("general_x", (3360, 2), (2048, 1)),
    ("general_y", (2, 2160), (1, 1318)),
    ("general", (37, 29), (11, 9)),
    ("grow_both", (7, 5), (9, 8)),
    ("grow_both_wide", (50, 17), (100, 40)),
    ("grow_x_shrink_y", (20, 10), (30, 7)),
    ("shrink_x_grow_y", (20, 10), (8, 15)),
    ("odd_height_grow", (64, 43), (64, 44)),
    ("row_1xN", (13, 9), (1, 5)),
    ("col_Nx1", (13, 9), (5, 1)),
    ("pixel_1x1", (13, 9), (1, 1)),
    ("from_1x1", (1, 1), (5, 3)),
]


def source(bits, channels, w, h, content, seed):
    """The input image of one case (h x w, or h x w x channels)."""
    rng = np.random.RandomState(seed)
    shape = (h, w) if channels == 1 else (h, w, channels)
    if content == "around127":
        return rng.randint(120, 136, shape).astype(np.uint8)
    if bits == 8:
        return rng.randint(0, 256, shape).astype(np.uint8)
    if bits == 16:
        return rng.randint(0, 65536, shape).astype(np.uint16)
    a = (rng.standard_normal(shape) * 100).astype(np.float32)
    if content == "special":
        u = rng.uniform(size=shape)
        a[u < 0.02] = np.nan
        a[(u >= 0.02) & (u < 0.04)] = np.inf
        a[(u >= 0.04) & (u < 0.06)] = -np.inf
        a[(u >= 0.06) & (u < 0.10)] = np.float32(1e-40)  # denormal
        a[(u >= 0.10) & (u < 0.13)] = np.float32(-3e-42)
        a[(u >= 0.13) & (u < 0.20)] = np.float32(-0.0)
    return a


def cases():
    """(key, bits, channels, (src_w, src_h), (dst_w, dst_h), content, seed, threshold or None) of every vector."""
    seed = 0
    for bits in TYPES:
        for ch in CHANNELS:
            contents = ["random"] + (["special"] if bits == 32 else [])
            for name, src, dst in SHAPES:
                for content in contents:
                    seed += 1
                    yield "%s_u%d_c%d_%s" % (name, bits, ch, content), bits, ch, src, dst, content, seed, None
    for ch in CHANNELS:
        for name, src, dst in SHAPES:
            seed += 1
            yield "%s_u8_c%d_thr127" % (name, ch), 8, ch, src, dst, "around127", seed, 127


def cv_resize(img, dst, threshold=None):
    """resize_camera's calls on one OpenCV thread; the result keeps the input's layout (cv2 drops a 1-channel axis)."""
    import cv2
    threads = cv2.getNumThreads()
    cv2.setNumThreads(1)
    try:
        out = cv2.resize(img, dst, interpolation=cv2.INTER_AREA)
        if threshold is not None:
            _, out = cv2.threshold(out, threshold, 255, cv2.THRESH_BINARY)
    finally:
        cv2.setNumThreads(threads)
    return out.reshape((dst[1], dst[0]) + img.shape[2:])


def same_values(a, b):
    """Equal samples: NaN where the other has NaN (its payload is not a value), every other bit pattern equal (-0 too)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype != np.float32:
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a).view(np.uint32), np.where(nb, 0, b).view(np.uint32))


def main():
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    out = {}
    for key, bits, ch, src, dst, content, seed, thr in cases():
        out[key] = cv_resize(source(bits, ch, src[0], src[1], content, seed), dst, thr)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "resize_vectors.npz"), **out)
    print(len(out), "vectors")


if __name__ == "__main__":
    main()
