"""Generator of tests/golden/rigsim_vectors.npz: RigSimulator's downscale (cv::resize INTER_AREA by the integer factor
--anti_alias_supersample) of its float B, G, R image and float depth map, pinned to cv2 4.13.

For factors 2, 3 and 4 and for 3 and 1 channels, a 12 x 24 image of random values in [0, 255] with the samples a
render writes where nothing is hit: depth FLT_MAX, whose sums overflow to inf, next to ordinary depths; plus inf
itself.  Keys: src_c<cn> (the input), dst_c<cn>_k<k> (cv2's output)."""
import os

import cv2
import numpy as np

assert cv2.__version__.startswith("4.13")
rng = np.random.default_rng(29)
FLT_MAX = np.finfo(np.float32).max
out = {}
for cn in (3, 1):
    src = (rng.random((12, 24, cn), dtype=np.float32) * np.float32(255)).astype(np.float32)
    flat = src.reshape(-1)
    pick = rng.random(flat.shape) < 0.25
    flat[pick] = FLT_MAX
    flat[rng.random(flat.shape) < 0.02] = np.inf
    src = src if cn == 3 else src[:, :, 0]
    out["src_c%d" % cn] = src
    for k in (2, 3, 4):
        out["dst_c%d_k%d" % (cn, k)] = cv2.resize(src, (24 // k, 12 // k), interpolation=cv2.INTER_AREA)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "rigsim_vectors.npz"), **out)
