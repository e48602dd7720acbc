#!/usr/bin/env python3
"""Generates tests/golden/linear_vectors.npz with the cv2 wheel of this image (cv2 4.13.0): cv::resize(src, dst, Size(),
f, f) with the default INTER_LINEAR on float32 images, the resize CreateObjFromDisparityEquirect applies for --scale < 1.
Sources are seeded, so only the cv2 outputs are stored with them.  Run: python tests/golden/gen_linear_vectors.py"""
import os

import cv2
import numpy as np

CASES = [(37, 23, 0.37), (64, 48, 0.5), (101, 67, 0.37), (40, 40, 0.8), (13, 9, 0.6), (200, 100, 0.25), (33, 17, 0.5),
         (7, 5, 0.5), (384, 192, 0.37), (30, 20, 0.999), (9, 9, 0.2)]


def source(i, w, h):
    rng = np.random.RandomState(100 + i)
    return rng.uniform(0.01, 1.0, (h, w)).astype(np.float32)


def main():
    assert cv2.__version__ == "4.13.0", cv2.__version__
    out = {}
    for i, (w, h, f) in enumerate(CASES):
        out["linear_%d" % i] = cv2.resize(source(i, w, h), None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "linear_vectors.npz"), **out)


if __name__ == "__main__":
    main()
