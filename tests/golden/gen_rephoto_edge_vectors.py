#!/usr/bin/env python3
"""Generates tests/golden/rephoto_edge_vectors.npz with the cv2 wheel of this image (cv2 4.13.0, single thread): the
score of ComputeRephotographyErrors (RephotographyUtil.h, restated by gen_rephoto_vectors.py's compute_ssim and
average_score) at the shapes and radii where a separable blur goes wrong.  rephoto_vectors.npz is left as it is.

  base_*     rephoto_vectors.npz's own x, y and mask at the radii it does not cover (4, 5, 31)
  odd        37 x 23, odd and non-square, NaN inputs (x and y) inside the mask
  cube       the cubemap layout 6e x e (e = 13) with the coverage of a partial render: a NaN-free colour cube with
             uncovered (zero) texels, as the app scores it
  tiny       5 x 3: every kernel of radius >= 3 is wider than the image, so BORDER_REFLECT_101 bounces several times
  row, col   1 x 29 and 29 x 1: a 1-pixel dimension, where REFLECT_101 maps every offset to the one row or column
  empty      an empty mask: every average is 0
Every case is scored at radius 1, 2, 4, 5 and 31 (the API's maximum) with MSSIM and NCC.  Inputs are seeded.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_rephoto_vectors import average_score, compute_ssim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
RADII = (1, 2, 4, 5, 31)
METHODS = (("MSSIM", (1, 1, 1)), ("NCC", (0, 0, 1)))


def _pair(rng, h, w):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([np.sin(xx / 2.0 + yy / 7.0) * 0.3 + 0.5, np.cos(yy / 3.0) * 0.3 + 0.5,
                     (xx + 2 * yy) / (w + 2 * h + 1.0)], -1)
    x = (base + rng.uniform(-0.1, 0.1, base.shape)).astype(np.float32)
    y = (base + rng.uniform(-0.15, 0.15, base.shape)).astype(np.float32)
    return x, y


def cases():
    rng = np.random.RandomState(4242)
    out = {}
    x, y = _pair(rng, 23, 37)
    x[4, 30] = np.nan  # a pixel of x and one channel of y inside the mask
    y[17, 6, 2] = np.nan
    m = np.where(rng.uniform(size=(23, 37)) < 0.7, 255, 0).astype(np.uint8)
    m[4, 30] = m[17, 6] = 255
    m[:, -3:] = 0
    out["odd"] = (x, y, m)
    e = 13
    x, y = _pair(rng, 6 * e, e)
    cov = np.zeros((6 * e, e), bool)
    cov[: 2 * e] = True
    cov[2 * e: 3 * e, : e // 2] = True
    cov[4 * e + 3: 5 * e + 5] = True
    x[~cov] = 0  # zeroOutNans: the app scores uncovered texels as black
    y[~cov] = 0
    out["cube"] = (x, y, np.where(cov, 1, 0).astype(np.uint8))
    x, y = _pair(rng, 3, 5)
    out["tiny"] = (x, y, np.full((3, 5), 255, np.uint8))
    x, y = _pair(rng, 1, 29)
    m = np.ones((1, 29), np.uint8)
    m[0, :3] = 0
    out["row"] = (x, y, m)
    x, y = _pair(rng, 29, 1)
    m = np.ones((29, 1), np.uint8)
    m[-4:] = 0
    out["col"] = (x, y, m)
    x, y = _pair(rng, 9, 11)
    out["empty"] = (x, y, np.zeros((9, 11), np.uint8))
    return out


def main():
    import cv2
    cv2.setNumThreads(1)
    out = {}
    old = np.load(os.path.join(HERE, "rephoto_vectors.npz"))
    inputs = dict(cases())
    inputs["base"] = (old["x"], old["y"], old["mask"])
    for name, (x, y, m) in inputs.items():
        if name != "base":
            out[name + "_x"], out[name + "_y"], out[name + "_mask"] = x, y, m
        for r in RADII:
            if name == "base" and r in (1, 2):
                continue  # in rephoto_vectors.npz
            for method, (a, b, g) in METHODS:
                s = compute_ssim(x, y, r, a, b, g).astype(np.float32)
                out["%s_score_%s_r%d" % (name, method, r)] = s
                out["%s_avg_%s_r%d" % (name, method, r)] = average_score(s, m)
    np.savez_compressed(os.path.join(HERE, "rephoto_edge_vectors.npz"), **out)


if __name__ == "__main__":
    main()
