#!/usr/bin/env python3
"""Generates tests/golden/rephoto_vectors.npz with the cv2 wheel of this image (cv2 4.13.0, single thread).  Pins the
score half of ComputeRephotographyErrors (source/render/RephotographyUtil.h) to OpenCV's own calls:
  computeSSIM         cv::GaussianBlur((2r + 1)^2, sigma 1.5, BORDER_REFLECT_101) of fp32 B, G, R images, the fp32
                      MatExpr sequence, cv::pow with exponents 1 (MSSIM) and 0 (NCC: luminance = contrast = 1)
  averageScore        cv::mean(channel, mask) with NaN scores removed from the mask
  stackResults' JET   convertTo(CV_8U, 255), 255 - x, applyColorMap(COLORMAP_JET) of a 3-channel image, zero outside
                      the mask; and the JET table itself
Inputs are seeded; x carries NaN pixels so that the score map has NaN regions inside the mask.
"""
import os

import cv2
import numpy as np

cv2.setNumThreads(1)


def compute_ssim(x, y, r, alpha, beta, gamma):
    w = 2 * r + 1
    blur = lambda m: cv2.GaussianBlur(m, (w, w), 1.5, 0)  # noqa: E731
    f = np.float32
    muX, muY = blur(x), blur(y)
    mu2X, mu2Y, muXY = muX * muX, muY * muY, muX * muY
    sig2X = blur((x - muX) * (x - muX))
    sig2Y = blur((y - muY) * (y - muY))
    sigXY = blur((x - muX) * (y - muY))
    with np.errstate(invalid="ignore"):
        sigX, sigY = cv2.sqrt(sig2X), cv2.sqrt(sig2Y)
    c1, c2 = f(0.0001), f(0.0009)
    c3 = f(np.float64(c2) / 2.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        lum = (f(2) * muXY + c1) * (f(1) / (mu2X + mu2Y + c1))
        con = (f(2) * (sigX * sigY) + c2) * (f(1) / (sig2X + sig2Y + c2))
        st = (sigXY + c3) * (f(1) / (sigX * sigY + c3))
    lum, con, st = cv2.pow(lum, alpha), cv2.pow(con, beta), cv2.pow(st, gamma)
    return (con * lum) * st


def average_score(score, mask):
    out = np.zeros(3)
    for c in range(3):
        m = mask.copy()
        m[np.isnan(score[..., c])] = 0
        out[c] = cv2.mean(np.ascontiguousarray(score[..., c]), m)[0]
    return out


def jet_panel(score, mask):
    s8 = cv2.addWeighted(score, 255.0, score, 0.0, 0.0, dtype=cv2.CV_8U)  # Mat::convertTo(CV_8U, 255)
    s8 = cv2.subtract(np.full_like(s8, 255), s8)
    j = cv2.applyColorMap(s8, cv2.COLORMAP_JET)
    j[mask == 0] = 0
    return j


def main():
    rng = np.random.RandomState(2024)
    out = {}
    edge = 16
    h, w = 6 * edge, edge
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([np.sin(xx / 3.0) * 0.3 + 0.5, np.cos(yy / 5.0) * 0.3 + 0.5, (xx + yy) / (w + h)], -1)
    x = (base + rng.uniform(-0.1, 0.1, base.shape)).astype(np.float32)
    y = (base + rng.uniform(-0.15, 0.15, base.shape)).astype(np.float32)
    x[7, 3] = np.nan  # NaN inside the mask: the blur spreads it to a (2r+1)^2 neighbourhood of NaN scores
    x[40, 9, 1] = np.nan
    mask = np.where(rng.uniform(size=(h, w)) < 0.8, 255, 0).astype(np.uint8)
    mask[:, :2] = 0
    out["x"], out["y"], out["mask"] = x, y, mask
    for r in (1, 2):
        for name, (a, b, g) in (("MSSIM", (1, 1, 1)), ("NCC", (0, 0, 1))):
            s = compute_ssim(x, y, r, a, b, g).astype(np.float32)
            out["score_%s_r%d" % (name, r)] = s
            out["avg_%s_r%d" % (name, r)] = average_score(s, mask)
            out["jet_%s_r%d" % (name, r)] = jet_panel(s, mask)
    # a score map with values outside [0, 1] and NaN for the 8-bit conversion
    wild = rng.uniform(-0.3, 1.3, (h, w, 3)).astype(np.float32)
    wild[5, :, 0] = np.nan
    wild[6, :4] = np.array([0.5 / 255, 1.5 / 255, 2.5 / 255, 254.5 / 255], np.float32)[:, None]
    out["wild"] = wild
    out["jet_wild"] = jet_panel(wild, mask)
    out["jet_lut"] = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_JET).reshape(256, 3)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "rephoto_vectors.npz"), **out)


if __name__ == "__main__":
    main()
