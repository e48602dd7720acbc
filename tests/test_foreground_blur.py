"""derp_gaussian_blur (include/derp_blur.h), the blur GenerateForegroundMasks applies at --blur_radius.  model_blur below
restates OpenCV's bit-exact fixed-point Gaussian in numpy (exact integer sums) and is pinned here to
cv2.GaussianBlur((2 r + 1)^2, sigma 0) on 16-bit 3-channel images, for every radius the library takes (0 to 64), down to
images smaller than the kernel.  Radius 4 (ksize 9) uses OpenCV's 9-tap table kernel (4 13 30 51 60 51 30 13 4) / 256,
not the sampled Gaussian, and matches exactly like the rest.  The GPU leg (tests/test_gpu_foreground_blur.py) runs the
CUDA library on the same matrix against both."""
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi

MAX_RADIUS = 64
DERP_EINVAL = -1  # include/derp_b200.h
RADII = list(range(MAX_RADIUS + 1))
FIXED_SHAPES = [(97, 64), (5, 3), (1, 1), (1, 40), (40, 1), (300, 7)]  # (width, height)
CONTENTS = ["random", "white", "checker"]


def shapes(radius):
    """The fixed shapes plus shapes narrower and shorter than the (2 r + 1)-tap kernel: reflected once and folded often."""
    out = list(FIXED_SHAPES)
    for small in sorted({2, max(1, radius), max(1, 2 * radius)}):
        out += [(small, 23), (19, small)]
    return out


def image(w, h, content, seed):
    if content == "random":
        return np.random.RandomState(seed).randint(0, 65536, (h, w, 3)).astype(np.uint16)
    if content == "white":
        return np.full((h, w, 3), 65535, np.uint16)
    board = ((np.arange(h)[:, None] + np.arange(w)[None, :]) % 2 * 65535).astype(np.uint16)
    return np.repeat(board[:, :, None], 3, axis=2)


def matrix(radius):
    """(width, height, content, image) of the exactness matrix at one radius."""
    for i, (w, h) in enumerate(shapes(radius)):
        for content in CONTENTS:
            yield w, h, content, image(w, h, content, 1000 * radius + i)


def taps(radius):
    """OpenCV's taps for ksize 2 r + 1, sigma 0, with 16 fraction bits (getGaussianKernelBitExact, then
    getGaussianKernelFixedPoint_ED): the table kernels of sizes 1 to 9; above those exp(-x^2 / (8 sigma^2)) at
    x = 1 - n, 3 - n, ..., -2 with sigma = fma(n, 0.15, 0.35), scaled by 1 / (2 sum + 1), error-diffused to integers
    over the left half (ties to even), mirrored, the centre tap 2^16 minus the rest."""
    import math
    from fractions import Fraction
    n = 2 * radius + 1
    table = {1: [1], 3: [1, 2, 1], 5: [1, 4, 6, 4, 1], 7: [2, 7, 14, 18, 14, 7, 2], 9: [4, 13, 30, 51, 60, 51, 30, 13, 4]}
    if n in table:
        return np.array(table[n], np.uint64) * np.uint64(65536 // sum(table[n]))
    sigma = float(Fraction(n) * Fraction(0.15) + Fraction(0.35))  # one rounding, as fma
    scale = -0.125 / (sigma * sigma)
    half = [math.exp(float(x * x) * scale) for x in range(1 - n, -1, 2)]
    total = 0.0
    for t in half:
        total += t
    mul = 1.0 / (total * 2 + 1)
    left, err = [], 0.0
    for t in half:
        a = t * mul * 65536.0 + err
        v = round(a)
        err = a - v
        left.append(v)
    return np.array(left + [65536 - 2 * sum(left)] + left[::-1], np.uint64)


def reflect101(i, size):
    """BORDER_REFLECT_101 of index array i, folded as often as needed (period 2 (size - 1))."""
    if size == 1:
        return np.zeros_like(i)
    period = 2 * (size - 1)
    i = np.abs(i) % period
    return np.where(i < size, i, period - i)


def model_blur(img, radius):
    """The fixed-point blur: u32 row sums (exact: at most 65535 * 2^16), u64 column sums rounded by (s + 2^31) >> 32."""
    h, w, _ = img.shape
    k = taps(radius)
    src = img.astype(np.uint64)
    xs, ys = np.arange(w), np.arange(h)
    rows = np.zeros((h, w, 3), np.uint64)
    for i in range(2 * radius + 1):
        rows += k[i] * src[:, reflect101(xs + i - radius, w)]
    assert rows.max(initial=0) < 2 ** 32
    cols = np.zeros((h, w, 3), np.uint64)
    for j in range(2 * radius + 1):
        cols += k[j] * rows[reflect101(ys + j - radius, h)]
    return ((cols + np.uint64(1 << 31)) >> np.uint64(32)).astype(np.uint16)


def cv_blur(img, radius):
    """cv2.GaussianBlur on one OpenCV thread: with several, cv2 4.13 now and then writes wrong values into a row of a short
    16-bit image (seen on 300 x 7 at ksize 5: a few pixels of row 1 off by hundreds, about once in a thousand calls)."""
    import cv2
    k = 2 * radius + 1
    threads = cv2.getNumThreads()
    cv2.setNumThreads(1)
    try:
        return cv2.GaussianBlur(img, (k, k), 0)
    finally:
        cv2.setNumThreads(threads)


@pytest.mark.parametrize("radius", RADII)
def test_model_matches_opencv(radius):
    for w, h, content, img in matrix(radius):
        got = model_blur(img, radius)
        want = cv_blur(img, radius)
        assert np.array_equal(got, want), (radius, w, h, content, int((got != want).sum()))


def test_radius_4_is_the_table_kernel():
    """ksize 9 is OpenCV's table kernel: a 1-row impulse of 65535 returns the taps in 16-bit units, less their 1/65536."""
    import cv2
    img = np.zeros((1, 21, 3), np.uint16)
    img[0, 10] = 65535
    want = np.array([4, 13, 30, 51, 60, 51, 30, 13, 4]) * 256
    assert np.array_equal(cv_blur(img, 4)[0, 6:15, 0], want)
    assert np.array_equal(taps(4), want)
    assert np.array_equal(np.rint(cv2.getGaussianKernel(9, 0)[:, 0] * 65536), want)


def test_bad_arguments():
    """The library refuses a radius above 64 (and other bad arguments) before it touches a device."""
    blur = capi.Blur(capi.load_cuda())
    img = np.zeros((4, 4, 3), np.uint16)
    out = np.zeros_like(img)
    for w, h, r in ((4, 4, MAX_RADIUS + 1), (4, 4, 1000), (4, 4, -1), (0, 4, 1), (4, 0, 1)):
        assert blur.lib.derp_gaussian_blur(0, img.ctypes.data, w, h, r, out.ctypes.data) == DERP_EINVAL, (w, h, r)
    assert blur.lib.derp_gaussian_blur(0, None, 4, 4, 1, out.ctypes.data) == DERP_EINVAL
    assert blur.lib.derp_gaussian_blur(0, img.ctypes.data, 4, 4, 1, None) == DERP_EINVAL
    with pytest.raises(capi.DerpError):
        blur.gaussian_blur(img, MAX_RADIUS + 1)


def test_exports_every_declared_symbol():
    """include/derp_blur.h: the product exports every declared entry point, and the binding covers them."""
    import re
    hdr = open(os.path.join(capi.ROOT, "include", "derp_blur.h")).read()
    declared = sorted(re.findall(r"^int (derp_[a-z0-9_]+)\(", hdr, re.M))
    assert declared == capi.BLUR_SYMBOLS
    lib = capi.Blur(capi.load_cuda())
    for name in declared + ["derp_last_error"]:
        assert hasattr(lib.lib, name), name


def test_header_declares_it_in_c99(tmp_path):
    """include/derp_blur.h is plain C: a C99 program calls the entry point through that header alone."""
    src = tmp_path / "blur.c"
    src.write_text('#include "derp_blur.h"\n#include <stdint.h>\n'
                   'int main(void) { uint16_t px[3] = {0, 0, 0};\n'
                   '  return derp_gaussian_blur(0, px, 1, 1, 65, px) == DERP_EINVAL ? 0 : 1; }\n')
    exe = tmp_path / "blur"
    libdir = os.path.dirname(capi.CUDA_LIB)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", capi.ROOT + "/include", str(src),
                           "-o", str(exe), "-L", libdir, "-lderp_b200", "-Wl,-rpath," + libdir])
    assert subprocess.run([str(exe)]).returncode == 0


def test_app_refuses_radius_above_64(tmp_path):
    """GenerateForegroundMasks --blur_radius=65 stops before reading anything or creating an output directory."""
    from tests.test_apps import run
    out = tmp_path / "masks"
    p = run("GenerateForegroundMasks", "--rig=" + str(tmp_path / "rig.json"), "--color=" + str(tmp_path / "fg"),
            "--background_color=" + str(tmp_path / "bg"), "--foreground_masks=" + str(out), "--first=000000",
            "--last=000000", "--blur_radius=65", check=False)
    assert p.returncode != 0 and "blur_radius" in p.stderr, p.stderr[-2000:]
    assert not out.exists()
