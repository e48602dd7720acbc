"""derp_gaussian_blur on the GPU and GenerateForegroundMasks at every --blur_radius the UI's slider offers (1 to 20).
The CUDA library against cv2.GaussianBlur and against the numpy restatement of tests/test_foreground_blur.py on its matrix
(every radius 0 to 64) and on 2048 x 1024 images, the app's default width; radius 1 against the blur inside
derp_foreground_mask; every kind of caller pointer; and the app end to end against the cv2 chain of
BackgroundSubtractionUtil.h, and at radii 2 and 3 against the host blur (io::gaussianBlurU16C3) it used to run."""
import json
import os

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests.test_foreground_blur import RADII, cv_blur, image, matrix, model_blur

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def blur(cuda):
    return capi.Blur(cuda)


@pytest.mark.parametrize("radius", RADII)
def test_matches_opencv_and_model(blur, radius):
    for w, h, content, img in matrix(radius):
        got = blur.gaussian_blur(img, radius)
        assert np.array_equal(got, cv_blur(img, radius)), (radius, w, h, content)
        assert np.array_equal(got, model_blur(img, radius)), (radius, w, h, content)


@pytest.mark.parametrize("radius", [2, 4, 10, 20])
def test_app_width(blur, radius):
    rng = np.random.RandomState(radius)
    img = rng.randint(0, 65536, (1024, 2048, 3)).astype(np.uint16)
    img[100:400, 300:900] = 65535  # flat regions next to noise: sums at the top of the range
    img[600:700] = 0
    got = blur.gaussian_blur(img, radius)
    assert np.array_equal(got, cv_blur(img, radius))
    assert np.array_equal(got, model_blur(img, radius))


def test_radius_1_is_the_foreground_mask_blur(cuda, blur):
    """derp_foreground_mask(blur_radius = 1) == its blur 0 on images derp_gaussian_blur blurred with radius 1, at thresholds
    dense enough that any blurred value off by one unit would move some pixel across one of them."""
    rng = np.random.RandomState(11)
    H, W = 120, 161
    bg = rng.randint(0, 65536, (H, W, 3)).astype(np.uint16)
    fr = np.clip(bg.astype(np.int64) + rng.randint(-3000, 3000, bg.shape), 0, 65535).astype(np.uint16)
    bb, fb = blur.gaussian_blur(bg, 1), blur.gaussian_blur(fr, 1)
    flips = 0
    for thr in np.linspace(0.0005, 0.05, 60).astype(np.float32):
        inside = cuda.foreground_mask(bg, fr, 1, float(thr), 0)
        outside = cuda.foreground_mask(bb, fb, 0, float(thr), 0)
        assert np.array_equal(inside, outside), thr
        flips += int(inside.sum())
    assert 0 < flips < 60 * H * W


@pytest.mark.parametrize("kind", ["device", "pinned", "misaligned", "device1"])
def test_caller_pointers(blur, kind):
    """The caller-pointer rule of include/derp_b200.h, as tests/test_gpu_caller_pointers.py checks it for every entry point."""
    import torch
    from tests.test_gpu_caller_pointers import same_as_host
    if kind == "device1" and torch.cuda.device_count() < 2:
        pytest.skip("needs a second CUDA device")
    img = image(83, 45, "random", 3)

    def body(r):
        for radius in (0, 1, 4, 20):
            r_out = r.out(img.nbytes)
            blur.check(blur.lib.derp_gaussian_blur(0, r.inp(img), 83, 45, radius, r_out))

    same_as_host(body, kind)


def test_in_place(blur):
    """src == dst, in device memory (used in place) and in host memory (staged)."""
    import torch
    img = image(130, 70, "random", 4)
    t = torch.from_numpy(img.copy()).cuda()
    blur.check(blur.lib.derp_gaussian_blur(0, t.data_ptr(), 130, 70, 9, t.data_ptr()))
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), cv_blur(img, 9))
    buf = img.copy()
    blur.check(blur.lib.derp_gaussian_blur(0, buf.ctypes.data, 130, 70, 9, buf.ctypes.data))
    assert np.array_equal(buf, cv_blur(img, 9))


# ---- the app ----------------------------------------------------------------------------------------------------------
S, WF, HF, WO = 2, 120, 90, 80


def _dataset(tmp_path):
    import cv2
    from facebook360_dep_b200 import synth
    rig = synth.ring_rig(S, WF, HF, kind="FTHETA")
    os.makedirs(tmp_path / "rigs", exist_ok=True)
    json.dump(rig, open(tmp_path / "rigs" / "rig.json", "w"))
    rng = np.random.RandomState(2)
    ids = [c["id"] for c in rig["cameras"]]
    for s, cid in enumerate(ids):
        bg = np.clip(rng.normal(30000, 9000, (HF, WF, 3)), 0, 65535).astype(np.uint16)
        fr = bg.copy()
        fr[20:60, 30 + 5 * s:80] = rng.randint(0, 65536, (40, 50 - 5 * s, 3)).astype(np.uint16)
        for d, im, name in (("bg", bg, "000000"), ("fg", fr, "000007")):
            os.makedirs(tmp_path / d / cid, exist_ok=True)
            cv2.imwrite(str(tmp_path / d / cid / (name + ".png")), im)
    return ids


def _run_app(tmp_path, radius, closing):
    from tests.test_apps import run
    mdir = tmp_path / ("masks_%d_%d" % (radius, closing))
    run("GenerateForegroundMasks", "--rig=" + str(tmp_path / "rigs" / "rig.json"), "--color=" + str(tmp_path / "fg"),
        "--background_color=" + str(tmp_path / "bg"), "--foreground_masks=" + str(mdir), "--first=000007", "--last=000007",
        "--width=%d" % WO, "--blur_radius=%d" % radius, "--morph_closing_size=%d" % closing)
    return mdir


def _resized(tmp_path, d, cid, name):
    import cv2
    ho = int(np.rint(WO * HF / np.float32(WF)))
    return cv2.resize(cv2.imread(str(tmp_path / d / cid / (name + ".png")), cv2.IMREAD_UNCHANGED), (WO, ho),
                      interpolation=cv2.INTER_AREA)


@pytest.mark.parametrize("radius", [4, 9, 20])
def test_app_matches_cv2_chain(tmp_path, cuda, radius):
    """generateForegroundMask's cv2 calls (as tests/test_z_late_additions.py runs them) at the UI's closing range."""
    import cv2
    ids = _dataset(tmp_path)
    a32 = np.float32(1.0) / np.float32(65535.0)
    for closing in (1, 4, 20):
        mdir = _run_app(tmp_path, radius, closing)
        for cid in ids:
            b, f = _resized(tmp_path, "bg", cid, "000000"), _resized(tmp_path, "fg", cid, "000007")
            diff = cv2.absdiff(cv_blur(b, radius).astype(np.float32) * a32, cv_blur(f, radius).astype(np.float32) * a32)
            m = (np.sqrt((diff.astype(np.float64) ** 2).sum(-1)) > np.float64(np.float32(0.04))).astype(np.uint8)
            m = cv2.morphologyEx(m, cv2.MORPH_CLOSE, cv2.getStructuringElement(cv2.MORPH_RECT, (closing, closing)))
            got = cv2.imread(str(mdir / cid / "000007.png"), cv2.IMREAD_UNCHANGED)
            assert got.dtype == np.uint8 and np.array_equal(got, m * 255), (radius, closing, cid)
            assert 0 < m.sum() < m.size


@pytest.mark.parametrize("radius", [2, 3])
def test_app_matches_former_host_blur(tmp_path, cuda, radius):
    """Radii 2 and 3 used to blur on the host (io::gaussianBlurU16C3, IoSelfTest --mode=gauss) before a derp_foreground_mask
    without blur: the app's masks are those of that path."""
    import cv2
    from tests.test_apps import run
    ids = _dataset(tmp_path)
    mdir = _run_app(tmp_path, radius, 4)
    for cid in ids:
        blurred = []
        for d, name in (("bg", "000000"), ("fg", "000007")):
            img = _resized(tmp_path, d, cid, name)
            h, w = img.shape[:2]
            src, out = str(tmp_path / "g.raw"), str(tmp_path / "g.out")
            img.tofile(src)
            run("IoSelfTest", "--mode=gauss", "--in=" + src, "--width=%d" % w, "--height=%d" % h, "--size=%d" % radius,
                "--out=" + out)
            blurred.append(np.fromfile(out, np.uint16).reshape(h, w, 3))
        want = cuda.foreground_mask(blurred[0], blurred[1], 0, 0.04, 4)
        got = cv2.imread(str(mdir / cid / "000007.png"), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(got, want * 255), (radius, cid)
