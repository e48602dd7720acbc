"""derp_resize_area (include/derp_resize.h) and ResizeFrames, the render pipeline's pyramid resize (scripts/render/
resize.py), without a GPU: the golden vectors against live cv2, a numpy restatement of the 8-bit fixed-point enlarge pinned
to cv2, the level sizes against resize.py's arithmetic, the app's flag surface, its refusals and FATAL without a GPU, and
the header as C99 with its exports.  tests/test_gpu_resize_frames.py runs the library and the app on an H100."""
import json
import math
import os
import re
import struct
import subprocess
import zlib

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests.golden import gen_resize_vectors as gv

DERP_EINVAL = -1  # include/derp_b200.h
WIDTHS = [2048, 1024, 512, 256, 200, 128, 100, 80, 60, 50]  # scripts/render/config.py:46
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")
APP = os.path.join(BIN, "ResizeFrames")
GOLDEN_RIG = os.path.join(capi.ROOT, "tests", "golden", "sweep_rig16.json")
VECTORS = os.path.join(capi.ROOT, "tests", "golden", "resize_vectors.npz")


def level_sizes(resolution):
    """resize_camera's level sizes: height = round(ratio * width) (Python's round: half to even), height += height % 2."""
    ratio = resolution[1] / resolution[0]
    out = []
    for width in WIDTHS:
        height = round(ratio * width)
        height += height % 2
        out.append((width, height))
    return out


# ---- the golden vectors ------------------------------------------------------------------------------------------------
def test_vectors_match_opencv():
    """tests/golden/resize_vectors.npz is what this cv2 computes (when it is 4.13: the fixture pins that version)."""
    cv2 = pytest.importorskip("cv2")
    if not cv2.__version__.startswith("4.13"):
        pytest.skip("cv2 %s is not the 4.13 the vectors were made with" % cv2.__version__)
    vec = np.load(VECTORS)
    keys = set()
    for key, bits, ch, src, dst, content, seed, thr in gv.cases():
        keys.add(key)
        got = gv.cv_resize(gv.source(bits, ch, src[0], src[1], content, seed), dst, thr)
        assert gv.same_values(got, vec[key]), key
    assert keys == set(vec.files)


def test_vectors_cover_every_type_and_path():
    vec = np.load(VECTORS)
    for bits, dtype in gv.TYPES.items():
        for ch in gv.CHANNELS:
            for name, _, _ in gv.SHAPES:
                assert vec["%s_u%d_c%d_random" % (name, bits, ch)].dtype == dtype
    special = [vec[k] for k in vec.files if k.endswith("_special")]
    flat = np.concatenate([a.ravel() for a in special])
    assert np.isnan(flat).any() and np.isposinf(flat).any() and np.isneginf(flat).any()
    assert (np.signbit(flat) & (flat == 0)).any(), "a -0 result"
    thr = [vec[k] for k in vec.files if k.endswith("_thr127")]
    assert all(set(np.unique(a)) <= {0, 255} for a in thr) and any((a == 255).any() and (a == 0).any() for a in thr)


# ---- the 8-bit enlarge in fixed point ----------------------------------------------------------------------------------
def linear_axis(ssize, dsize, x_axis):
    """INTER_AREA's bilinear taps on one axis (resize.cpp, area_mode): s = floor(d * scale), f = (float)((d + 1) - (s + 1) /
    scale), folded to [0, 1) in float; on x, a column whose second tap passes the last one takes it alone from xmax on.
    Returns (s, fixed-point weights round((1 - f) * 2048) and round(f * 2048), xmax)."""
    inv = dsize / ssize
    scale = 1.0 / inv
    s_, w0, w1, xmax = [], [], [], dsize
    for d in range(dsize):
        s = math.floor(d * scale)
        f = np.float32((d + 1) - (s + 1) * inv)
        f = np.float32(0) if f <= 0 else np.float32(f - np.float32(math.floor(f)))
        if x_axis and s + 1 >= ssize:
            xmax = min(xmax, d)
            if s >= ssize - 1:
                f, s = np.float32(0), ssize - 1
        s_.append(s)
        w0.append(int(np.rint(np.float32(np.float32(1) - f) * np.float32(2048))))
        w1.append(int(np.rint(f * np.float32(2048))))
    return np.array(s_), np.array(w0, np.int64), np.array(w1, np.int64), xmax


def enlarge_u8(img, dw, dh, simd=True):
    """cv2.resize(INTER_AREA) of an 8-bit image when an axis grows: exact int rows (HResizeLinear, weights in 1/2048), then
    the columns with the SIMD rounding ((((r0 >> 4) * b0) >> 16) + (((r1 >> 4) * b1) >> 16) + 2) >> 2, or (simd=False)
    the scalar form (r0 * b0 + r1 * b1 + 2^21) >> 22."""
    img = img.reshape(img.shape[:2] + (-1,)).astype(np.int64)
    sh, sw = img.shape[:2]
    xs, xa, xb, xmax = linear_axis(sw, dw, True)
    ys, ya, yb, _ = linear_axis(sh, dh, False)
    x1 = np.minimum(xs + 1, sw - 1)
    two = (np.arange(dw) < xmax)[None, :, None]
    rows = np.where(two, img[:, xs] * xa[None, :, None] + img[:, x1] * xb[None, :, None], img[:, xs] * 2048)
    r0, r1 = rows[ys], rows[np.minimum(ys + 1, sh - 1)]
    b0, b1 = ya[:, None, None], yb[:, None, None]
    if simd:
        out = ((((r0 >> 4) * b0) >> 16) + (((r1 >> 4) * b1) >> 16) + 2) >> 2
    else:
        out = (r0 * b0 + r1 * b1 + (1 << 21)) >> 22
    return out.astype(np.uint8)


@pytest.mark.parametrize("src,dst", [((2048, 1365), (2048, 1366)), ((1920, 1080), (2048, 1152)), ((100, 37), (200, 80)),
                                     ((7, 5), (9, 8)), ((20, 10), (30, 7)), ((20, 10), (8, 15))])
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_u8_enlarge_model_matches_opencv(src, dst, channels):
    cv2 = pytest.importorskip("cv2")
    img = gv.source(8, channels, src[0], src[1], "random", src[0] + dst[1] + channels)
    want = gv.cv_resize(img, dst).reshape(dst[1], dst[0], -1)
    assert np.array_equal(enlarge_u8(img, *dst), want)
    if channels == 3 and src[1] < dst[1]:  # the rows grow: the scalar rounding is not OpenCV's
        assert not np.array_equal(enlarge_u8(img, *dst, simd=False), want)
    assert cv2.__version__


# ---- level sizes -------------------------------------------------------------------------------------------------------
def test_level_sizes_of_the_golden_rig():
    rig = json.load(open(GOLDEN_RIG))
    assert {tuple(c["resolution"]) for c in rig["cameras"]} == {(3360, 2160)}
    assert level_sizes((3360, 2160)) == [(2048, 1318), (1024, 658), (512, 330), (256, 166), (200, 130), (128, 82),
                                         (100, 64), (80, 52), (60, 40), (50, 32)]
    assert level_sizes((1920, 1080))[4] == (200, 112)  # ratio * width is exactly 112.5: half to even
    assert level_sizes((2048, 1365))[0] == (2048, 1366)


def write_rig(path, resolutions, ids=None):
    from facebook360_dep_b200 import synth
    rig = synth.ring_rig(len(resolutions), 64, 64, kind="FTHETA")
    for i, (cam, res) in enumerate(zip(rig["cameras"], resolutions)):
        cam["resolution"] = list(res)
        if ids:
            cam["id"] = ids[i]
    json.dump(rig, open(path, "w"))
    return [c["id"] for c in rig["cameras"]]


def png8(path, w, h, colour_type, channels):
    """An 8-bit PNG of zeros with the given colour type (4: gray + alpha, which cv2 does not write)."""
    def chunk(t, data):
        return struct.pack(">I", len(data)) + t + data + struct.pack(">I", zlib.crc32(t + data) & 0xffffffff)
    raw = b"".join(b"\0" + bytes(channels * w) for _ in range(h))
    open(path, "wb").write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, colour_type, 0, 0, 0)) +
                           chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def png_gray(path, w, h):
    png8(path, w, h, 0, 1)


def png_gray_alpha(path, w, h):
    png8(path, w, h, 4, 2)


def dataset(tmp, resolutions, frames=("000000",), ext=".png", ids=None):
    """A rig of cameras at `resolutions` and a small 8-bit gray PNG per camera and frame, under `ext` (a file of another
    extension is never read)."""
    os.makedirs(tmp / "src", exist_ok=True)
    ids = write_rig(tmp / "rig.json", resolutions, ids)
    for cid, (w, h) in zip(ids, resolutions):
        os.makedirs(tmp / "src" / cid, exist_ok=True)
        for f in frames:
            png_gray(tmp / "src" / cid / (f + ext), 4, 3)
    return ids


def run(tmp, *args):
    return subprocess.run([APP, "--rig=" + str(tmp / "rig.json"), "--src_dir=" + str(tmp / "src"),
                           "--dst_dir=" + str(tmp / "dst")] + list(args), capture_output=True, text=True)


def no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


@pytest.mark.parametrize("resolutions", [[(3360, 2160)], [(1920, 1080), (2048, 1365)], [(1001, 777), (333, 555)],
                                         [(1280.5, 721.25), (4000, 2999)]])
def test_app_level_sizes(tmp_path, resolutions):
    """The sizes the app logs for each camera (before it needs a GPU) are resize.py's, also for odd heights and rig
    resolutions that are not integers."""
    no_gpu()
    ids = dataset(tmp_path, resolutions)
    r = run(tmp_path)
    assert r.returncode != 0
    for cid, res in zip(ids, resolutions):
        m = re.search(r"levels of %s:((?: \d+x\d+)+)" % re.escape(cid), r.stderr)
        assert m, r.stderr[-2000:]
        got = [tuple(int(v) for v in s.split("x")) for s in m.group(1).split()]
        assert got == level_sizes(res), (cid, res)


# ---- flags, refusals, no GPU -------------------------------------------------------------------------------------------
def test_flag_surface():
    """resize.py's flags (--src_dir --dst_dir --rig --first --last), the pipeline's --threshold and --gpu."""
    src = open(os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host", "ResizeFrames.cpp")).read()
    found = {m.group(2): (m.group(1), m.group(3).strip()) for m in
             re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,', src)}
    assert found == {"dst_dir": ("string", '""'), "first": ("string", '""'), "last": ("string", '""'),
                     "rig": ("string", '""'), "src_dir": ("string", '""'), "threshold": ("int32", "-1"),
                     "gpu": ("int32", "0")}
    h = subprocess.run([APP, "--help"], capture_output=True, text=True)
    for flag in found:
        assert "-" + flag + " " in h.stdout, flag


def test_refusals(tmp_path):
    """Each check stops the app with a message before any image is resized or any level directory is made."""
    cases = []
    a = tmp_path / "ext"
    dataset(a, [(64, 48)], ext=".jpg")
    cases.append((a, [], "only .png and .pfm"))
    b = tmp_path / "two"  # the 2-channel image is the last one: every header is read before any image is resized
    ids = dataset(b, [(64, 48), (64, 48)], frames=("000000", "000001"))
    png_gray_alpha(b / "src" / ids[-1] / "000001.png", 4, 3)
    cases.append((b, [], "2-channel images are not supported"))
    g = tmp_path / "colour_pfm"
    ids = dataset(g, [(64, 48)], ext=".pfm")
    open(g / "src" / ids[0] / "000000.pfm", "wb").write(b"PF\n4 3\n-1.0\n" + bytes(4 * 3 * 3 * 4))
    cases.append((g, [], "only 1-channel (Pf) .pfm"))
    m = tmp_path / "mixed"  # each camera's own extension: the second camera's .jpg is refused
    ids = dataset(m, [(64, 48), (64, 48)])
    os.rename(m / "src" / ids[1] / "000000.png", m / "src" / ids[1] / "000000.jpg")
    cases.append((m, [], "only .png and .pfm"))
    c = tmp_path / "dirs"
    dataset(c, [(64, 48), (64, 48)])
    os.makedirs(c / "src" / "extra")
    cases.append((c, [], "Cameras from rig differ"))
    d = tmp_path / "missing"
    ids = dataset(d, [(64, 48), (64, 48)], frames=("000003", "000004", "000005"))
    os.remove(d / "src" / ids[1] / "000004.png")
    cases.append((d, [], "Non-existent file for resize"))
    e = tmp_path / "range"
    dataset(e, [(64, 48)], frames=("000003", "000004"))
    cases.append((e, ["--first=000002"], "Non-existent file for resize"))
    for root, args, msg in cases:
        r = run(root, *args)
        assert r.returncode != 0 and msg in r.stderr, (root.name, r.stderr[-1500:])
        assert not (root / "dst").exists(), root.name
    assert subprocess.run([APP], capture_output=True, text=True).returncode != 0  # the required flags


def test_cv2_reads_pfm_rows_bottom_up(tmp_path):
    """cv2.imread, like imageio (FreeImage) in resize.py, hands out a PFM's rows last first, and cv2.imwrite stores them
    back in that order: resize_camera resizes a PFM that stores its top row first (io::writePfm, DerpCLI's disparities)
    upside down, and INTER_AREA is not symmetric under that flip.  ResizeFrames resizes the rows in the same order."""
    cv2 = pytest.importorskip("cv2")
    img = gv.source(32, 1, 30, 20, "random", 3)
    open(tmp_path / "a.pfm", "wb").write(b"Pf\n30 20\n-1.0\n" + img.tobytes())
    assert gv.same_values(cv2.imread(str(tmp_path / "a.pfm"), cv2.IMREAD_UNCHANGED), img[::-1].copy())
    assert cv2.imwrite(str(tmp_path / "b.pfm"), img)
    assert open(tmp_path / "b.pfm", "rb").read().endswith(img[::-1].tobytes())
    assert not gv.same_values(gv.cv_resize(img, (50, 33)), gv.cv_resize(img[::-1].copy(), (50, 33))[::-1])


def test_mixed_extensions_pass_the_checks(tmp_path):
    """A camera of .png frames next to one of .pfm frames: each camera's extension is its own, so the checks pass and
    the app stops only where it needs a GPU."""
    no_gpu()
    ids = dataset(tmp_path, [(64, 48), (64, 48)])
    os.remove(tmp_path / "src" / ids[1] / "000000.png")
    open(tmp_path / "src" / ids[1] / "000000.pfm", "wb").write(b"Pf\n4 3\n-1.0\n" + bytes(4 * 3 * 4))
    r = run(tmp_path)
    assert r.returncode != 0 and "derp_device_alloc" in r.stderr, r.stderr[-1500:]


def test_fatal_without_gpu(tmp_path):
    no_gpu()
    dataset(tmp_path, [(64, 48)])
    r = run(tmp_path)
    assert r.returncode != 0 and "derp_device_alloc" in r.stderr, r.stderr[-1500:]
    assert not (tmp_path / "dst").exists()


# ---- the ABI -----------------------------------------------------------------------------------------------------------
def test_bad_arguments():
    """Refused before any device is touched: bit depths, channel counts, sizes, byte counts that overflow, null pointers."""
    lib = capi.Resize(capi.load_cuda())
    img = np.zeros(64, np.float32)
    out = np.zeros(64, np.float32)
    f = lib.lib.derp_resize_area
    for bits, ch, sw, sh, dw, dh in ((12, 1, 4, 4, 2, 2), (64, 1, 4, 4, 2, 2), (8, 2, 4, 4, 2, 2), (8, 0, 4, 4, 2, 2),
                                     (8, 5, 4, 4, 2, 2), (8, 1, 0, 4, 2, 2), (8, 1, 4, -1, 2, 2), (8, 1, 4, 4, 0, 2),
                                     (8, 1, 4, 4, 2, 0), (32, 4, 2 ** 30, 2 ** 30, 2, 2), (32, 4, 2, 2, 2 ** 29, 2)):
        assert f(0, img.ctypes.data, bits, ch, sw, sh, out.ctypes.data, dw, dh, -1) == DERP_EINVAL, (bits, ch, sw, sh, dw, dh)
    assert f(0, None, 8, 1, 4, 4, out.ctypes.data, 2, 2, -1) == DERP_EINVAL
    assert f(0, img.ctypes.data, 8, 1, 4, 4, None, 2, 2, -1) == DERP_EINVAL
    with pytest.raises(ValueError):
        lib.resize_area(np.zeros((4, 4), np.int32), 2, 2)


def test_exports_every_declared_symbol():
    hdr = open(os.path.join(capi.ROOT, "include", "derp_resize.h")).read()
    declared = sorted(re.findall(r"^int (derp_[a-z0-9_]+)\(", hdr, re.M))
    assert declared == capi.RESIZE_SYMBOLS
    lib = capi.Resize(capi.load_cuda())
    for name in declared + ["derp_last_error"]:
        assert hasattr(lib.lib, name), name


def test_header_declares_it_in_c99(tmp_path):
    src = tmp_path / "resize.c"
    src.write_text('#include "derp_resize.h"\n#include <stdint.h>\n'
                   'int main(void) { uint8_t px[4] = {0, 0, 0, 0};\n'
                   '  return derp_resize_area(0, px, 8, 2, 1, 1, px + 2, 1, 1, -1) == DERP_EINVAL ? 0 : 1; }\n')
    exe = tmp_path / "resize"
    libdir = os.path.dirname(capi.CUDA_LIB)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", capi.ROOT + "/include",
                           str(src), "-o", str(exe), "-L", libdir, "-lderp_b200", "-Wl,-rpath," + libdir])
    assert subprocess.run([str(exe)]).returncode == 0
