"""ComputeRephotographyErrors without a GPU: the oracle's score against cv2 4.13 (tests/golden/rephoto_vectors.npz,
generator tests/golden/gen_rephoto_vectors.py), properties of the oracle's cubemap render, and the app's command line."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import rephoto_oracle

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "rephoto_vectors.npz"))
# the same score at edge shapes and radii (generator tests/golden/gen_rephoto_edge_vectors.py)
E = np.load(os.path.join(os.path.dirname(__file__), "golden", "rephoto_edge_vectors.npz"))
EDGE_CASES = ("odd", "cube", "tiny", "row", "col", "empty")
HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")
APP = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin", "ComputeRephotographyErrors")


@pytest.fixture(scope="module")
def oracle():
    """The CPU restatement of include/derp_rephoto.h (tests/rephoto_oracle.cpp), built into a temporary directory."""
    return rephoto_oracle.load()


def check_score_vs_cv2(score, avg, ref, ref_avg, mask):
    """test_score_matches_cv2's comparison: NaN where cv2 has NaN, scores within 1e-5, averages within 1e-6.  The
    tolerance is the class of cv2's float filters (test_oracle_cv.py): SIMD / FMA-dispatched sums, 1e-6 of the value
    scale per blur, amplified by the SSIM quotients."""
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(score), nan), int((np.isnan(score) != nan).sum())
    if not nan.all():
        assert np.abs(score - ref)[~nan].max() <= 1e-5, np.abs(score - ref)[~nan].max()
    assert np.abs(avg - ref_avg).max() <= 1e-6, (avg, ref_avg)
    if not mask.any():
        assert np.array_equal(avg, np.zeros(3))  # cv::mean over an empty mask


def edge_case(case, method, radius):
    """(x, y, mask, cv2 score, cv2 averages) of one edge-shape vector set"""
    return (E[case + "_x"], E[case + "_y"], E[case + "_mask"], E["%s_score_%s_r%d" % (case, method, radius)],
            E["%s_avg_%s_r%d" % (case, method, radius)])


@pytest.mark.parametrize("method", ["MSSIM", "NCC"])
@pytest.mark.parametrize("radius", [1, 2, 4, 5, 31])
def test_score_matches_cv2(oracle, method, radius):
    score, avg = oracle.rephoto_score(G["x"], G["y"], G["mask"], method, radius)
    src = G if radius <= 2 else {k[5:]: E[k] for k in E.files if k.startswith("base_")}
    ref = src["score_%s_r%d" % (method, radius)]
    nan = np.isnan(ref)
    assert nan.any() and (nan[..., 0] & (G["mask"] > 0)).any()  # NaN scores inside the mask are part of the case
    assert (~nan[..., 0] & (G["mask"] > 0)).any()
    check_score_vs_cv2(score, avg, ref, src["avg_%s_r%d" % (method, radius)], G["mask"])


@pytest.mark.parametrize("method", ["MSSIM", "NCC"])
@pytest.mark.parametrize("radius", [1, 2, 4, 5, 31])
@pytest.mark.parametrize("case", EDGE_CASES)
def test_score_edge_shapes_match_cv2(oracle, case, method, radius):
    """Odd non-square and cubemap-layout images, kernels wider than the image (reflect101 bouncing several times),
    1-pixel-wide and -tall images, NaN inputs inside the mask and an empty mask."""
    x, y, mask, ref, ref_avg = edge_case(case, method, radius)
    score, avg = oracle.rephoto_score(x, y, mask, method, radius)
    check_score_vs_cv2(score, avg, ref, ref_avg, mask)


def test_golden_score_vectors_unchanged():
    """rephoto_vectors.npz is the cv2 pin the GPU and CPU tests share; the edge vectors live in a file of their own."""
    h = hashlib.sha256()
    for k in sorted(G.files):
        a = G[k]
        h.update(k.encode())
        h.update(str(a.dtype).encode())
        h.update(str(a.shape).encode())
        h.update(np.ascontiguousarray(a).tobytes())
    assert len(G.files) == 18 and h.hexdigest() == "a6bd991d35e2b4bc67ebb7bf030c35581f06e04141ee3d065ba5282e234a9583"
    assert not any(k.startswith("base_") and k[5:] in G.files for k in E.files)


def _jet(oracle, score, mask):
    h, w = mask.shape
    f = oracle.lib.oracle_rephoto_jet_panel
    f.restype = None
    f.argtypes = [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p]
    s = np.ascontiguousarray(score, np.float32)
    m = np.ascontiguousarray(mask, np.uint8)
    out = np.empty((h, w, 3), np.uint8)
    f(s.ctypes.data, m.ctypes.data, w, h, out.ctypes.data)
    return out


def test_jet_panel_bit_exact(oracle):
    """stackResults' heat map (the app's rephoto_plot.h): convertTo 8 bit, 255 - x, applyColorMap(JET) of the 3-channel
    image, black outside the mask — byte for byte against cv2, including NaN, negative, > 1 and half-way scores."""
    for tag in ("MSSIM_r1", "NCC_r2"):
        assert np.array_equal(_jet(oracle, G["score_" + tag], G["mask"]), G["jet_" + tag])
    assert np.array_equal(_jet(oracle, G["wild"], G["mask"]), G["jet_wild"])
    ramp = np.repeat((np.arange(256, dtype=np.float32) / 255)[:, None, None], 3, 2)  # 255 - x walks the whole table
    assert np.array_equal(_jet(oracle, ramp, np.ones((256, 1), np.uint8))[::-1, 0], G["jet_lut"])


def _face_dirs(edge):
    """World direction of every pixel centre of the stacked cubemap (createCubemapTexture's face table)."""
    table = [((1, 0, 0), (0, 0, -1), (0, -1, 0)), ((-1, 0, 0), (0, 0, 1), (0, -1, 0)), ((0, 1, 0), (1, 0, 0), (0, 0, 1)),
             ((0, -1, 0), (1, 0, 0), (0, 0, -1)), ((0, 0, 1), (1, 0, 0), (0, -1, 0)), ((0, 0, -1), (-1, 0, 0), (0, -1, 0))]
    r, c = np.mgrid[0:edge, 0:edge].astype(np.float64)
    nx = (c + 0.5) / edge * 2 - 1
    ny = (edge - 1 - r + 0.5) / edge * 2 - 1  # GL rows count from the bottom
    out = []
    for ma, sc, tc in table:
        out.append(np.asarray(sc) * nx[..., None] + np.asarray(tc) * ny[..., None] + np.asarray(ma))
    return np.concatenate(out, 0)


def test_own_canopy_reproduces_its_image(oracle):
    """One camera at constant disparity rendered from its own centre: wherever the cubemap is covered, the colour is
    the trilinear sample of the camera's image where the pixel's ray meets the sensor.  The image is a linear ramp
    (B = (x + .5) / w, G = (y + .5) / h), which bilinear filtering and the box mips reproduce exactly, so the sample is
    the sensor coordinate itself."""
    W = H = 64
    rig = synth.wall_rig(1, W, H, kind="RECTILINEAR", hfov_deg=90.0)
    cam = rig["cameras"][0]
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    img = np.stack([(xx + 0.5) / W, (yy + 0.5) / H, np.full_like(xx, 0.25), np.ones_like(xx)], -1)
    disp = np.full((H, W), 0.5, np.float32)
    ctr = np.array(cam["origin"], np.float32)
    col, _, _ = oracle.rephoto_cubemap(capi.rig_descs(rig), [disp], [img], ctr, H)
    cov = col[..., 3] > 0
    assert 0.1 < cov.mean() < 0.5 and np.array_equal(col[..., 3][cov], np.ones(cov.sum(), np.float32))
    d = _face_dirs(H)
    fwd, right, up = (np.asarray(cam[k]) for k in ("forward", "right", "up"))
    f = cam["focal"]
    depth = d @ fwd
    with np.errstate(divide="ignore", invalid="ignore"):
        px = W / 2 + f[0] * (d @ right) / depth
        py = H / 2 + f[1] * (d @ up) / depth
    inner = cov & (np.abs(px / W - 0.5) < 0.35) & (np.abs(py / H - 0.5) < 0.35)
    assert inner.sum() > 500
    assert np.abs(col[..., 0][inner] * W - px[inner]).max() < 0.25
    assert np.abs(col[..., 1][inner] * H - py[inner]).max() < 0.25
    assert np.abs(col[..., 2][inner] - 0.25).max() < 2e-5  # the constant channel: the RGBA16 value of 0.25


def test_empty_others_give_empty_mask(oracle):
    rig = synth.ring_rig(2, 32, 32)
    col, dsp, _ = oracle.rephoto_cubemap(capi.rig_descs({"cameras": []}), [], [], np.zeros(3, np.float32), 32,
                                         want_disparity=True)
    assert not np.isnan(col).any() and not col.any() and not dsp.any()
    # a camera that sees nothing valid: disparity 0 (depth inf) drops every triangle
    col, _, wn = oracle.rephoto_cubemap(capi.rig_descs({"cameras": rig["cameras"][:1]}), [np.zeros((32, 32), np.float32)],
                                        [np.ones((32, 32, 4), np.float32)], np.zeros(3, np.float32), 32, want_winners=True)
    assert not col.any() and (wn == -1).all()


def test_canopies_blend_in_camera_order_with_equal_weights(oracle):
    """Two canopies of the same camera, disparity and alpha, differing only in colour: each canopy keeps its own
    surviving primitive per pixel (the same one, the later of equal-depth fragments in draw order), and the soft-max
    blend of equal weights is the mean colour."""
    W = 48
    rig = synth.ring_rig(1, W, W)
    cams = capi.rig_descs({"cameras": rig["cameras"] * 2})
    disp = np.full((W, W), 0.4, np.float32)
    a = np.zeros((W, W, 4), np.float32)
    a[...] = (0.2, 0.4, 0.6, 1)
    b = np.zeros((W, W, 4), np.float32)
    b[...] = (0.6, 0.2, 0.0, 1)
    ctr = np.array(rig["cameras"][0]["origin"], np.float32) + np.float32(0.05)
    col, _, wn = oracle.rephoto_cubemap(cams, [disp, disp], [a, b], ctr, W, want_winners=True)
    assert np.array_equal(wn[0], wn[1]) and (wn[0] >= 0).mean() > 0.2
    cov = (wn[0] >= 0) & (col[..., 3] > 0)  # a fragment whose weight expf(30 a) - 1 rounds to 0 leaves 0 / 0 -> 0
    assert cov.mean() > 0.2
    assert np.abs(col[cov][:, :3] - np.float32([0.4, 0.3, 0.3])).max() < 1e-4


# ComputeRephotographyErrors.cpp:46-54
REF_FLAGS = {"cameras": ("string", ""), "color": ("string", ""), "disparity": ("string", ""), "first": ("string", ""),
             "last": ("string", ""), "method": ("string", "MSSIM"), "output": ("string", ""), "rig": ("string", ""),
             "stat_radius": ("int32", "1")}


@pytest.fixture(scope="module")
def app():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return APP


def test_flag_surface_matches_reference(app):
    src = open(os.path.join(HOST, "ComputeRephotographyErrors.cpp")).read()
    found = {m.group(2): (m.group(1), m.group(3).strip('"'))
             for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*"', src)}
    assert {k: v for k, v in found.items() if k != "gpu"} == REF_FLAGS
    assert found["gpu"] == ("int32", "0")
    h = subprocess.run([app, "--help"], capture_output=True, text=True)
    for name in REF_FLAGS:
        assert "-" + name + " " in h.stdout


@pytest.mark.parametrize("bad,message", [
    (["--method=SSIM"], "invalid method SSIM"),
    (["--stat_radius=0"], "FLAGS_stat_radius > 0"),
    (["--rig="], "FLAGS_rig != \"\""),
])
def test_app_aborts_on_bad_flags(app, tmp_path, bad, message):
    rig = synth.ring_rig(2, 8, 8)
    json.dump(rig, open(tmp_path / "rig.json", "w"))
    args = ["--color=" + str(tmp_path), "--disparity=" + str(tmp_path), "--rig=" + str(tmp_path / "rig.json"),
            "--output=" + str(tmp_path / "out"), "--first=000000", "--last=000000"]
    p = subprocess.run([app] + args + bad, capture_output=True, text=True)
    assert p.returncode != 0 and message in p.stderr, p.stderr[-500:]


def test_rephoto_header_is_plain_c_and_exported(tmp_path, oracle):
    """include/derp_rephoto.h compiles as C99 and links against the product library alone; the product and the CPU
    checker export every entry point it declares, and the Python binding binds exactly those."""
    hdr = open(os.path.join(capi.ROOT, "include", "derp_rephoto.h")).read()
    declared = sorted(set(re.findall(r"\b(derp_rephoto_[a-z0-9_]+)\s*\(", hdr)))
    assert declared == capi.REPHOTO_SYMBOLS
    prod = C.CDLL(capi.CUDA_LIB, mode=C.RTLD_LOCAL)
    for name in declared:
        assert hasattr(prod, name) and hasattr(oracle.lib, name), name
    src = tmp_path / "rephoto.c"
    src.write_text('#include "derp_rephoto.h"\n#include <stdio.h>\nint main(void) { double avg[3]; '
                   'printf("%s\\n", derp_backend()); '
                   'return derp_rephoto_score(0, 0, 0, 0, 1, 1, DERP_REPHOTO_MSSIM, 1, 0, avg) == DERP_EINVAL ? 0 : 1; }\n')
    libdir = os.path.dirname(capi.CUDA_LIB)
    exe = tmp_path / "rephoto"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(capi.ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lderp_b200",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "cuda-sm_90a"


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rig = synth.ring_rig(2, 16, 16)
    lib = capi.Rephoto(capi.load_cuda())
    with pytest.raises(capi.DerpError) as e:
        lib.rephoto_cubemap(capi.rig_descs(rig), [np.ones((16, 16), np.float32)] * 2, [np.ones((16, 16, 4), np.float32)] * 2,
                            np.zeros(3, np.float32), 16)
    assert e.value.code == capi.ECUDA
    with pytest.raises(capi.DerpError) as e:
        lib.rephoto_score(np.zeros((6, 1, 3)), np.zeros((6, 1, 3)), np.ones((6, 1)))
    assert e.value.code == capi.ECUDA
