"""GenerateCameraOverlaps and GenerateEquirect without a GPU: the command lines against the reference's DEFINE lines,
the refusals where the reference is undefined, no CPU fallback, the slice tables and file names against the reference's
arithmetic, and the 8-bit conversion pinned to cv2 4.13 (tests/golden/sweep_vectors.npz, generator
tests/golden/gen_sweep_vectors.py)."""
import os
import re
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import sweep_util as su

HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "sweep_vectors.npz"))

# the reference's DEFINE lines: name -> (type, default, help)
REF_FLAGS = {
    "GenerateCameraOverlaps": {
        "cameras": ("string", "", "cameras to render (comma-separated)"),
        "color": ("string", "", "path to input color images (required)"),
        "frame": ("string", "000000", "frame to process (lexical)"),
        "max_depth_m": ("uint64", "10", "max depth in cm"),
        "min_depth_m": ("uint64", "1", "min depth in cm"),
        "num_depths": ("uint64", "50", "num depths"),
        "output": ("string", "", "path to output directory (required)"),
        "rig": ("string", "", "path to camera rig .json (required)"),
        "scale": ("double", "0.5", "image scale factor")},
    "GenerateEquirect": {
        "black_bg": ("bool", "false", "set the background to be optionally black (red by default)"),
        "camera_id": ("string", "", "id of camera selected to be centered"),
        "cameras": ("string", "", "cameras to render (comma-separated)"),
        "color": ("string", "", "path to input color images (required)"),
        "crop_equirect": ("bool", "false", "crop the equirect to only include visible images"),
        "depth_max": ("double", "10.0", "max depth in m"),
        "depth_min": ("double", "1.0", "min depth in m"),
        "frame": ("string", "000000", "frame to process (lexical)"),
        "height": ("uint64", "512", "equirect height in pixels"),
        "num_depths": ("uint64", "50", "num depths"),
        "output": ("string", "", "path to output directory (required)"),
        "rig": ("string", "", "path to camera rig .json (required)"),
        "scale": ("double", "1", "image scale factor"),
        "threads": ("int32", "-1", "number of threads (-1 = max allowed, 0 = no threading)")},
}


@pytest.fixture(scope="module")
def apps():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return BIN


@pytest.mark.parametrize("name", sorted(REF_FLAGS))
def test_flag_surface_matches_reference(apps, name):
    src = open(os.path.join(HOST, name + ".cpp")).read()
    found = {m.group(2): (m.group(1), m.group(3).strip('"'), m.group(4))
             for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*"([^"]*)"', src)}
    assert {k: v for k, v in found.items() if k != "gpu"} == REF_FLAGS[name]
    assert found["gpu"] == ("int32", "0", "CUDA device to use")
    h = subprocess.run([os.path.join(apps, name), "--help"], capture_output=True, text=True)
    for flag in REF_FLAGS[name]:
        assert "-" + flag + " " in h.stdout


def _run(apps, name, args):
    return subprocess.run([os.path.join(apps, name)] + args, capture_output=True, text=True, timeout=300)


def _inputs(tmp_path, w=24, h=16):
    rig, color, _ = su.dataset(str(tmp_path), "FTHETA", 3, w, h)
    return ["--rig=" + rig, "--color=" + color, "--output=" + str(tmp_path / "out")]


@pytest.mark.parametrize("name,bad,message", [
    ("GenerateCameraOverlaps", ["--num_depths=1"], "--num_depths must be at least 2"),
    ("GenerateCameraOverlaps", ["--num_depths=-3"], "num_depths"),
    ("GenerateCameraOverlaps", ["--cameras=nope"], "no destinations!"),
    ("GenerateCameraOverlaps", ["--rig="], "FLAGS_rig != \"\""),
    ("GenerateEquirect", ["--camera_id=nope"], "Camera id nope not found"),
    ("GenerateEquirect", ["--scale=1.02"], "larger than its scaled image"),
    ("GenerateEquirect", ["--color="], "FLAGS_color != \"\""),
])
def test_apps_refuse(apps, tmp_path, name, bad, message):
    p = _run(apps, name, _inputs(tmp_path) + bad)
    assert p.returncode != 0 and message in p.stderr, p.stderr[-800:]


@pytest.mark.parametrize("name", sorted(REF_FLAGS))
def test_fatal_without_gpu(apps, tmp_path, name):
    """No CPU fallback: without a GPU the first library call fails and the app stops with a FATAL error."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = _run(apps, name, _inputs(tmp_path) + ["--num_depths=2"])
    assert p.returncode != 0 and "failed:" in p.stderr and "Loading images..." in p.stderr, p.stderr[-800:]
    assert not any(f.endswith(".png") for _, _, fs in os.walk(tmp_path / "out") for f in fs)


# ---- host steps ----------------------------------------------------------------------------------------------------
_PROBE = r'''#include "sweep_host.h"
int main(int argc, char** argv) {
  const std::string what = argv[1];
  if (what == "overlaps") {
    for (float d : sweep_host::overlapDisparities(std::stoull(argv[2]), std::stoull(argv[3]), std::stoull(argv[4])))
      std::printf("%a %s\n", d, sweep_host::overlapFile(d).c_str());
  } else if (what == "equirect") {
    for (float d : sweep_host::equirectDepths(std::stoull(argv[2]), std::stod(argv[3]), std::stod(argv[4])))
      std::printf("%a %s\n", d, sweep_host::equirectFile(d).c_str());
  } else {
    std::vector<float> v;
    float x;
    while (std::fread(&x, 4, 1, stdin) == 1) v.push_back(x);
    const std::vector<uint8_t> o = sweep_host::toPng8(v.data(), v.size() / 4);
    std::fwrite(o.data(), 1, o.size(), stdout);
  }
  return 0;
}
'''


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    d = tmp_path_factory.mktemp("probe")
    (d / "p.cpp").write_text(_PROBE)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", HOST, str(d / "p.cpp"), "-o", str(d / "p"), "-lz",
                           "-pthread"])
    return str(d / "p")


def _lines(probe, *args):
    out = subprocess.run([probe] + [str(a) for a in args], capture_output=True, text=True, check=True).stdout.split("\n")
    return [(np.float32(float.fromhex(a)), b) for a, b in (l.split() for l in out if l)]


def _ref_overlaps(n, min_cm, max_cm):
    """GenerateCameraOverlaps.cpp:100-120 with ImageUtil.cpp:100-107 in the reference's types."""
    f32 = np.float32
    lo, hi = float(f32(1.0) / f32(min_cm)), float(f32(1.0) / f32(max_cm))
    out = []
    for d in range(n):
        frac = float(d) / float(n - 1)
        disp = f32(frac * lo + (1 - frac) * hi)
        depth_cm = f32(f32(f32(1.0) / disp) * f32(100))
        out.append((disp, "%05d_cm.png" % int(depth_cm)))
    return out


def _ref_equirect(n, dmin, dmax):
    """GenerateEquirect.cpp:264-281 and saveImage's int(depth * 100) on the double."""
    f32 = np.float32
    disp_min, disp_max = f32(1.0 / dmax), f32(1.0 / dmin)
    out = []
    for i in range(n - 1, -1, -1):
        frac = f32(f32(i) / f32(n - 1)) if n > 1 else f32(np.nan)
        disp = disp_min if n == 1 else f32(f32(frac * disp_min) + f32(f32(f32(1) - frac) * disp_max))
        depth = f32(f32(1.0) / disp)
        out.append((depth, "%05d_cm.png" % int(float(depth) * 100)))
    return out


@pytest.mark.parametrize("n,lo,hi", [(50, 1, 10), (2, 1, 10), (7, 3, 1000), (150, 1, 500), (13, 10, 10)])
def test_overlap_slices_and_names(probe, n, lo, hi):
    got, want = _lines(probe, "overlaps", n, lo, hi), _ref_overlaps(n, lo, hi)
    assert [(a.view(np.uint32), b) for a, b in got] == [(a.view(np.uint32), b) for a, b in want]


@pytest.mark.parametrize("n,lo,hi", [(50, 1.0, 10.0), (1, 1.0, 10.0), (2, 0.3, 7.7), (33, 0.1, 1000.0), (9, 2.0, 2.0)])
def test_equirect_slices_and_names(probe, n, lo, hi):
    got, want = _lines(probe, "equirect", n, lo, hi), _ref_equirect(n, lo, hi)
    assert [(a.view(np.uint32), b) for a, b in got] == [(a.view(np.uint32), b) for a, b in want]


def test_png_conversion_matches_cv2(probe):
    """imwrite(file, 255.0f * image): fp32 product, cvRound (ties to even), saturation, NaN and +-inf -> 0."""
    img = np.ascontiguousarray(G["img"], np.float32)
    out = subprocess.run([probe, "convert"], input=img.tobytes(), capture_output=True, check=True).stdout
    got = np.frombuffer(out, np.uint8).reshape(G["png"].shape)
    assert len(G["ties"]) > 20 and np.isnan(img).any() and np.isinf(img).any() and (img < 0).any()
    assert np.array_equal(got, G["png"])
    assert np.array_equal(su.to_png8(img), G["png"])  # the tests' restatement, used by the GPU end-to-end tests


def test_png_writer_round_trip(tmp_path):
    import cv2
    a = np.random.default_rng(1).integers(0, 256, (5, 7, 4), np.uint8)
    su.write_png(str(tmp_path / "a.png"), a)
    assert np.array_equal(cv2.imread(str(tmp_path / "a.png"), cv2.IMREAD_UNCHANGED), a)
    assert np.array_equal(su.read_png(str(tmp_path / "a.png")), a)
