"""ProjectEquirectsToCameras and ProjectCamerasToEquirects without a GPU: the flag surfaces against the reference's DEFINE
lines, the refusals, no CPU fallback, the per-axis rescale against the reference's rescaleCameras, the product's DERP_HD
per-pixel projection run on the host against the reference's own code (oracle/eqrproject.mk), the acos / atan2
overload the reference resolves, and the header's exports."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import eqr_project_util as eu
from tests import sweep_util as su

HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")

REF_FLAGS = {
    "ProjectEquirectsToCameras": {
        "cameras": ("string", "", "comma-separated cameras to render (empty for all)"),
        "depth": ("double", "1000", "depth to project at (m)"),
        "eqr_masks": ("string", "", "path to input equirect masks (required)"),
        "file_type": ("string", "png", "Supports any image type allowed in OpenCV"),
        "first": ("string", "000000", "first frame to process (lexical) (required)"),
        "last": ("string", "000000", "last frame to process (lexical) (required)"),
        "output": ("string", "", "output directory (required)"),
        "rig": ("string", "", "path to camera rig .json (required)"),
        "threads": ("int32", "-1", "number of threads (-1 = auto, 0 = none)"),
        "width": ("int32", "0", "width of projected camera images (0 = size from rig file)")},
    "ProjectCamerasToEquirects": {
        "cameras": ("string", "", "comma-separated cameras to render (empty for all)"),
        "color": ("string", "", "path to input color images (required)"),
        "depth": ("double", "1000", "depth to project at (m)"),
        "eqr_width": ("int32", "1024", "equirect width (pixels)"),
        "file_type": ("string", "png", "Supports any image type allowed in OpenCV"),
        "first": ("string", "000000", "first frame to process (lexical)"),
        "last": ("string", "000000", "last frame to process (lexical)"),
        "output": ("string", "", "output directory (required)"),
        "rig": ("string", "", "path to camera rig .json (required)")},
}


@pytest.fixture(scope="module")
def host():
    return capi.SweepView(capi.load_cuda(), host=True)


@pytest.fixture(scope="module")
def ref():
    lib = eu.load_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libeqrproject_ref.so has not been built")
    return lib


@pytest.fixture(scope="module")
def apps():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return BIN


def _defines(name):
    src = open(os.path.join(HOST, name + ".cpp")).read()
    return {m.group(2): (m.group(1), m.group(3).strip('"'), m.group(4))
            for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*"([^"]*)"', src)}


@pytest.mark.parametrize("name", sorted(REF_FLAGS))
def test_flag_surface_matches_reference(apps, name):
    found = _defines(name)
    assert {k: v for k, v in found.items() if k != "gpu"} == REF_FLAGS[name]
    assert found["gpu"] == ("int32", "0", "CUDA device to use")
    h = subprocess.run([os.path.join(apps, name), "--help"], capture_output=True, text=True)
    for flag in REF_FLAGS[name]:
        assert "-" + flag + " " in h.stdout


def _dataset(tmp_path, w=24, h=16):
    rig, color, r = su.dataset(str(tmp_path), "FTHETA", 3, w, h)
    for c in r["cameras"]:
        os.makedirs(tmp_path / "masks" / c["id"], exist_ok=True)
        eu.write_png_gray8(str(tmp_path / "masks" / c["id"] / "000000.png"), np.full((32, 64), 255, np.uint8))
    return rig, color, str(tmp_path / "masks")


def _run(apps, name, args):
    return subprocess.run([os.path.join(apps, name)] + args, capture_output=True, text=True, timeout=300)


def _args(tmp_path, name):
    rig, color, masks = _dataset(tmp_path)
    inp = "--eqr_masks=" + masks if name == "ProjectEquirectsToCameras" else "--color=" + color
    return ["--rig=" + rig, inp, "--output=" + str(tmp_path / "out")]


@pytest.mark.parametrize("name,bad,message", [
    ("ProjectEquirectsToCameras", ["--eqr_masks="], 'FLAGS_eqr_masks != ""'),
    ("ProjectEquirectsToCameras", ["--rig="], 'FLAGS_rig != ""'),
    ("ProjectEquirectsToCameras", ["--output="], 'FLAGS_output != ""'),
    ("ProjectEquirectsToCameras", ["--first="], 'FLAGS_first != ""'),
    ("ProjectEquirectsToCameras", ["--depth=0"], "FLAGS_depth > 0"),
    ("ProjectEquirectsToCameras", ["--width=-2"], "FLAGS_width >= 0"),
    ("ProjectEquirectsToCameras", ["--width=33"], "equirect width must be a multiple of 2"),
    ("ProjectEquirectsToCameras", ["--cameras=nope"], "rig.cams.size() > 0"),
    ("ProjectEquirectsToCameras", ["--last=000001"], "missing file"),
    ("ProjectEquirectsToCameras", ["--file_type=jpg"], "this build writes png"),
    ("ProjectCamerasToEquirects", ["--color="], 'FLAGS_color != ""'),
    ("ProjectCamerasToEquirects", ["--depth=-1"], "FLAGS_depth > 0"),
    ("ProjectCamerasToEquirects", ["--eqr_width=-2"], "FLAGS_eqr_width >= 0"),
    ("ProjectCamerasToEquirects", ["--eqr_width=31"], "equirect width must be a multiple of 2"),
    ("ProjectCamerasToEquirects", ["--eqr_width=0"], "empty equirect"),
    ("ProjectCamerasToEquirects", ["--cameras=nope"], "rig.cams.size() > 0"),
    ("ProjectCamerasToEquirects", ["--last=000001"], "missing file"),
    ("ProjectCamerasToEquirects", ["--file_type=jpg"], "this build writes png"),
])
def test_apps_refuse(apps, tmp_path, name, bad, message):
    p = _run(apps, name, _args(tmp_path, name) + bad)
    assert p.returncode != 0 and message in p.stderr, p.stderr[-800:]
    assert not (tmp_path / "out").exists()


@pytest.mark.parametrize("name,log", [("ProjectEquirectsToCameras", "Loading equirect masks..."),
                                      ("ProjectCamerasToEquirects", "Loading colors...")])
def test_fatal_without_gpu(apps, tmp_path, name, log):
    """No CPU fallback: without a GPU the first library call fails and the app stops with a FATAL error."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = _run(apps, name, _args(tmp_path, name) + ["--width=20"] * (name == "ProjectEquirectsToCameras"))
    assert p.returncode != 0 and "failed:" in p.stderr and log in p.stderr, p.stderr[-800:]
    assert not any(f.endswith(".png") for _, _, fs in os.walk(tmp_path / "out") for f in fs)


# ---- rescaleCameras ------------------------------------------------------------------------------------------------
_PROBE = r'''#include "sweep_host.h"
int main(int argc, char** argv) {
  const io::Rig rig = io::loadRig(argv[1]);
  for (const DerpCameraDesc& c : rig.cams) {
    const DerpCameraDesc d = sweep_host::rescaledToWidth(c, std::stoi(argv[2]));
    std::printf("%a %a %a %a %a %a\n", d.resolution[0], d.resolution[1], d.principal[0], d.principal[1], d.focal[0],
                d.focal[1]);
  }
  return 0;
}
'''


@pytest.mark.parametrize("kind,w,h,width", [("golden", 0, 0, 1024), ("golden", 0, 0, 100), ("FTHETA", 40, 30, 46),
                                            ("RECTILINEAR", 37, 29, 50), ("EQUISOLID", 41, 27, 8)])
def test_rescale_matches_reference(ref, tmp_path, kind, w, h, width):
    """The per-axis rescale at --width, including heights that round to odd before the + 1."""
    import json
    r = eu.rig_json(kind, 3, w, h)
    json.dump(r, open(tmp_path / "rig.json", "w"))
    (tmp_path / "p.cpp").write_text(_PROBE)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", HOST, str(tmp_path / "p.cpp"), "-o", str(tmp_path / "p"),
                           "-lz", "-pthread"])
    out = subprocess.run([str(tmp_path / "p"), str(tmp_path / "rig.json"), str(width)], capture_output=True, text=True,
                         check=True).stdout.split("\n")
    want = eu.rescaled_to_width(ref, capi.rig_descs(r), width)
    for line, d in zip([l for l in out if l], want):
        got = [float.fromhex(v) for v in line.split()]
        assert got == [d.resolution[0], d.resolution[1], d.principal[0], d.principal[1], d.focal[0], d.focal[1]]


def test_rescale_cases_cover_odd_heights():
    """At least one case above has ceil(width * ry / float(rx)) odd, so the + 1 is exercised."""
    import math
    cases = [(40, 30, 46), (3360, 2160, 100)]
    odd = [math.ceil(W * ry / float(np.float32(rx))) % 2 for rx, ry, W in cases]
    assert all(odd)


# ---- the per-pixel projection on the host --------------------------------------------------------------------------
@pytest.mark.parametrize("kind", eu.KINDS + ["poles"])
@pytest.mark.parametrize("depth", [0.7, 3.0, 1000.0])
def test_host_projection_matches_reference(host, ref, kind, depth):
    descs = eu.rig(kind)
    masks = eu.checkerboards(len(descs))
    a = host.project_masks(descs, masks, depth)
    b = ref.project_masks(descs, masks, depth)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y)
    assert all(set(np.unique(x)) <= {0, 255} for x in a)
    assert sum(int((x == 255).sum()) for x in a) > 0


@pytest.mark.parametrize("width", [0, 100, 96])
def test_host_projection_golden_rig(host, ref, width):
    """The golden 16-camera rig, rescaled to --width by the reference's own rescaleCameras (at full size: width 0
    takes the first two cameras only, to keep the host run short)."""
    descs = eu.rig("golden")
    if width:
        descs = eu.rescaled_to_width(ref, descs, width)
    else:
        descs = (capi.CameraDesc * 2)(descs[0], descs[7])
    masks = eu.checkerboards(len(descs), base=(4096, 2048) if not width else (256, 128))
    a = host.project_masks(descs, masks, 5.0)
    b = ref.project_masks(descs, masks, 5.0)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_near_pole_is_defined(host, ref):
    """Cameras looking straight up and down, at the pixel of the pole: no crash, 0 or 255 as the reference decides."""
    descs = eu.rig("poles", w=41, h=41)
    masks = [np.ones((8, 16), np.uint8), np.ones((9, 18), np.uint8)]
    a = host.project_masks(descs, masks, 2.0)
    b = ref.project_masks(descs, masks, 2.0)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert a[1][20, 20] == 255  # the exact pole (z = -1) reads the bottom row


def test_reference_resolves_float_acos_and_atan2():
    """worldToEquirect (ImageUtil.cpp:127-140) calls acosf and atan2f: the float overloads, which the product uses."""
    obj = os.path.join(capi.ROOT, "oracle", "_ref", "ImageUtil.o")
    if not os.path.exists(obj):
        pytest.skip("oracle/_ref/ImageUtil.o has not been built")
    dis = subprocess.run(["objdump", "-dr", "--no-show-raw-insn", "-C", obj], capture_output=True, text=True,
                         check=True).stdout
    body = re.search(r"\n[0-9a-f]+ <fb360_dep::image_util::worldToEquirect\(.*?>:\n(.*?)\n\n", dis, re.S).group(1)
    calls = re.findall(r"R_X86_64_PLT32\s+(\w+)", body)
    assert calls == ["acosf", "atan2f"], calls


def test_refusals(host):
    descs = eu.rig("FTHETA", 2, 16, 12)
    masks = eu.checkerboards(2)
    for depth in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(capi.DerpError) as e:
            host.project_masks(descs, masks, depth)
        assert e.value.code == capi.EINVAL
    with pytest.raises(capi.DerpError):
        host.project_masks(descs, [masks[0], np.zeros((0, 4), np.uint8)], 1.0)


def test_project_header_is_plain_c_and_exported(tmp_path):
    hdr = open(os.path.join(capi.ROOT, "include", "derp_sweepview.h")).read()
    declared = sorted(set(re.findall(r"\b(derp_(?:test_)?project_[a-z0-9_]+)\s*\(", hdr)))
    assert declared == sorted(capi.PROJECT_SYMBOLS)
    prod = C.CDLL(capi.CUDA_LIB, mode=C.RTLD_LOCAL)
    for name in declared:
        assert hasattr(prod, name), name
    src = tmp_path / "p.c"
    src.write_text('#include "derp_sweepview.h"\n#include <stdio.h>\nint main(void) { printf("%s\\n", derp_backend()); '
                   'if (derp_project_last_host_pixels() != 0) return 2; '
                   'return derp_project_equirect_masks(0, 0, 0, 1.0, 0, 0, 0) == DERP_EINVAL ? 0 : 1; }\n')
    libdir = os.path.dirname(capi.CUDA_LIB)
    exe = tmp_path / "p"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(capi.ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lderp_b200",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "cuda-sm_90a", (out.returncode, out.stdout)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = capi.SweepView(capi.load_cuda())
    descs = eu.rig("FTHETA", 2, 16, 12)
    with pytest.raises(capi.DerpError) as e:
        lib.project_masks(descs, eu.checkerboards(2), 1.0)
    assert e.value.code == capi.ECUDA
