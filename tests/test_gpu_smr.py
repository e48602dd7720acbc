"""SimpleMeshRenderer on the GPU: derp_canopy_render against the CPU checker in every projection and mode, and the app
end to end after DerpCLI in all nine formats.  Everything is seeded."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import canopy_oracle
from tests.test_gpu_rephoto import _derpcli_disparities, check_disparity_colour

pytestmark = pytest.mark.gpu
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")


@pytest.fixture(scope="module")
def gcuda():
    return capi.Canopy(capi.load_cuda())


@pytest.fixture(scope="module")
def goracle():
    return canopy_oracle.load()


def _bgra(img_u16):
    h, w = img_u16.shape[:2]
    return np.concatenate([img_u16.astype(np.float32) * np.float32(1 / 65535), np.ones((h, w, 1), np.float32)], -1)


def _rig(case, W):
    if case == "ring16":
        return synth.ring_rig(16, W, W, kind="FTHETA")
    return synth.wall_rig(8, W, W, kind="RECTILINEAR")


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("case", ["ring16", "wall8"])
@pytest.mark.parametrize("projection", ["cubemap", "equirect", "perspective"])
@pytest.mark.parametrize("blend,ipd", [(True, 0.0), (False, 0.032), (True, -0.032)])
def test_canopy_matches_checker(gcuda, goracle, case, projection, blend, ipd):
    """Mesh at 48^2, colour at twice that size (so the colour and disparity-colour scenes raster separately)."""
    W = 48
    rig = _rig(case, W)
    colors, disps = synth.render_rig(rig, 2 * W, 2 * W, scene=synth.Scene(seed=7))
    disps = [np.ascontiguousarray(d[::2, ::2]) for d in disps]
    bgra = [_bgra(c) for c in colors]
    descs = capi.rig_descs(rig)
    pos = np.float32([0.01, -0.02, 0.005])
    size, matrix = {"cubemap": ((40, 40), None), "equirect": ((80, 40), None),
                    "perspective": ((72, 40), capi.snapshot_matrix(pos, [0.3, 0.9, 0.1], [0, 0, 1], 100.0, 72, 40))}[projection]
    out = []
    for lib in (gcuda, goracle):
        kw = dict(projection=projection, size=size, matrix=matrix, ipd=ipd, alpha_blend=blend, want_winners=True)
        c, _, wc = lib.render(descs, disps, bgra, pos, want_disparity=False, **kw)
        _, d, wd = lib.render(descs, disps, bgra, pos, want_color=False, want_disparity=True, **kw)
        out.append((c, wc, d, wd))
    (gc, gwc, gd, gwd), (oc, owc, od, owd) = out
    assert np.array_equal(gwc, owc) and np.array_equal(gwd, owd), (int((gwc != owc).sum()), int((gwd != owd).sum()))
    assert (gwc >= 0).any(axis=0).mean() > (0.5 if case == "ring16" else 0.1)
    assert _same(gc, oc), float(np.nanmax(np.abs(gc - oc)))
    assert np.array_equal(gd[..., 3] > 0, od[..., 3] > 0)
    # disparity colour: a rare value one RGBA16 step apart (check_disparity_colour says why)
    check_disparity_colour(gd, od, (case, projection, blend, ipd))


def test_shared_raster_matches_separate_scenes(gcuda):
    """With colour at the mesh's size one raster serves both scenes; it must equal two separate renders."""
    W = 48
    rig = _rig("ring16", W)
    colors, disps = synth.render_rig(rig, W, W, scene=synth.Scene(seed=8))
    bgra = [_bgra(c) for c in colors]
    descs = capi.rig_descs(rig)
    pos = np.zeros(3, np.float32)
    both = gcuda.render(descs, disps, bgra, pos, "equirect", (96, 48), ipd=0.032, want_disparity=True)
    c = gcuda.render(descs, disps, bgra, pos, "equirect", (96, 48), ipd=0.032)[0]
    d = gcuda.render(descs, disps, bgra, pos, "equirect", (96, 48), ipd=0.032, want_color=False, want_disparity=True)[1]
    assert _same(both[0], c) and _same(both[1], d)


def _png16(goracle, img):
    f = goracle.lib.oracle_smr_png16
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    img = np.ascontiguousarray(img, np.float32)
    out = np.empty(img.shape[:2] + (3,), np.uint16)
    f(img.ctypes.data, img.shape[0] * img.shape[1], out.ctypes.data)
    return out


def test_app_all_formats_end_to_end(gcuda, goracle, tmp_path):
    """scripts/test/test_simple_mesh_renderer.py: after DerpCLI, every format renders; each file has the format's shape
    and equals the binding's output through the app's png conversion."""
    W, S, width = 64, 8, 96
    h = width // 2
    rig = synth.ring_rig(S, W, W, kind="FTHETA")
    colors, _ = synth.render_rig(rig, W, W, scene=synth.Scene(seed=5))
    inp, lvl0, disps = _derpcli_disparities(tmp_path, rig, colors, W)
    color_dir = inp + "/video/color_levels/level_0"
    bgra = [_bgra(cv2.imread(os.path.join(color_dir, c["id"], "000000.png"), cv2.IMREAD_UNCHANGED))
            for c in rig["cameras"]]
    descs = capi.rig_descs(rig)
    pos = np.zeros(3, np.float32)

    def eqr(disp, ipd=0.0):
        return gcuda.render(descs, disps, bgra, pos, "equirect", (2 * h, h), ipd=ipd, want_color=not disp,
                            want_disparity=disp)[1 if disp else 0]

    snap_m = capi.snapshot_matrix(pos, [-1, 0, 0], [0, 0, 1], 90.0, width, h)
    left, right = eqr(False, 0.032), eqr(False, -0.032)
    expect = {
        "eqrcolor": eqr(False), "eqrdisp": eqr(True),
        "cubecolor": gcuda.render(descs, disps, bgra, pos, "cubemap", (h, h))[0],
        "cubedisp": gcuda.render(descs, disps, bgra, pos, "cubemap", (h, h), want_color=False, want_disparity=True)[1],
        "tbstereo": np.concatenate([left, right], 0),
        "lr180": np.concatenate([left[:, h // 2:h // 2 + h], right[:, h // 2:h // 2 + h]], 1),
        "tb3dof": np.concatenate([eqr(False), eqr(True)], 0),
        "snapcolor": gcuda.render(descs, disps, bgra, pos, "perspective", (width, h), snap_m)[0],
        "snapdisp": gcuda.render(descs, disps, bgra, pos, "perspective", (width, h), snap_m, want_color=False,
                                 want_disparity=True)[1],
    }
    shapes = {"eqrcolor": (h, 2 * h), "eqrdisp": (h, 2 * h), "cubecolor": (6 * h, h), "cubedisp": (6 * h, h),
              "tbstereo": (2 * h, 2 * h), "lr180": (h, 2 * h), "tb3dof": (2 * h, 2 * h), "snapcolor": (h, width),
              "snapdisp": (h, width)}
    for fmt, want in expect.items():
        out = str(tmp_path / ("smr_" + fmt))
        p = subprocess.run([os.path.join(BIN, "SimpleMeshRenderer"), "--rig=" + inp + "/rigs/rig_calibrated.json",
                            "--color=" + color_dir, "--disparity=" + lvl0, "--output=" + out, "--first=000000",
                            "--last=000000", "--format=" + fmt, "--width=%d" % width], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-2000:]
        assert "Processing frame 000000" in p.stderr and "File saved in" in p.stderr
        img = cv2.imread(os.path.join(out, "000000.png"), cv2.IMREAD_UNCHANGED)
        assert img is not None and img.dtype == np.uint16 and img.shape == shapes[fmt] + (3,), (fmt, img.shape)
        assert np.array_equal(img, _png16(goracle, want)), fmt
        assert (img > 0).mean() > 0.2, fmt
