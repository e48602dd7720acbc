"""ProjectEquirectsToCameras and ProjectCamerasToEquirects on the H100: the CUDA library against the reference's own
per-pixel code (oracle/eqrproject.mk) with 0 differing bytes, the share of pixels the device leaves to the host, the
equirect export against the canopy checker, and both apps end to end, including a geometric round trip."""
import json
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import canopy_oracle
from tests import eqr_project_util as eu
from tests import sweep_util as su

pytestmark = pytest.mark.gpu
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")


@pytest.fixture(scope="module")
def gcuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return capi.SweepView(capi.load_cuda())


@pytest.fixture(scope="module")
def ref():
    lib = eu.load_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libeqrproject_ref.so has not been built")
    return lib


def _compare(gcuda, ref, descs, masks, depth, label):
    a = gcuda.project_masks(descs, masks, depth)
    host_px = gcuda.last_host_pixels()
    b = ref.project_masks(descs, masks, depth)
    total = sum(x.size for x in a)
    diff = sum(int((x != y).sum()) for x, y in zip(a, b))
    print("%s depth %g: %d pixels, %d differ, %d resolved on the host (%.4f %%)" %
          (label, depth, total, diff, host_px, 100.0 * host_px / total))
    assert diff == 0
    assert host_px < 0.01 * total
    return a


@pytest.mark.parametrize("kind", eu.KINDS + ["poles"])
@pytest.mark.parametrize("depth", [0.7, 3.0, 1000.0])
def test_library_matches_reference(gcuda, ref, kind, depth):
    """Every camera model; "poles" looks straight up and down; camera 0 of the rings looks along +x, so its centre
    column lies on the theta = 0 seam."""
    descs = eu.rig(kind, 4, 160, 120)
    _compare(gcuda, ref, descs, eu.checkerboards(len(descs), base=(512, 256)), depth, kind)


@pytest.mark.parametrize("width", [100, 1024])
def test_library_golden_rescaled(gcuda, ref, width):
    descs = eu.rescaled_to_width(ref, eu.rig("golden"), width)
    _compare(gcuda, ref, descs, eu.checkerboards(len(descs), base=(1024, 512)), 5.0, "golden --width %d" % width)


def test_library_golden_full_size(gcuda, ref):
    """The golden 16-camera rig at 3360 x 2160 with 4096 x 2048 masks."""
    descs = eu.rig("golden")
    _compare(gcuda, ref, descs, eu.checkerboards(len(descs), base=(4096, 2048)), 1000.0, "golden full size")


def test_device_resident_masks(gcuda, ref):
    import torch
    descs = eu.rig("FTHETA", 4, 160, 120)
    masks = eu.checkerboards(len(descs), base=(512, 256))
    dev = [torch.from_numpy(m).cuda() for m in masks]
    a = gcuda.project_masks(descs, [(d.data_ptr(), d.shape[1], d.shape[0]) for d in dev], 2.0)
    b = ref.project_masks(descs, masks, 2.0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- ProjectCamerasToEquirects -------------------------------------------------------------------------------------
def _read_png16(path):
    data = open(path, "rb").read()
    pos, idat, w, h, ch = 8, b"", 0, 0, 0
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        t, d = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if t == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", d[:10])
            assert depth == 16 and ctype == 6
            ch = 4
        elif t == b"IDAT":
            idat += d
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 2 * ch * w)
    assert (raw[:, 0] == 0).all()
    rgba = raw[:, 1:].copy().view(">u2").reshape(h, w, ch).astype(np.uint16)
    return rgba[..., [2, 1, 0, 3]]  # B, G, R, A


def _to16(bgra):
    v = (np.asarray(bgra, np.float32) * np.float32(65535.0)).astype(np.float32)
    ok = np.isfinite(v)
    return np.clip(np.rint(np.where(ok, v, 0)), 0, 65535).astype(np.uint16)


def _dataset(tmp, kind, n, w, h, white=False):
    rig, color, r = su.dataset(str(tmp), kind, n, w, h)
    if white:
        for c in r["cameras"]:
            su.write_png(os.path.join(color, c["id"], "000000.png"), np.full((h, w, 4), 255, np.uint8))
    return rig, color, r


@pytest.mark.parametrize("eqr_width", [64, 256])
def test_cameras_to_equirects_matches_canopy_checker(gcuda, tmp_path, eqr_width):
    rig, color, r = _dataset(tmp_path, "FTHETA", 3, 48, 32)
    out = tmp_path / "out"
    p = subprocess.run([os.path.join(BIN, "ProjectCamerasToEquirects"), "--rig=" + rig, "--color=" + color,
                        "--output=" + str(out), "--depth=2.5", "--eqr_width=%d" % eqr_width], capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    oracle = canopy_oracle.load()
    descs = capi.rig_descs(r)
    for i, c in enumerate(r["cameras"]):
        img = su.read_png(os.path.join(color, c["id"], "000000.png")).astype(np.float32) * np.float32(1.0 / 255.0)
        disp = np.full((32, 48), np.float32(1.0 / 2.5), np.float32)
        want, _, _ = oracle.render((capi.CameraDesc * 1)(descs[i]), [disp], [img], [0, 0, 0], projection="equirect",
                                   size=(eqr_width, eqr_width // 2), alpha_blend=False, shader="on_screen")
        got = _read_png16(str(out / c["id"] / "000000.png"))
        assert got.shape == (eqr_width // 2, eqr_width, 4)
        assert np.array_equal(got, _to16(want))
        assert (got[..., 3] > 0).any()


def test_apps_round_trip(gcuda, tmp_path):
    """A white camera image goes to an equirect; its alpha comes back through ProjectEquirectsToCameras as a mask.
    Every in-circle pixel more than 2 px from the sensor or image-circle edge must come back 255."""
    w, h, depth = 64, 48, 3.0
    rig, color, r = _dataset(tmp_path, "FTHETA", 2, w, h, white=True)
    for c in r["cameras"]:
        c["fov"] = 1.2  # an image circle inside the sensor
    json.dump(r, open(rig, "w"))
    eqr = tmp_path / "eqr"
    p = subprocess.run([os.path.join(BIN, "ProjectCamerasToEquirects"), "--rig=" + rig, "--color=" + color,
                        "--output=" + str(eqr), "--depth=%g" % depth, "--eqr_width=2048"], capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    masks = tmp_path / "masks"
    for c in r["cameras"]:
        a = _read_png16(str(eqr / c["id"] / "000000.png"))[..., 3]
        os.makedirs(masks / c["id"])
        eu.write_png_gray8(str(masks / c["id"] / "000000.png"), np.where(a > 32767, 255, 0).astype(np.uint8))
    back = tmp_path / "back"
    p = subprocess.run([os.path.join(BIN, "ProjectEquirectsToCameras"), "--rig=" + rig, "--eqr_masks=" + str(masks),
                        "--output=" + str(back), "--depth=%g" % depth], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    assert "Loading equirect masks..." in p.stderr and "output resolution: 64x48" in p.stderr
    descs = capi.rig_descs(r)
    for i, c in enumerate(r["cameras"]):
        m = eu.read_png_gray8(str(back / c["id"] / "000000.png"))
        assert m.shape == (h, w) and set(np.unique(m)) <= {0, 255}
        # the image circle: |sensor| < circle radius (FTHETA: focal * fov), with a 2 px margin
        d = descs[i]
        yy, xx = np.mgrid[0:h, 0:w] + 0.5
        cx = d.principal[0] if d.has_principal else w / 2
        cy = d.principal[1] if d.has_principal else h / 2
        rad = np.hypot((xx - cx), (yy - cy))
        inside = (rad < d.focal[0] * 1.2 - 2) & (xx > 2) & (xx < w - 2) & (yy > 2) & (yy < h - 2)
        assert inside.sum() > 100
        assert (m[inside] == 255).all(), int((m[inside] != 255).sum())


def test_equirects_to_cameras_app_matches_reference(gcuda, ref, tmp_path):
    """The app at --width with 1-pixel checkerboard masks: PNG bytes decode to the reference's mask * 255."""
    rig, _, r = _dataset(tmp_path, "RECTILINEAR", 3, 40, 30)
    masks = tmp_path / "masks"
    boards = eu.checkerboards(3, base=(128, 64))
    for c, b in zip(r["cameras"], boards):
        os.makedirs(masks / c["id"])
        eu.write_png_gray8(str(masks / c["id"] / "000000.png"), b * 255)
    out = tmp_path / "out"
    p = subprocess.run([os.path.join(BIN, "ProjectEquirectsToCameras"), "--rig=" + rig, "--eqr_masks=" + str(masks),
                        "--output=" + str(out), "--depth=4", "--width=46", "--cameras=cam2,cam0"],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    descs = capi.rig_descs(r)
    sel = {"cam0": 0, "cam2": 2}
    for cid, i in sel.items():
        d = eu.rescaled_to_width(ref, (capi.CameraDesc * 1)(descs[i]), 46)
        want = ref.project_masks(d, [boards[i]], 4.0)[0]
        got = eu.read_png_gray8(str(out / cid / "000000.png"))
        assert np.array_equal(got, want)
    assert not (out / "cam1").exists()
