"""GPU tests of the sweep-view slices (include/derp_sweepview.h) against the reference's own GenerateCameraOverlaps.cpp
and GenerateEquirect.cpp (the checkers of oracle/sweepview.mk).  Float planes are compared bit for bit (any two NaNs
equal); the only allowed differences come from the device's FTHETA atan2 polynomial in the source projection
(derp_camera.cuh), so RECTILINEAR rigs must match exactly and FTHETA rigs within 1 in 10^5 values."""
import os

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import sweep_oracle, sweep_util as su

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    return capi.SweepView(capi.load_cuda())


def _bound(kind, total):
    return 0 if kind == "RECTILINEAR" else total // 100000


@pytest.mark.parametrize("kind,n,w,h,scale,slices", [("FTHETA", 4, 64, 48, 1.0, 2), ("RECTILINEAR", 6, 57, 43, 1.0, 50),
                                                     ("FTHETA", 16, 201, 131, 0.25, 50), ("golden", 16, 3360, 2160,
                                                                                          0.0625, 2),
                                                     ("RECTILINEAR", 8, 101, 77, 0.5, 2)])
def test_overlaps_match_reference(gpu, kind, n, w, h, scale, slices):
    ref = sweep_oracle.load_overlaps_ref()
    if ref is None:
        pytest.skip("checker not built")
    descs = su.rig(kind, n, w, h, scale)
    ims = su.images(descs, seed=n)
    disp = su.slice_disparities(slices, 1, 10)
    if slices == 2:
        disp = np.concatenate([disp, np.array([1 / 0.1], np.float32)])  # inside the rig radius
    a = gpu.overlaps(descs, ims, n - 1, disp)
    b = ref.overlaps(descs, ims, n - 1, disp)
    diffs = su.diff_count(a, b)
    print("%s %d cams, %d values: %d differ" % (kind, n, a.size, diffs))
    assert diffs <= _bound(kind, a.size)
    assert np.isfinite(a).any()


@pytest.mark.parametrize("kind,n,res,height", [("FTHETA", 8, (64, 48), 37), ("RECTILINEAR", 6, (57, 43), 37),
                                               ("golden", 16, (3360 * 0.05, 2160 * 0.05), 512)])
@pytest.mark.parametrize("black_bg,center,crop", [(False, -1, False), (True, 2, True), (False, -1, True)])
def test_equirect_match_reference(gpu, kind, n, res, height, black_bg, center, crop):
    ref = sweep_oracle.load_equirect_ref()
    if ref is None:
        pytest.skip("checker not built")
    if kind == "golden":
        descs = su.rig("golden", 16, 0, 0, 0.05)
    else:
        descs = su.rig(kind, n, res[0], res[1])
    ims = su.images(descs, seed=1)
    # with a crop the nearest depth stays outside the rig radius, where some camera sees every slice
    depths = su.equirect_depths(2 if height == 512 else 4, 0.5 if crop else 0.1, 10.0)
    bounds = None
    if crop:
        gb = gpu.crop_bounds(descs, height, depths, center=center)
        rb = ref.crop_bounds(descs, height, depths, center=center)
        box_diffs = int((gb != rb).sum())
        print("%s crop boxes: %d of %d values differ" % (kind, box_diffs, rb.size))
        assert box_diffs == 0
        bounds = gb
    a = gpu.equirect(descs, ims, height, depths, bounds=bounds, black_bg=black_bg, center=center)
    widths = [x.shape[1] for x in a]
    b = ref.equirect(descs, ims, height, depths, bounds=bounds, black_bg=black_bg, center=center, widths=widths)
    total = sum(x.size for x in a)
    diffs = sum(su.diff_count(x, y) for x, y in zip(a, b))
    print("%s %d cams, height %d, crop %s, %d values: %d differ" % (kind, n, height, crop, total, diffs))
    assert diffs <= _bound(kind, total)


def test_overlaps_full_size_one_destination(gpu):
    """One destination of the default shape (16-camera 3360 x 2160 ring, --scale 0.5) on a few slices."""
    ref = sweep_oracle.load_overlaps_ref()
    if ref is None:
        pytest.skip("checker not built")
    descs = su.rig("golden", 16, 0, 0, 0.5)
    ims = su.images(descs, seed=7)
    disp = su.slice_disparities(50, 1, 10)[[0, 25, 49]]
    a = gpu.overlaps(descs, ims, 3, disp)
    b = ref.overlaps(descs, ims, 3, disp)
    diffs = su.diff_count(a, b)
    print("full size: %d values, %d differ" % (a.size, diffs))
    assert a.shape == (3, 1080, 1680, 4)
    assert diffs <= a.size // 100000


def test_device_resident_images(gpu):
    """Images uploaded once with derp_device_alloc / derp_device_copy give the same slices as host images."""
    import torch
    descs = su.rig("FTHETA", 4, 64, 48)
    ims = su.images(descs, seed=2)
    disp = su.slice_disparities(5)
    dev = [torch.from_numpy(x).cuda() for x in ims]
    a = gpu.overlaps(descs, ims, 1, disp)
    ptrs = (capi.C.c_void_p * 4)(*[t.data_ptr() for t in dev])
    sizes = np.array([[x.shape[1], x.shape[0]] for x in ims], np.int32).reshape(-1)
    out = np.empty_like(a)
    rc = gpu.lib.derp_sweep_overlaps(0, descs, 4, ptrs, sizes.ctypes.data, 1, disp.ctypes.data, len(disp),
                                     out.ctypes.data)
    assert rc == 0
    assert su.diff_count(a, out) == 0


def test_hit_counter(gpu):
    """derp_sweep_last_hits counts the (sample, camera) pairs whose camera saw the point."""
    descs = su.rig("FTHETA", 4, 64, 48)
    ims = su.images(descs, seed=2)
    a = gpu.overlaps(descs, ims, 0, su.slice_disparities(3))
    hits = gpu.last_hits()
    inside = np.isfinite(a[..., 0]) & (a[..., 3] != 0)
    assert inside.sum() <= hits <= a.shape[0] * a.shape[1] * a.shape[2] * 4
    gpu.equirect(descs, ims, 16, su.equirect_depths(2))
    assert 0 < gpu.last_hits() <= 2 * 16 * 32 * 4


def _expected_files(names, planes):
    """Slices written in index order: where two share a name, the later one is the file."""
    out = {}
    for n, p in zip(names, planes):
        out[n] = p
    return out


@pytest.mark.parametrize("kind", ["FTHETA", "RECTILINEAR"])
def test_overlaps_app_end_to_end(tmp_path, kind):
    ref = sweep_oracle.load_overlaps_ref()
    if ref is None:
        pytest.skip("checker not built")
    import subprocess
    rig_path, color, rig = su.dataset(str(tmp_path), kind, 5, 45, 31, seed=4)
    app = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin", "GenerateCameraOverlaps")
    p = subprocess.run([app, "--rig=" + rig_path, "--color=" + color, "--output=" + str(tmp_path / "out"),
                        "--scale=1", "--num_depths=20", "--min_depth_m=1", "--max_depth_m=30", "--cameras=cam1,cam3"],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    assert "Loading images..." in p.stderr and "Depth 20 of 20..." in p.stderr
    descs = capi.rescaled_descs(capi.rig_descs(rig), 1.0)
    ims = [su.area_scaled(su.read_png(os.path.join(color, c["id"], "000000.png")), 1) for c in rig["cameras"]]
    disp = su.slice_disparities(20, 1, 30)
    names = ["%05d_cm.png" % int(np.float32(np.float32(1) / d) * np.float32(100)) for d in disp]
    total = diffs = 0
    for dst in (1, 3):
        planes = ref.overlaps(descs, ims, dst, disp)
        want = _expected_files(names, planes)
        cam_dir = tmp_path / "out" / "overlaps" / rig["cameras"][dst]["id"]
        assert sorted(os.listdir(cam_dir)) == sorted(want)
        for name, plane in want.items():
            got = su.read_png(str(cam_dir / name))
            exp = su.to_png8(plane)
            total += got.size
            diffs += int((got != exp).sum())
    print("%s overlaps app: %d of %d bytes differ" % (kind, diffs, total))
    assert diffs <= _bound(kind, total)


@pytest.mark.parametrize("crop,extra", [(False, ["--black_bg"]), (True, ["--camera_id=cam2"])])
def test_equirect_app_end_to_end(tmp_path, crop, extra):
    ref = sweep_oracle.load_equirect_ref()
    if ref is None:
        pytest.skip("checker not built")
    import subprocess
    rig_path, color, rig = su.dataset(str(tmp_path), "FTHETA", 6, 40, 30, seed=5)
    app = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin", "GenerateEquirect")
    args = [app, "--rig=" + rig_path, "--color=" + color, "--output=" + str(tmp_path / "out"), "--height=37",
            "--num_depths=5", "--depth_min=0.5", "--depth_max=10", "--cameras=cam0,cam2,cam3,cam5"] + extra
    if crop:
        args.append("--crop_equirect")
    p = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-1500:]
    keep = [0, 2, 3, 5]
    sub = {"cameras": [rig["cameras"][i] for i in keep]}
    descs = capi.rescaled_descs(capi.rig_descs(sub), 1.0)
    ims = [su.area_scaled(su.read_png(os.path.join(color, rig["cameras"][i]["id"], "000000.png")), 1) for i in keep]
    depths = su.equirect_depths(5, 0.5, 10.0)
    center = 1 if crop else -1
    bounds = ref.crop_bounds(descs, 37, depths, center=center) if crop else None
    widths = None if not crop else [capi.SweepView(capi.load_cuda()).crop_width(37, b) for b in bounds]
    planes = ref.equirect(descs, ims, 37, depths, bounds=bounds, black_bg="--black_bg" in extra, center=center,
                          widths=widths)
    names = ["%05d_cm.png" % int(float(d) * 100) for d in depths]
    want = _expected_files(names, planes)
    out_dir = tmp_path / "out" / "equirect"
    assert sorted(os.listdir(out_dir)) == sorted(want)
    total = diffs = 0
    for name, plane in want.items():
        got = su.read_png(str(out_dir / name))
        exp = su.to_png8(plane)
        assert got.shape == exp.shape
        total += got.size
        diffs += int((got != exp).sum())
    print("equirect app (crop %s): %d of %d bytes differ" % (crop, diffs, total))
    assert diffs <= total // 100000
