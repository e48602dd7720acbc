"""CPU tests of the sweep-view slices (include/derp_sweepview.h): the product's DERP_HD per-pixel code run on the host,
and its host-side centerRig, against the reference's own GenerateCameraOverlaps.cpp / GenerateEquirect.cpp compiled
into the checkers of oracle/sweepview.mk.  On the host the camera model uses the C library's atan2, so FTHETA rigs
must match bit for bit here too."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import sweep_oracle, sweep_util as su


@pytest.fixture(scope="module")
def host():
    return capi.SweepView(capi.load_cuda(), host=True)


@pytest.fixture(scope="module")
def ov_ref():
    lib = sweep_oracle.load_overlaps_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libsweep_overlaps_ref.so has not been built")
    return lib


@pytest.fixture(scope="module")
def eq_ref():
    lib = sweep_oracle.load_equirect_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libsweep_equirect_ref.so has not been built")
    return lib


@pytest.mark.parametrize("kind,n,w,h,scale", [("FTHETA", 4, 40, 30, 1.0), ("RECTILINEAR", 6, 37, 29, 1.0),
                                               ("FTHETA", 5, 61, 45, 0.5)])
def test_overlaps_host_matches_reference(host, ov_ref, kind, n, w, h, scale):
    descs = su.rig(kind, n, w, h, scale)
    ims = su.images(descs, seed=n)
    disp = su.slice_disparities(2, 1, 10)
    disp = np.concatenate([disp, su.slice_disparities(5, 1, 10), np.array([1 / 0.05, 1 / 0.15], np.float32)])
    for dst in (0, n - 1):
        a = host.overlaps(descs, ims, dst, disp)
        b = ov_ref.overlaps(descs, ims, dst, disp)
        assert a.shape == b.shape
        assert su.diff_count(a, b) == 0
        assert np.isfinite(a).any()


@pytest.mark.parametrize("kind,n,res,height", [("FTHETA", 4, (40, 30), 17), ("RECTILINEAR", 6, (37, 29), 12)])
@pytest.mark.parametrize("black_bg", [False, True])
def test_equirect_host_matches_reference(host, eq_ref, kind, n, res, height, black_bg):
    descs = su.rig(kind, n, res[0], res[1])
    ims = su.images(descs, seed=3)
    depths = su.equirect_depths(3, 0.5, 10.0)
    a = host.equirect(descs, ims, height, depths, black_bg=black_bg)
    b = eq_ref.equirect(descs, ims, height, depths, black_bg=black_bg)
    for x, y in zip(a, b):
        assert su.diff_count(x, y) == 0
    for center in (-1, 1):
        bounds = eq_ref.crop_bounds(descs, height, depths, center=center)
        widths = [host.crop_width(height, bb) for bb in bounds]
        a = host.equirect(descs, ims, height, depths, bounds=bounds, black_bg=black_bg, center=center)
        b = eq_ref.equirect(descs, ims, height, depths, bounds=bounds, black_bg=black_bg, center=center, widths=widths)
        for x, y in zip(a, b):
            assert su.diff_count(x, y) == 0


@pytest.mark.parametrize("kind,center", [("golden", 0), ("golden", 5), ("golden", 15), ("FTHETA", 2),
                                         ("RECTILINEAR", 3)])
def test_center_rig_bit_identical(host, eq_ref, kind, center):
    descs = su.rig(kind, 8, 64, 48)
    _, ra, oa = host.center_rig(descs, center)
    _, rb, ob = eq_ref.center_rig(descs, center)
    assert np.array_equal(ra.view(np.uint64), rb.view(np.uint64))
    assert np.array_equal(oa.view(np.uint64), ob.view(np.uint64))
    # the centred camera looks at the equirect's centre (-1, 0, 0)
    assert np.allclose(-ra[center][2], [-1, 0, 0], atol=1e-9)


def test_crop_width_refusals(host):
    assert host.crop_width(512, [10, 30, 5, 25]) == int(512 / 20 * 20)
    for box in ([1024, 0, 512, 0], [10, 10, 5, 25], [10, 30, 5, 5]):
        with pytest.raises(capi.DerpError) as e:
            host.crop_width(512, box)
        assert e.value.code == capi.EINVAL and "nothing visible" in str(e.value)


def test_equirect_refuses_camera_larger_than_image(host):
    descs = su.rig("FTHETA", 4, 40, 30)
    ims = [x[:-1] for x in su.images(descs)]
    with pytest.raises(capi.DerpError) as e:
        host.equirect(descs, ims, 8, su.equirect_depths(2))
    assert e.value.code == capi.EINVAL and "exceeds its image" in str(e.value)


def test_sweep_header_is_plain_c_and_exported(tmp_path):
    hdr = open(os.path.join(capi.ROOT, "include", "derp_sweepview.h")).read()
    declared = sorted(set(re.findall(r"\b(derp_(?:test_)?sweep_[a-z0-9_]+)\s*\(", hdr)))
    assert declared == sorted(capi.SWEEP_SYMBOLS + capi.SWEEP_TEST_HOOKS)
    prod = C.CDLL(capi.CUDA_LIB, mode=C.RTLD_LOCAL)
    for name in declared:
        assert hasattr(prod, name), name
    src = tmp_path / "sweep.c"
    src.write_text('#include "derp_sweepview.h"\n#include <stdio.h>\nint main(void) { double b[4] = {0, 4, 0, 2}; '
                   'uint64_t w = 0; printf("%s\\n", derp_backend()); '
                   'if (derp_sweep_crop_width(8, b, &w) != DERP_OK || w != 16) return 2; '
                   'return derp_sweep_overlaps(0, 0, 0, 0, 0, 0, 0, 0, 0) == DERP_EINVAL ? 0 : 1; }\n')
    libdir = os.path.dirname(capi.CUDA_LIB)
    exe = tmp_path / "sweep"
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
    descs = su.rig("FTHETA", 2, 16, 16)
    with pytest.raises(capi.DerpError) as e:
        lib.overlaps(descs, su.images(descs), 0, su.slice_disparities(2))
    assert e.value.code == capi.ECUDA
