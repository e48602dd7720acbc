"""The host half of the interval proofs' premises (derp_interval.cuh, derp_rigsim.cuh): glibc's sin, cos, atan, asin,
atan2, acosf and atan2f are within the budgeted 2 ulp of the exact value (mpmath) on the adversarial argument sets the
GPU test also runs, and the host twins of the device probes agree with each other where they describe one value."""
import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import interval_util as iu

FNS = ["sin", "cos", "atan", "asin", "atan2", "acosf", "atan2f"]


@pytest.mark.parametrize("fn", FNS)
def test_glibc_within_budget(fn):
    a, b = iu.adversarial(fn)
    err = iu.ulp_errors(fn, a, b, iu.host(fn, a, b))
    print("glibc %s: %d arguments, max %.3f ulp" % (fn, len(a), err.max()))
    assert err.max() <= iu.HOST_ULPS, (fn, a[err.argmax()], None if b is None else b[err.argmax()], err.max())


def test_sky_texel_host_twin_is_the_references_formula():
    """skyTexelHost against RigSimulator.cpp:224-231 written out in numpy with glibc's acosf / atan2f."""
    lib = capi.RigSim(capi.load_cuda())
    rng = np.random.default_rng(3)
    d = rng.normal(size=(4000, 3)).astype(np.float32)
    d[:50, 1] = 0  # the seam
    d[50:100, 1] = -0.0
    d[:100, 0] = -np.abs(d[:100, 0])
    rows, cols = 37, 75
    got = lib.sky_texel(d, rows, cols, host=True)
    for (x, y, z), (row, col) in zip(d, got):
        phi = np.float32(iu.LIBM.acosf(float(np.clip(z, np.float32(-1), np.float32(1)))))
        theta = np.float32(np.pi + float(np.float32(iu.LIBM.atan2f(float(y), float(x)))))
        sx = np.float32((float(theta) / (2 * np.pi)) * cols)
        sy = np.float32((float(phi) / np.pi) * rows)
        assert (row, col) == (min(int(sy), rows - 1), int(sx) % cols)


def test_count_timing_host_twin_matches_equirect_host():
    """countTiming at arbitrary points (the provenCount twin) equals the equirect host loop at its pixel points."""
    import json
    import os
    ra = capi.RigAnalysis(capi.load_cuda())
    rig = json.load(open(os.path.join(capi.ROOT, "tests", "golden", "sweep_rig16.json")))
    descs = capi.rig_descs(rig)
    W, H, dist = 24, 12, 2.5
    counts, timing = ra.equirect(descs, W, H, dist, host=True)
    lat = np.pi / 2 - (np.arange(H) + 0.5) / H * np.pi
    lon = -np.pi + (np.arange(W) + 0.5) / W * 2 * np.pi
    cl, sl = np.array([iu.LIBM.cos(v) for v in lat]), np.array([iu.LIBM.sin(v) for v in lat])
    co, so = np.array([iu.LIBM.cos(v) for v in lon]), np.array([iu.LIBM.sin(v) for v in lon])
    pts = np.stack([cl[:, None] * co[None, :] * dist, cl[:, None] * so[None, :] * dist,
                    np.repeat(sl[:, None] * dist, W, 1)], -1).reshape(-1, 3)
    c2, t2 = ra.proven_count(descs, pts, host=True)
    assert np.array_equal(c2, counts.ravel())
    assert np.array_equal(t2.view(np.uint32), timing.ravel().view(np.uint32))


@pytest.mark.parametrize("kind,fov,dist", iu.SEES_CAMERAS)
def test_count_timing_host_twin_matches_checker_at_boundaries(tmp_path, kind, fov, dist):
    """provenCount's host twin (countTiming) against the RigAnalyzer checker, the reference's Camera::sees, at the
    boundary points of the GPU's decided-box tests: sensor edges, the FOV cone and the optical axis, with the boxes'
    corners and interior points."""
    import json
    from tests import riganalyzer_util as ru
    ref = ru.load_ref()
    if ref is None:
        pytest.skip("the RigAnalyzer checker (oracle/riganalyzer.mk) is not built")
    lib = capi.load_cuda()
    rng = np.random.default_rng(5)
    desc = iu.camera(kind, fov=fov, distortion=dist)
    second = iu.camera(kind, fov=fov, distortion=dist, forward=(1, 0.25, -0.1))
    path = str(tmp_path / "rig.json")
    json.dump({"cameras": [iu.desc_json(desc, "cam0"), iu.desc_json(second, "cam1")]}, open(path, "w"))
    pts = np.vstack([iu.edge_points(lib, desc, d, rng) for d in (0.7, 3.0)])
    pts = np.vstack([pts] + [iu.box_samples(iu.boxes_around(pts, k), rng).reshape(-1, 3) for k in (1, 1024)])
    counts, _ = capi.RigAnalysis(lib).proven_count(capi.rig_descs(json.load(open(path))), pts, host=True)
    assert np.array_equal(counts, ref.count(path, pts))
