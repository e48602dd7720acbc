"""RigAnalyzer on the GPU (include/derp_riganalysis.h and the RigAnalyzer app) against the checker, the reference's own
RigAnalyzer.cpp compiled by oracle/riganalyzer.mk: 0 differing values in the coverage histograms, the equirect counts
and timing, every camera's overlap map and the cross-section; the share of points resolved on the host; and the app's
stdout, .ppm, .obj and rig JSON against the checker's main."""
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import riganalyzer_util as ru

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return capi.RigAnalysis(capi.load_cuda())


@pytest.fixture(scope="module")
def ref():
    r = ru.load_ref()
    if r is None:
        pytest.skip("the RigAnalyzer checker (oracle/riganalyzer.mk) is not built")
    return r


def _share(lib, points, label):
    host = lib.last_host_points()
    print("%s: %d of %d points resolved on the host (%.4f %%)" % (label, host, points, 100.0 * host / points))
    return host


def _ref_cameras(ref, path, ids, distance, tmp_path):
    """saveCamera of each camera id, in parallel (the checker's calls release the GIL and share the flags)."""
    ref.set_flags(["--overlap_distance=%r" % distance])

    def one(cid):
        out = str(tmp_path / ("ref_%s.ppm" % cid))
        assert ref.lib.ref_ra_save(2, path.encode(), out.encode(), cid.encode()) == 0
        return ru.read_ppm(out)[1]

    with ThreadPoolExecutor(max(1, min(len(ids), os.cpu_count() or 1))) as ex:
        return list(ex.map(one, ids))


def test_coverage_at_app_defaults(lib, ref):
    """main's histograms: 100 000 samples, 20 distances from 0.5, the golden rig."""
    s = ref.samples(100000)
    d = ru.descs_of(ru.GOLDEN_RIG)
    dists = [0.5 / (1 - i / 20.0) for i in range(20)]
    got = lib.coverage(d, s, dists)
    _share(lib, len(s) * len(dists), "coverage")
    for k, dist in enumerate(dists):
        want = np.bincount(ref.count(ru.GOLDEN_RIG, s * dist), minlength=len(d) + 1)
        assert np.array_equal(got[k], want), dist


@pytest.mark.parametrize("distance", [1e4, 0.5, 0.05])
def test_equirect_golden_rig(lib, ref, tmp_path, distance):
    d = ru.descs_of(ru.GOLDEN_RIG)
    counts, timing = lib.equirect(d, 1800, 900, distance)
    host = _share(lib, 1800 * 900, "equirect at %g" % distance)
    assert host < 0.01 * 1800 * 900
    hc, ht = lib.equirect(d, 1800, 900, distance, host=True)
    assert np.array_equal(counts, hc) and np.array_equal(timing.view(np.uint32), ht.view(np.uint32))
    ref.save("equirect", ru.GOLDEN_RIG, str(tmp_path / "e.ppm"), args=["--overlap_distance=%r" % distance])
    assert np.array_equal(counts, ru.read_ppm(tmp_path / "e.ppm")[1])
    ref.save("equirect", ru.GOLDEN_RIG, str(tmp_path / "t.ppm"), args=["--overlap_distance=%r" % distance,
                                                                          "--show_timing"])
    assert np.array_equal(((1.0 - timing.astype(np.float64)) * 255.0).astype(np.int64),
                          ru.read_ppm(tmp_path / "t.ppm")[1])


@pytest.mark.parametrize("distance", [1e4, 0.5, 0.05])
def test_every_camera_of_the_golden_rig(lib, ref, tmp_path, distance):
    """saveCamera for all 16 cameras at 3360 x 2160."""
    rig = json.load(open(ru.GOLDEN_RIG))
    ids = [c["id"] for c in rig["cameras"]]
    d = ru.descs_of(ru.GOLDEN_RIG)
    got, host = [], 0
    for i in range(len(ids)):
        got.append(lib.camera(d, i, distance))
        host += lib.last_host_points()
    print("camera mode at %g: %d of %d pixels on the host" % (distance, host, 16 * 3360 * 2160))
    assert host < 0.01 * 16 * 3360 * 2160
    for cid, g, w in zip(ids, got, _ref_cameras(ref, ru.GOLDEN_RIG, ids, distance, tmp_path)):
        assert np.array_equal(g, w), cid


@pytest.mark.parametrize("kind", ru.TYPES)
@pytest.mark.parametrize("limited", [False, True])
def test_models(lib, ref, tmp_path, kind, limited):
    fov = (1.2 if kind in ("RECTILINEAR", "ORTHOGRAPHIC") else 1.9) if limited else None
    dist = [0.01, -0.002] if limited else None
    path = ru.write_rig(tmp_path / "rig.json", ru.ring_rig(kind, n=5, fov=fov, distortion=dist, res=(640, 480)))
    d = ru.descs_of(path)
    s = ref.samples(20000)
    dists = [0.05, 0.5, 1e4]
    got = lib.coverage(d, s, dists)
    for k, dd in enumerate(dists):
        assert np.array_equal(got[k], np.bincount(ref.count(path, s * dd), minlength=len(d) + 1)), dd
    ref.save("cross_section", path, str(tmp_path / "x.ppm"))
    assert np.array_equal(lib.cross_section(d), ru.read_ppm(tmp_path / "x.ppm")[1])
    counts, _ = lib.equirect(d, 1800, 900, 1e4)
    ref.save("equirect", path, str(tmp_path / "e.ppm"))
    assert np.array_equal(counts, ru.read_ppm(tmp_path / "e.ppm")[1])
    for distance in (1e4, 0.5, 0.05):
        ids = ["cam%d" % i for i in range(5)]
        want = _ref_cameras(ref, path, ids, distance, tmp_path)
        for i in range(5):
            assert np.array_equal(lib.camera(d, i, distance), want[i]), (i, distance)


def test_cross_section_golden_rig(lib, ref, tmp_path):
    ref.save("cross_section", ru.GOLDEN_RIG, str(tmp_path / "x.ppm"))
    assert np.array_equal(lib.cross_section(ru.descs_of(ru.GOLDEN_RIG)), ru.read_ppm(tmp_path / "x.ppm")[1])


def test_rig_of_more_than_64_cameras(lib, ref, tmp_path):
    path = ru.write_rig(tmp_path / "rig.json", ru.ring_rig("FTHETA", n=72, fov=1.7, res=(160, 120)))
    d = ru.descs_of(path)
    s = ref.samples(20000)
    got = lib.coverage(d, s, [0.3, 1e4])
    for k, dd in enumerate([0.3, 1e4]):
        assert np.array_equal(got[k], np.bincount(ref.count(path, s * dd), minlength=len(d) + 1))
    counts, timing = lib.equirect(d, 1800, 900, 1e4)
    hc, ht = lib.equirect(d, 1800, 900, 1e4, host=True)
    assert np.array_equal(counts, hc) and np.array_equal(timing.view(np.uint32), ht.view(np.uint32))
    assert counts.max() > 32  # more cameras than the device's sorted timing list: those points go to the host
    ref.save("cross_section", path, str(tmp_path / "x.ppm"))
    assert np.array_equal(lib.cross_section(d), ru.read_ppm(tmp_path / "x.ppm")[1])
    assert np.array_equal(lib.camera(d, 3, 1e4), _ref_cameras(ref, path, ["cam3"], 1e4, tmp_path)[0])


def test_device_resident_outputs(lib):
    import torch
    d = ru.descs_of(ru.GOLDEN_RIG)
    c = torch.empty((900, 1800), dtype=torch.int32, device="cuda")
    t = torch.empty((900, 1800), dtype=torch.float32, device="cuda")
    lib.equirect(d, 1800, 900, 1e4, out=(c.data_ptr(), t.data_ptr()))
    cam = torch.empty((2160, 3360), dtype=torch.int32, device="cuda")
    lib.camera(d, 2, 1e4, out=cam.data_ptr())
    x = torch.empty((400, 400), dtype=torch.int32, device="cuda")
    lib.cross_section(d, out=x.data_ptr())
    torch.cuda.synchronize()
    hc, ht = lib.equirect(d, 1800, 900, 1e4)
    assert np.array_equal(c.cpu().numpy(), hc) and np.array_equal(t.cpu().numpy().view(np.uint32), ht.view(np.uint32))
    assert np.array_equal(cam.cpu().numpy(), lib.camera(d, 2, 1e4))
    assert np.array_equal(x.cpu().numpy(), lib.cross_section(d))


# ---- the app against the checker's main ------------------------------------------------------------------------------
def _both(ref, tmp_path, args, outputs=()):
    """Runs the app and the checker's main with args plus each output flag pointed into their own directories;
    returns (app stdout, ref stdout, app dir, ref dir, app stderr)."""
    dirs = []
    for who in ("app", "ref"):
        p = tmp_path / who
        p.mkdir(exist_ok=True)
        dirs.append(p)
    full = [list(args) + ["--%s=%s" % (o, p / ("out_" + o)) for o in outputs] for p in dirs]
    r = ru.run_app(full[0])
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout, ref.main(full[1]), dirs[0], dirs[1], r.stderr


E2E_CASES = [
    ["--output_camera_id=cam3", "--scale_resolution=0.5"],
    ["--show_timing", "--output_camera_id=cam0", "--scale_resolution=0.25"],
    ["--rearrange=ballcam24", "--output_camera_id=cam7", "--scale_resolution=0.25"],
    ["--perturb_cameras", "--perturb_positions=0.01", "--perturb_rotations=0.05", "--perturb_principals=3",
     "--perturb_seed=7", "--output_camera_id=cam5", "--scale_resolution=0.25"],
]


@pytest.mark.parametrize("case", range(len(E2E_CASES)))
def test_app_matches_reference(lib, ref, tmp_path, case):
    outs = ["output_obj", "output_equirect", "output_camera", "output_cross_section"]
    a, b, da, db, _ = _both(ref, tmp_path, ["--rig=" + ru.GOLDEN_RIG] + E2E_CASES[case], outs)
    assert a == b
    assert a.count("\n") == 20
    for o in outs:
        assert os.path.exists(db / ("out_" + o)), o
        assert open(da / ("out_" + o), "rb").read() == open(db / ("out_" + o), "rb").read(), o


def test_app_log_lines(lib, tmp_path):
    """saveEquirect's log lines: holes, and the max and the raster-order mean of minTimingDiff in ms."""
    r = ru.run_app(["--rig=" + ru.GOLDEN_RIG, "--sample_count=100", "--output_equirect=" + str(tmp_path / "e.ppm")])
    assert r.returncode == 0, r.stderr[-2000:]
    counts, timing = lib.equirect(ru.descs_of(ru.GOLDEN_RIG), 1800, 900, 1e4)
    t = timing.astype(np.float64).ravel()
    ave = 0.0
    for v in t:
        ave += v
    frame = float(np.float32(1000.0) / np.float32(60.0))
    for line in ("Holes found (in pixels) = %g" % float((counts == 0).sum()),
                 "Max of min timing distance = %gms" % (frame * t.max()),
                 "Ave of min timing distance = %gms" % (frame * ave / (1800 * 900))):
        assert line in r.stderr, line


def _rig_state(path):
    rig = json.load(open(path))
    keys = ["origin", "forward", "up", "right", "resolution", "focal", "principal", "distortion", "fov", "id", "group",
            "type"]
    return [{k: c.get(k) for k in keys} for c in rig["cameras"]]


def _revolve_file(tmp_path, n):
    p = tmp_path / "revolve.txt"
    p.write_text("=== header\n" + "".join("0 0 %r\n" % (2 * np.pi * i / n) for i in range(n)))
    return str(p)


def _edit_cases(tmp_path):
    eul = tmp_path / "eulers.txt"
    eul.write_text("=== five cameras\n0 0 0\n90 0 0\n0 90 0\n-30 45 60\n180 0 90\n")
    cases = []
    for name in ["ballcam24", "tetra", "tetratilted", "ring4", "cube", "carbon0", "carbon1", "diamond"]:
        cases += [["--rearrange=" + name], ["--rearrange=" + name, "--custom=60", "--one_based_indexing"]]
    cases += [["--eulers=" + str(eul)], ["--revolve=" + _revolve_file(tmp_path, 5)]]
    cases += [["--perturb_cameras", "--perturb_positions=0.02", "--perturb_rotations=0.1", "--perturb_principals=5",
               "--perturb_seed=%d" % s] for s in (1, 2, 99)]
    cases += [["--rotate_cam_z=cam3"], ["--z_is_up"], ["--z_is_down"], ["--rotate=0.1 -0.2 0.3"],
              ["--scale_rig=0.01"], ["--radius=0.3"], ["--scale_resolution=0.37"],
              ["--rearrange=cube", "--z_is_up", "--scale_rig=2", "--radius=0.5", "--scale_resolution=0.5"]]
    return cases


def test_rig_edits_match_reference(lib, ref, tmp_path):
    """Every rig edit against the checker's rig state (its --output_rig: 17 significant digits round-trip every
    double, as the app's shortest doubles do), bit for bit."""
    for args in _edit_cases(tmp_path):
        a, b, da, db, _ = _both(ref, tmp_path, ["--rig=" + ru.GOLDEN_RIG, "--sample_count=100"] + args, ["output_rig"])
        assert a == b, args
        got, want = _rig_state(da / "out_output_rig"), _rig_state(db / "out_output_rig")
        assert got == want, args
        comments = json.load(open(da / "out_output_rig"))["comments"]
        assert comments[0] == "command line:" and (" " + args[-1] + " ") in comments[1]


def test_perturb_focals_and_revolve_past_64_cameras(lib, ref, tmp_path):
    rig = ru.write_rig(tmp_path / "ring.json", ru.ring_rig("FTHETA", n=16, fov=1.7, res=(320, 240)))
    for args in (["--perturb_cameras", "--perturb_focals=4", "--perturb_principals=2", "--perturb_seed=3"],
                 ["--revolve=" + _revolve_file(tmp_path, 5), "--show_timing"]):
        a, b, da, db, _ = _both(ref, tmp_path, ["--rig=" + rig] + args,
                                ["output_rig", "output_obj", "output_equirect", "output_cross_section"])
        assert a == b, args
        assert _rig_state(da / "out_output_rig") == _rig_state(db / "out_output_rig")
        for o in ("output_obj", "output_equirect", "output_cross_section"):
            assert open(da / ("out_" + o), "rb").read() == open(db / ("out_" + o), "rb").read(), (args, o)
