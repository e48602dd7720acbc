"""RigAnalyzer's host half (include/derp_riganalysis.h's per-point code, run on the host) against the checker, the
reference's own RigAnalyzer.cpp compiled by oracle/riganalyzer.mk, without a GPU: coverage counts on the golden rig and
on rigs of every camera model, a point on a camera's optical axis, points on the sensor's edges, the equirect / camera
/ cross-section maps; the rig JSON writer's SHORTEST doubles, the app's flag surface, its refusals and FATAL without a
GPU.  The app's rig edits, OBJ, PPM files and stdout need the GPU and are in test_gpu_rig_analyzer.py."""
import json
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import riganalyzer_util as ru

HOST = os.path.join(ru.ROOT, "facebook360_dep_b200", "csrc", "host")


@pytest.fixture(scope="module")
def lib():
    return capi.RigAnalysis(os.path.join(ru.ROOT, "facebook360_dep_b200", "libderp_b200.so"))


@pytest.fixture(scope="module")
def ref():
    r = ru.load_ref()
    if r is None:
        pytest.skip("the RigAnalyzer checker (oracle/riganalyzer.mk) is not built")
    return r


@pytest.fixture(scope="module")
def app():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return ru.APP


def test_abi_is_exported(lib):
    header = open(os.path.join(ru.ROOT, "include", "derp_riganalysis.h")).read()
    for name in capi.RIGANALYSIS_SYMBOLS:
        assert hasattr(lib.lib, name), name
        assert name + "(" in header, name


def _per_point(lib, descs, points):
    """The host's count at each point (one coverage histogram per point)."""
    out = []
    for p in points:
        h = lib.coverage(descs, [p], [1.0], host=True)
        out.append(int(np.argmax(h[0])))
    return np.array(out)


def test_samples_match_reference(ref):
    """The app's Fibonacci samples are getFibonacciUnits + discardPoles; the checker's own are the library's input here."""
    s = ref.samples(1000, 10.0)
    assert len(s) < 1000 and np.all(np.abs(s[:, 2]) < np.cos(np.radians(10.0)))


@pytest.mark.parametrize("distances", [[0.5, 0.7, 2.0], [10.0, 1e4]])
def test_coverage_golden_rig(lib, ref, distances):
    s = ref.samples(5000)
    d = ru.descs_of(ru.GOLDEN_RIG)
    got = lib.coverage(d, s, distances, host=True)
    for k, dist in enumerate(distances):
        want = np.bincount(ref.count(ru.GOLDEN_RIG, s * dist), minlength=len(d) + 1)
        assert np.array_equal(got[k], want), dist


MODEL_CASES = [(kind, fov, dist) for kind in ru.TYPES for fov, dist in
               [(None, None), (1.2 if kind in ("RECTILINEAR", "ORTHOGRAPHIC") else 1.9, [0.01, -0.002])]]


@pytest.mark.parametrize("kind,fov,distortion", MODEL_CASES)
def test_models_against_reference(lib, ref, tmp_path, kind, fov, distortion):
    """Coverage, cross-section, equirect and camera maps of a 4-camera ring of each model, default and limited fov."""
    path = ru.write_rig(tmp_path / "rig.json", ru.ring_rig(kind, fov=fov, distortion=distortion, res=(120, 90)))
    d = ru.descs_of(path)
    s = ref.samples(3000)
    for dist in (0.05, 0.3, 1e4):
        want = np.bincount(ref.count(path, s * dist), minlength=len(d) + 1)
        assert np.array_equal(lib.coverage(d, s, [dist], host=True)[0], want), dist
    ref.save("cross_section", path, str(tmp_path / "x.ppm"))
    assert np.array_equal(lib.cross_section(d, host=True), ru.read_ppm(tmp_path / "x.ppm")[1])
    for dist in ("0.5", "1e4"):
        ref.save("camera", path, str(tmp_path / "c.ppm"), "cam1", ["--overlap_distance=" + dist])
        assert np.array_equal(lib.camera(d, 1, float(dist), host=True), ru.read_ppm(tmp_path / "c.ppm")[1]), dist


def test_equirect_golden_rig(lib, ref, tmp_path):
    """saveEquirect's counts and timing view (with --show_timing) at the default distance."""
    d = ru.descs_of(ru.GOLDEN_RIG)
    counts, timing = lib.equirect(d, 1800, 900, 1e4, host=True)
    ref.save("equirect", ru.GOLDEN_RIG, str(tmp_path / "e.ppm"))
    assert np.array_equal(counts, ru.read_ppm(tmp_path / "e.ppm")[1])
    ref.save("equirect", ru.GOLDEN_RIG, str(tmp_path / "t.ppm"), args=["--show_timing"])
    assert np.array_equal(((1.0 - timing.astype(np.float64)) * 255.0).astype(np.int64), ru.read_ppm(tmp_path / "t.ppm")[1])


def test_optical_axis_point_is_seen(lib, ref, tmp_path):
    """A point on a camera's exact optical axis projects to a NaN pixel, which isOutsideSensor does not reject."""
    for kind in ru.TYPES:
        rig = {"cameras": [ru.camera_json(kind, pos=(0, 0, 0), fwd=(1, 0, 0), up=(0, 0, 1))]}
        path = ru.write_rig(tmp_path / ("axis_%s.json" % kind), rig)
        pts = np.array([[5.0, 0, 0], [1e4, 0, 0], [0.5, 0, 0]])
        want = ref.count(path, pts)
        assert np.array_equal(_per_point(lib, ru.descs_of(path), pts), want), kind
        assert want.tolist() == [1, 1, 1], kind


def test_sensor_edge_points(lib, ref, tmp_path):
    """Points whose pixel lands exactly on a sensor edge (x = 0 is inside, x = width is outside), and a dense band of
    directions across the edges of every model."""
    rig = {"cameras": [ru.camera_json("RECTILINEAR", res=(200, 150), pos=(0, 0, 0), fwd=(0, 0, -1), up=(0, 1, 0),
                                      focal=100.0)]}
    path = ru.write_rig(tmp_path / "edge.json", rig)
    # principal (100, 75), focal (100, -100): x = 100 cx / -cz + 100, y = -100 cy / -cz + 75
    pts = np.array([[-1.0, 0, -1], [1.0, 0, -1], [0, 0.75, -1], [0, -0.75, -1], [-1.0, 0.75, -1], [0.999, -0.7499, -1]])
    want = ref.count(path, pts)
    assert np.array_equal(_per_point(lib, ru.descs_of(path), pts), want)
    assert want[0] == 1 and want[1] == 0
    rng = np.random.default_rng(5)
    for kind in ru.TYPES:
        path = ru.write_rig(tmp_path / ("band_%s.json" % kind), ru.ring_rig(kind, n=2, res=(120, 90)))
        d = ru.descs_of(path)
        a = rng.uniform(-np.pi, np.pi, 4000)
        e = rng.uniform(-1.2, 1.2, 4000)
        s = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], 1)
        want = np.bincount(ref.count(path, s * 2.0), minlength=len(d) + 1)
        assert np.array_equal(lib.coverage(d, s, [2.0], host=True)[0], want), kind


SHORTEST_TABLE = [(0.1, "0.1"), (1.0, "1"), (-0.0, "-0"), (1e-7, "1E-7"), (1e21, "1E21"), (123456.789, "123456.789"),
                  (1e-6, "0.000001"), (1.5e-7, "1.5E-7"), (1e20, "100000000000000000000"), (-2.5, "-2.5"),
                  (0.30000000000000004, "0.30000000000000004"), (3360.0, "3360")]


def test_shortest_doubles(tmp_path):
    """--output_rig's doubles: folly's SHORTEST layout (decimal for exponents in [-6, 21), E otherwise, no '.0')."""
    src = tmp_path / "t.cpp"
    src.write_text('#include "%s"\n#include <cstdio>\nint main(int c, char** v) {\n'
                   '  for (int i = 1; i < c; ++i) std::printf("%%s\\n", rigjson::shortest(std::strtod(v[i], 0)).c_str());\n'
                   '}\n' % os.path.join(HOST, "rig_json.h"))
    exe = tmp_path / "t"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)] + [repr(v) for v, _ in SHORTEST_TABLE], capture_output=True, text=True).stdout
    assert out.split("\n")[:-1] == [s for _, s in SHORTEST_TABLE]
    for v, s in SHORTEST_TABLE:
        assert float(s.replace("E", "e")) == v


def _app_defines():
    import re
    src = open(os.path.join(HOST, "RigAnalyzer.cpp")).read()
    return {m.group(2): [m.group(1), m.group(3).strip().strip('"'), re.sub(r'"\s*"', "", m.group(4)).strip().strip('"')]
            for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*((?:"[^"]*"\s*)*)\)', src)}


def test_flag_surface_matches_reference(app):
    """The reference's DEFINE_ lines (RigAnalyzer.cpp:30-65, tests/golden/riganalyzer_flags.json) plus --gpu."""
    found = _app_defines()
    assert found.pop("gpu") == ["int32", "0", "CUDA device to use"]
    assert found == ru.FLAGS
    h = subprocess.run([app, "--help"], capture_output=True, text=True)
    for flag in ru.FLAGS:
        assert "-" + flag + " " in h.stdout, flag


def test_refusals(app, tmp_path):
    rig = ru.write_rig(tmp_path / "rig.json", ru.ring_rig("FTHETA"))
    cases = [
        ([], "Check failed"),  # --rig is required
        (["--rig=" + rig, "--sample_count=0"], "sample_count"),
        (["--rig=" + rig, "--discard_poles=90"], "leaves no samples"),
        (["--rig=" + rig, "--rearrange=unknown"], "unknown arrangement"),
        (["--rig=" + rig, "--rotate=1 2"], "bad --rotate vector"),
        (["--rig=" + rig, "--rotate_cam_z=missing"], "not found"),
    ]
    for args, msg in cases:
        r = ru.run_app(args, cwd=str(tmp_path))
        assert r.returncode != 0, args
        assert msg in r.stderr, (args, r.stderr[-400:])


def test_fatal_without_gpu(app, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    rig = ru.write_rig(tmp_path / "rig.json", ru.ring_rig("FTHETA"))
    r = ru.run_app(["--rig=" + rig, "--sample_count=10", "--output_obj=" + str(tmp_path / "r.obj")])
    assert r.returncode != 0 and "derp_rig_coverage" in r.stderr
    assert r.stdout == "" and not os.path.exists(tmp_path / "r.obj")
