"""CreateObjFromDisparityEquirect on the GPU: derp_equirect_mesh[_simplified] of the CUDA library against the reference's
own MeshUtil.h / MeshSimplifier.cpp (oracle/_ref) with 0 differing vertex bits and faces, and the app end to end after
DerpCLI and SimpleMeshRenderer, byte for byte against the reference's writeObj / writeMtl."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests.test_eqr_obj import APP, CASES, SCALED, eqr, eqr_ref, jumps, make, same, specials  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES + SCALED)
def test_gpu_mesh_equals_reference(eqr, eqr_ref, case):
    name, w, h, scale, max_depth, tear = case
    for seed in range(2):
        d = make(name, w, h, seed)
        gv, gf = eqr.mesh(d, scale=scale, max_depth=max_depth, tear_ratio=tear)
        rv, rf = eqr_ref.mesh(d, scale=scale, max_depth=max_depth, tear_ratio=tear)
        assert same(gf, rf) and same(gv, rv)


@pytest.mark.parametrize("strictness,num_faces,scale", [(0.8, 400, 1.0), (1.0, 300, 1.0), (0.8, 10 ** 6, 1.0),
                                                        (0.8, 500, 0.5), (0.8, 300, 0.37)])
def test_gpu_simplified_equals_reference(eqr, eqr_ref, strictness, num_faces, scale):
    for d in (jumps(64, 32, 1), specials(58, 29, 2)):
        gv, gf = eqr.mesh(d, scale=scale, num_faces=num_faces, strictness=strictness)
        rv, rf = eqr_ref.mesh(d, scale=scale, num_faces=num_faces, strictness=strictness)
        assert same(gf, rf) and same(gv, rv)


def test_gpu_device_resident_input(eqr, eqr_ref):
    """The disparity as device memory of the current GPU is read in place (plain and resized)."""
    import torch
    d = specials(80, 40, 7)
    t = torch.from_numpy(d).cuda()
    for scale in (1.0, 0.37):
        gv, gf = eqr.mesh((t.data_ptr(), 80, 40), scale=scale)
        rv, rf = eqr_ref.mesh(d, scale=scale)
        assert same(gf, rf) and same(gv, rv)


def test_gpu_full_size(eqr, eqr_ref):
    """SimpleMeshRenderer's default equirect size, 3072 x 1536: 4.7 M vertexes, up to 9.4 M faces (fewer with tears)."""
    d = jumps(3072, 1536, 3)
    d[::97, ::89] = np.nan
    gv, gf = eqr.mesh(d)
    rv, rf = eqr_ref.mesh(d)
    assert same(gf, rf) and same(gv, rv)
    assert len(gv) == 3072 * 1536 and len(gf) > 7_000_000


def _ref_obj(ref, v, f, obj, color):
    fn = ref.lib.derp_ref_write_obj
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_char_p, C.c_char_p]
    v = np.ascontiguousarray(v, np.float64)
    f = np.ascontiguousarray(f, np.uint32)
    assert fn(v.ctypes.data, len(v), f.ctypes.data, len(f), obj.encode(), None if color is None else color.encode()) == 0


def test_app_end_to_end(eqr_ref, tmp_path):
    """DerpCLI on a small rig -> SimpleMeshRenderer --format eqrdisp / eqrcolor -> the app, with and without
    --create_mtl: the .obj and .mtl bytes equal the reference's writeObj / writeMtl of the reference's mesh of the same
    decoded PNG."""
    import cv2
    from tests.test_gpu_smr import BIN, _derpcli_disparities
    W, S, width = 64, 8, 96
    rig = synth.ring_rig(S, W, W, kind="FTHETA")
    colors, _ = synth.render_rig(rig, W, W, scene=synth.Scene(seed=5))
    inp, lvl0, _ = _derpcli_disparities(tmp_path, rig, colors, W)
    color_dir = inp + "/video/color_levels/level_0"
    out = {}
    for fmt in ("eqrdisp", "eqrcolor"):
        p = subprocess.run([os.path.join(BIN, "SimpleMeshRenderer"), "--rig=" + inp + "/rigs/rig_calibrated.json",
                            "--color=" + color_dir, "--disparity=" + lvl0, "--output=" + str(tmp_path / fmt),
                            "--first=000000", "--last=000000", "--format=" + fmt, "--width=%d" % width],
                           capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-2000:]
        out[fmt] = str(tmp_path / fmt / "000000.png")
    img = cv2.imread(out["eqrdisp"], cv2.IMREAD_UNCHANGED)
    disp = cv2.cvtColor(img.astype(np.float32) / 65535.0, cv2.COLOR_BGR2GRAY) if img.ndim == 3 else img / 65535.0
    # the same decoded PNG through the app's own reader, so that the comparison is of the mesh and the writer
    subprocess.run([os.path.join(BIN, "IoSelfTest"), "--mode=float", "--in=" + out["eqrdisp"],
                    "--out=" + str(tmp_path / "disp.bin")], check=True, capture_output=True)
    disp = np.fromfile(str(tmp_path / "disp.bin"), np.float32).reshape(disp.shape)
    for strictness in ("0", "0.8"):
        rv, rf = eqr_ref.mesh(disp, num_faces=2000, strictness=float(strictness))
        for mtl in (False, True):
            d = tmp_path / ("s%s_%d" % (strictness, mtl))
            d.mkdir()
            args = [APP, "--input_png_disp=" + out["eqrdisp"], "--input_png_color=" + out["eqrcolor"],
                    "--output_obj=" + str(d / "mesh.obj"), "--num_faces=2000", "--strictness=" + strictness]
            p = subprocess.run(args + (["--create_mtl"] if mtl else []), capture_output=True, text=True)
            assert p.returncode == 0, p.stderr[-2000:]
            want = tmp_path / ("want_s%s_%d" % (strictness, mtl))
            want.mkdir()
            _ref_obj(eqr_ref, rv, rf, str(want / "mesh.obj"), out["eqrcolor"] if mtl else None)
            assert (d / "mesh.obj").read_bytes() == (want / "mesh.obj").read_bytes()
            if mtl:
                assert (d / "mesh.mtl").read_bytes() == (want / "mesh.mtl").read_bytes()
                assert b"vt " in (d / "mesh.obj").read_bytes()
