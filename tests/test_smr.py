"""SimpleMeshRenderer without a GPU: the app's command line, its host-side image steps pinned to cv2 4.13
(tests/golden/smr_vectors.npz, generator tests/golden/gen_smr_vectors.py) and to numpy restatements, and properties of
the checker's canopy render (tests/canopy_oracle.cpp) in the exporter's modes."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import canopy_oracle

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "smr_vectors.npz"))
HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")
APP = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin", "SimpleMeshRenderer")

# SimpleMeshRenderer.cpp's DEFINE lines (the format's help is built from the format list there)
REF_FLAGS = {"cameras": ("string", ""), "color": ("string", ""), "disparity": ("string", ""),
             "background": ("string", ""), "background_equirect": ("string", ""), "file_type": ("string", "png"),
             "first": ("string", "000000"), "forward": ("string", "-1.0 0.0 0.0"), "height": ("int32", "-1"),
             "horizontal_fov": ("double", "90"), "ignore_alpha_blend": ("bool", "false"), "last": ("string", "000000"),
             "output": ("string", ""), "position": ("string", "0.0 0.0 0.0"), "rig": ("string", ""),
             "up": ("string", "0.0 0.0 1.0"), "width": ("int32", "3072"), "format": ("string", "")}


@pytest.fixture(scope="module")
def oracle():
    return canopy_oracle.load()


def _fn(oracle, name, res, args):
    f = getattr(oracle.lib, name)
    f.restype = res
    f.argtypes = args
    return f


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


# ---- command line ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def app():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return APP


def test_flag_surface_matches_reference(app):
    src = open(os.path.join(HOST, "SimpleMeshRenderer.cpp")).read()
    found = {m.group(2): (m.group(1), m.group(3).strip('"'))
             for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*"', src)}
    assert {k: v for k, v in found.items() if k != "gpu"} == REF_FLAGS
    assert found["gpu"] == ("int32", "0")
    h = subprocess.run([app, "--help"], capture_output=True, text=True)
    for name in REF_FLAGS:
        assert "-" + name + " " in h.stdout


def _inputs(tmp_path):
    rig = synth.ring_rig(2, 8, 8)
    json.dump(rig, open(tmp_path / "rig.json", "w"))
    for cam in rig["cameras"]:
        for sub in ("disp", "color"):
            os.makedirs(tmp_path / sub / cam["id"], exist_ok=True)
        with open(tmp_path / "disp" / cam["id"] / "000000.pfm", "wb") as f:
            f.write(b"Pf\n8 8\n-1.0\n" + np.full(64, 0.5, np.float32).tobytes())
        open(tmp_path / "color" / cam["id"] / "000000.png", "wb").close()
    return ["--rig=" + str(tmp_path / "rig.json"), "--disparity=" + str(tmp_path / "disp"),
            "--output=" + str(tmp_path / "out")]


@pytest.mark.parametrize("bad,message", [
    (["--format=eqr"], "Invalid format: eqr"),
    (["--format=eqrdisp", "--width=7"], "width must be a multiple of 2"),
    (["--format=eqrdisp", "--width=0"], "FLAGS_width > 0"),
    (["--format=eqrcolor"], "eqrcolor needs --color to be set"),
    ([], "on-screen rendering (an empty --format) is not available"),
    (["--format=eqrdisp", "--file_type=jpg"], "unsupported --file_type jpg: this build writes png and exr"),
    (["--format=eqrdisp", "--disparity="], "FLAGS_disparity != \"\""),
])
def test_app_aborts_on_bad_flags(app, tmp_path, bad, message):
    p = subprocess.run([app] + _inputs(tmp_path) + bad, capture_output=True, text=True)
    assert p.returncode != 0 and message in p.stderr, p.stderr[-500:]


# ---- host steps ------------------------------------------------------------------------------------------------------
def test_png_conversion_matches_cv2(oracle):
    """convertImage<cv::Vec3w>: x 65535, cvRound (ties to even), saturation, NaN -> 0, alpha dropped."""
    img = _f32(G["img"])
    out = np.empty(img.shape[:2] + (3,), np.uint16)
    _fn(oracle, "oracle_smr_png16", None, [C.c_void_p, C.c_int, C.c_void_p])(img.ctypes.data, img.shape[0] * img.shape[1],
                                                                           out.ctypes.data)
    assert len(G["ties"]) > 20 and np.isnan(img).any() and (img < 0).any() and (img > 1).any()
    assert np.array_equal(out, G["png"])


def test_exr_three_channels_read_back_by_cv2(tmp_path):
    """io::writeExrFloatChannels(..., 3): cv2 4.13 reads the B, G, R floats back bit for bit, NaN and inf included."""
    src = tmp_path / "w.cpp"
    src.write_text('#include "io.h"\nint main(int, char** argv) { std::vector<float> v(5 * 3 * 3);\n'
                   '  for (size_t i = 0; i < v.size(); ++i) v[i] = (float)i / 7 - 2;\n'
                   '  v[4] = NAN; v[10] = INFINITY; v[20] = -0.0f;\n'
                   '  io::writeExrFloatChannels(argv[1], v.data(), 5, 3, 3); return 0; }\n')
    exe = tmp_path / "w"
    subprocess.check_call(["g++", "-std=c++17", "-I", HOST, str(src), "-o", str(exe), "-lz"])
    path = str(tmp_path / "x.exr")
    subprocess.check_call([str(exe), path])
    code = ("import cv2, numpy as np, sys; a = cv2.imread(sys.argv[1], cv2.IMREAD_UNCHANGED); "
            "np.save(sys.argv[2], a)")
    env = dict(os.environ, OPENCV_IO_ENABLE_OPENEXR="1")
    subprocess.check_call([sys.executable, "-c", code, path, str(tmp_path / "a.npy")], env=env)
    got = np.load(tmp_path / "a.npy")
    want = (np.arange(45, dtype=np.float32) / np.float32(7) - np.float32(2)).reshape(3, 5, 3)
    want.reshape(-1)[4], want.reshape(-1)[10], want.reshape(-1)[20] = np.nan, np.inf, -0.0
    assert got.dtype == np.float32 and got.shape == (3, 5, 3)
    assert np.array_equal(got.view(np.uint32) & 0x7fffffff != 0x7fc00000, want.view(np.uint32) & 0x7fffffff != 0x7fc00000)
    assert np.array_equal(got, want, equal_nan=True) and np.signbit(got.reshape(-1)[20])


def _alpha_blend_np(fore, back):
    a = fore[..., 3:4]
    out = a * fore + (np.float32(1) - a) * back
    out[..., 3] = fore[..., 3] + (np.float32(1) - fore[..., 3]) * back[..., 3]
    nan = np.isnan(fore[..., 3])
    out[nan] = back[nan]
    return out


def test_alpha_blend_matches_numpy(oracle):
    rng = np.random.default_rng(3)
    fore = rng.random((10, 12, 4), dtype=np.float32)
    fore[..., 3][rng.random((10, 12)) < 0.3] = np.nan
    back = rng.random((10, 12, 4), dtype=np.float32)
    got = fore.copy()
    _fn(oracle, "oracle_smr_alpha_blend", None, [C.c_void_p, C.c_void_p, C.c_int])(got.ctypes.data, back.ctypes.data, 120)
    assert np.array_equal(got, _alpha_blend_np(fore, back))


def _bg_equirect(oracle, fore, equi, position, forward, up, fov):
    f = _fn(oracle, "oracle_smr_background_equirect", C.c_int,
            [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_double])
    out = _f32(fore).copy()
    equi = _f32(equi)
    vec = [_f32(v) for v in (position, forward, up)]
    assert f(out.ctypes.data, out.shape[1], out.shape[0], equi.ctypes.data, equi.shape[1], equi.shape[0],
             *[v.ctypes.data for v in vec], fov) == 0
    return out


def _bg_equirect_np(fore, equi, position, forward, up, fov):
    """backgroundEquirect restated in numpy (fp64 geometry), with the clamps of smr_host.h."""
    h, w = fore.shape[:2]
    eh, ew = equi.shape[:2]
    f, u = np.asarray(forward, np.float64), np.asarray(up, np.float64)
    right = np.cross(u, -f)
    u = np.cross(right, f)
    f, u = f / np.linalg.norm(f), u / np.linalg.norm(u)
    R = np.stack([np.cross(u, -f), u, -f])
    xmax = 0.1 * np.tan(np.radians(fov) / 2)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    pix = np.stack([((x + 0.5) / w * 2 - 1) * xmax, -((y + 0.5) / h * 2 - 1) * xmax * h / w, np.full_like(x, -0.1)], -1)
    world = (pix * 1e4) @ R + np.asarray(position, np.float64)
    lon = np.arctan2(-world[..., 1], -world[..., 0])
    lat = np.arcsin(np.clip(world[..., 2] / np.linalg.norm(world, axis=-1), -1, 1))
    ix = np.clip(((-lon / np.pi + 1) / 2 * ew).astype(int), 0, ew - 1)
    iy = np.clip(((-lat / np.pi + 0.5) * eh).astype(int), 0, eh - 1)
    back = equi[iy, ix]
    out = _alpha_blend_np(fore, back)
    keep = fore[..., 3] == 1
    out[keep] = fore[keep]
    return out


def test_background_equirect_matches_numpy_and_orientation(oracle):
    """NaN alpha takes the background, other alphas blend over it.  The equirect's centre column is -X, +Y lies to its
    right and its top row is +Z (the reference's comment says "-y to the right"; its formula gives +Y)."""
    eh, ew = 64, 128
    yy, xx = np.mgrid[0:eh, 0:ew]
    equi = np.stack([xx / ew, yy / eh, np.full(xx.shape, 0.5), np.ones(xx.shape)], -1).astype(np.float32)
    rng = np.random.default_rng(4)
    fore = rng.random((24, 32, 4), dtype=np.float32)
    fore[..., 3][rng.random((24, 32)) < 0.4] = np.nan
    fore[..., 3][rng.random((24, 32)) < 0.2] = 1
    args = ([0.1, 0.2, -0.05], [-1, 0.3, 0.2], [0, 0, 1], 100.0)
    got = _bg_equirect(oracle, fore, equi, *args)
    want = _bg_equirect_np(fore, equi, *args)
    close = np.abs(got - want) <= 1e-5
    assert close.mean() > 0.99, close.mean()  # nearest lookups may land a texel apart at a boundary (fp32 vs fp64)
    nanfg = np.full((2, 2, 4), np.nan, np.float32)
    for fwd, up, col, row in (([-1, 0, 0], [0, 0, 1], ew // 2, eh // 2), ([0, 1, 0], [0, 0, 1], 3 * ew // 4, eh // 2),
                              ([0, 0, 1], [1, 0, 0], None, 0)):
        px = _bg_equirect(oracle, nanfg, equi, [0, 0, 0], fwd, up, 90.0)
        c = px[..., 0] * ew
        r = px[..., 1] * eh
        # the four pixel centres lie symmetrically about the view direction
        if col is not None:
            assert abs(c.mean() - col) <= 1 and abs(r.mean() - row) <= 1, (fwd, c, r)
        else:
            assert r.max() <= eh // 4, (fwd, r)  # looking up: the upper rows of the equirect


def test_lr180_layout(oracle):
    w, h = 16, 8
    left = np.random.default_rng(1).random((h, w, 4), dtype=np.float32)
    right = left + 1
    out = np.empty((h, w, 4), np.float32)
    _fn(oracle, "oracle_smr_lr180", None, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p])(
        left.ctypes.data, right.ctypes.data, w, h, out.ctypes.data)
    assert np.array_equal(out, np.concatenate([left[:, w // 4:w // 4 + w // 2], right[:, w // 4:w // 4 + w // 2]], 1))


# ---- the checker's canopy render in the exporter's modes ------------------------------------------------------------
def _axis_rig(W):
    """Six cameras at the origin, one along each of +X, -X, +Y, -Y, +Z, -Z (FTHETA, 180 degrees)."""
    axes = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    cams = []
    for i, f in enumerate(axes):
        f = np.asarray(f, float)
        up = np.array([0, 0, 1.0]) if abs(f[2]) < 1 else np.array([1.0, 0, 0])
        right = np.cross(f, up)
        cams.append({"version": 1, "type": "FTHETA", "origin": [0.0, 0.0, 0.0], "forward": f.tolist(), "up": up.tolist(),
                     "right": right.tolist(), "resolution": [W, W], "focal": [W / np.pi, -W / np.pi], "fov": 1.5707963,
                     "id": "cam%d" % i})
    return {"cameras": cams}


def _const_colors(n, W):
    cols = []
    for i in range(n):
        c = np.zeros((W, W, 4), np.float32)
        c[..., 0] = (i + 1) / 8.0
        c[..., 3] = 1
        cols.append(c)
    return cols


def test_equirect_orientation(oracle):
    W = 32
    rig = _axis_rig(W)
    disps = [np.full((W, W), 0.5, np.float32)] * 6
    col, _, _ = oracle.render(capi.rig_descs(rig), disps, _const_colors(6, W), np.zeros(3, np.float32), "equirect",
                              (64, 32), alpha_blend=False)
    cam = np.rint(col[..., 0] * 8 - 1)
    assert cam[16, 32] == 1  # centre column, equator: -X
    assert cam[16, 48] == 2  # to its right: +Y
    assert cam[16, 16] == 3  # to its left: -Y
    assert (cam[0] == 4).all()  # top row: +Z
    assert (cam[-1] == 5).all()


def _face_matrix_np(face, p):
    table = [((1, 0, 0), (0, 0, -1), (0, -1, 0)), ((-1, 0, 0), (0, 0, 1), (0, -1, 0)), ((0, 1, 0), (1, 0, 0), (0, 0, 1)),
             ((0, -1, 0), (1, 0, 0), (0, 0, -1)), ((0, 0, 1), (1, 0, 0), (0, -1, 0)), ((0, 0, -1), (-1, 0, 0), (0, -1, 0))]
    ma, sc, tc = (np.asarray(v, np.float32) for v in table[face])
    T = np.eye(4, dtype=np.float32)
    T[0, :3], T[1, :3], T[2, :3] = sc, tc, -ma
    T[:3, 3] = T[:3, :3] @ -np.asarray(p, np.float32)
    P = np.float32([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, -0.2], [0, 0, -1, 0]])
    return P @ T


def test_snapshot_equals_cube_face(oracle):
    """forward -X, up -Y, 90 degrees, W = H = edge: the snapshot's matrix is the -X face's, exactly, and so is the
    render, bit for bit (winners included)."""
    W, E = 48, 64
    rig = synth.ring_rig(8, W, W, kind="FTHETA")
    colors, disps = synth.render_rig(rig, W, W, scene=synth.Scene(seed=2))
    bgra = [np.concatenate([c.astype(np.float32) / 65535, np.ones((W, W, 1), np.float32)], -1) for c in colors]
    pos = np.float32([0.02, -0.01, 0.0])
    M = capi.snapshot_matrix(pos, [-1, 0, 0], [0, -1, 0], 90.0, E, E)
    assert np.array_equal(M, _face_matrix_np(1, pos))
    d = capi.rig_descs(rig)
    cube = oracle.render(d, disps, bgra, pos, "cubemap", (E, E), want_disparity=True, want_winners=True)
    snap = oracle.render(d, disps, bgra, pos, "perspective", (E, E), M, want_disparity=True, want_winners=True)
    for a, b in zip(cube[:2], snap[:2]):
        assert np.array_equal(a[E:2 * E], b, equal_nan=True)
    assert np.array_equal(cube[2][:, E:2 * E], snap[2]) and (snap[2] >= 0).mean() > 0.3


def _eye_np(p, ipd):
    """canopyVS' eye() in fp64: ipd(lat), solve with two secant steps, inverse(A) * p.xy."""
    def ipd_at(lat):
        return ipd * np.exp(-np.exp(25 * (0.17 - 0.5 - lat / np.pi)) - np.exp(25 * (0.17 - 0.5 + lat / np.pi)))

    def err(d):
        return (p[..., 0] ** 2 + p[..., 1] ** 2) - (ipd_at(np.arctan(p[..., 2] / d)) / 2) ** 2 - d ** 2

    xy = np.hypot(p[..., 0], p[..., 1])
    d0 = np.sqrt(xy ** 2 - ipd_at(np.arctan(p[..., 2] / xy)) ** 2)
    for _ in range(2):
        d1 = 1.001 * d0
        e0, e1 = err(d0), err(d1)
        d0 = d0 - e0 / ((e1 - e0) / (d1 - d0))
    k = -d0 / (ipd_at(np.arctan(p[..., 2] / d0)) / 2)
    det = 1 + k * k
    return np.stack([(p[..., 0] + k * p[..., 1]) / det, (-k * p[..., 0] + p[..., 1]) / det], -1)


def test_eye_offset_matches_fp64(oracle):
    rng = np.random.default_rng(6)
    n = 2000
    r = rng.uniform(0.3, 50, n)
    lat = rng.uniform(-1.5, 1.5, n)
    lon = rng.uniform(-np.pi, np.pi, n)
    p = np.stack([r * np.cos(lat) * np.cos(lon), r * np.cos(lat) * np.sin(lon), r * np.sin(lat)], -1).astype(np.float32)
    f = _fn(oracle, "oracle_canopy_eye", None, [C.c_void_p, C.c_int, C.c_float, C.c_void_p])
    for ipd in (0.032, -0.032):
        out = np.empty((n, 2), np.float32)
        f(p.ctypes.data, n, ipd, out.ctypes.data)
        want = _eye_np(p.astype(np.float64), ipd)
        assert np.abs(out - want).max() <= 1e-6, np.abs(out - want).max()
        mag = np.hypot(out[:, 0], out[:, 1])
        eq = np.abs(lat) < 0.1
        assert np.abs(mag[eq] - 0.016).max() < 1e-3  # about ipd / 2 at the equator
        assert mag[np.abs(lat) > 1.45].max() < 1e-3  # near 0 at the poles


def test_single_canopy_without_blending_reproduces_its_texture(oracle):
    """Blending off: the weight is the fragment's alpha, so one canopy's colour is its own texture wherever it
    covers (a constant texture: every trilinear sample is the RGBA16 value)."""
    W = 32
    rig = synth.ring_rig(1, W, W)
    c = np.zeros((W, W, 4), np.float32)
    c[...] = (0.25, 0.5, 0.75, 1)
    col, _, _ = oracle.render(capi.rig_descs(rig), [np.full((W, W), 0.5, np.float32)], [c], np.zeros(3, np.float32),
                              "cubemap", (32, 32), alpha_blend=False)
    cov = col[..., 3] > 0
    assert cov.mean() > 0.2
    rgba16 = np.floor(np.float64([0.25, 0.5, 0.75]) * 65535 + 0.5) / 65535
    assert np.abs(col[cov][:, :3] - rgba16).max() <= 1e-6


def test_svd_rule_on_degenerate_jacobians(oracle):
    f = _fn(oracle, "oracle_canopy_svd_ratio", C.c_float, [C.c_float] * 4)
    assert f(0, 0, 0, 0) == 1.0  # zero Jacobian: ratio 1
    assert f(0.01, 0, 0, 0.01) == pytest.approx(1.0, abs=1e-6)
    assert f(0.01, 0, 0, 0.005) == pytest.approx(0.5, abs=1e-6)
    # rank 1: columns parallel; fp32 can make s1 - s2 negative there, and the rule gives sigma2 = 0, never NaN
    rng = np.random.default_rng(9)
    negative = 0
    for _ in range(2000):
        a, b = rng.uniform(-1, 1, 2).astype(np.float32) * np.float32(1e-3)
        t = np.float32(rng.uniform(-3, 3))
        c, d = a * t, b * t
        with np.errstate(invalid="ignore"):
            s1 = ((a * a + b * b) + c * c) + d * d
            sb = ((a * a + b * b) - c * c) - d * d
            sc = a * c + b * d
            s2 = np.sqrt(sb * sb + (np.float32(4) * sc) * sc)
        negative += bool(s1 - s2 < 0)
        r = f(a, b, c, d)
        assert r == r and 0 <= r <= 1e-3, (a, b, c, d, r)
    assert negative > 0


def test_canopy_header_is_plain_c_and_exported(tmp_path, oracle):
    hdr = open(os.path.join(capi.ROOT, "include", "derp_canopy.h")).read()
    declared = sorted(set(re.findall(r"\b(derp_canopy_[a-z0-9_]+)\s*\(", hdr)))
    assert declared == sorted(capi.CANOPY_SYMBOLS)
    prod = C.CDLL(capi.CUDA_LIB, mode=C.RTLD_LOCAL)
    for name in declared:
        assert hasattr(prod, name), name
    assert hasattr(oracle.lib, "derp_canopy_render")
    src = tmp_path / "canopy.c"
    src.write_text('#include "derp_canopy.h"\n#include <stdio.h>\nint main(void) { float p[3] = {0, 0, 0}, '
                   'f[3] = {-1, 0, 0}, u[3] = {0, 0, 1}, m[16]; printf("%s\\n", derp_backend()); '
                   'if (derp_canopy_snapshot_matrix(p, f, u, 90.0, 4, 4, m) != DERP_OK || m[1] != 1.0f) return 2; '
                   'return derp_canopy_render(0, 0, 0, 0, 2, 2, 0, 0, 0, DERP_CANOPY_CUBEMAP, 0, 0, 2, 2, 0.0f, 1, '
                   'DERP_CANOPY_SVD, 0, 0, 0) == DERP_EINVAL ? 0 : 1; }\n')
    libdir = os.path.dirname(capi.CUDA_LIB)
    exe = tmp_path / "canopy"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(capi.ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lderp_b200",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "cuda-sm_90a", (out.returncode, out.stdout)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rig = synth.ring_rig(2, 16, 16)
    lib = capi.Canopy(capi.load_cuda())
    with pytest.raises(capi.DerpError) as e:
        lib.render(capi.rig_descs(rig), [np.ones((16, 16), np.float32)] * 2, [np.ones((16, 16, 4), np.float32)] * 2,
                   np.zeros(3, np.float32), "equirect", (32, 16))
    assert e.value.code == capi.ECUDA
