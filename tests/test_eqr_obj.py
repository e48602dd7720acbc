"""CreateObjFromDisparityEquirect (source/conversion/CreateObjFromDisparityEquirect.cpp): disparity equirect -> OBJ.
CPU: the oracle restatement of the equirect mesh against the reference's own MeshUtil.h and MeshSimplifier.cpp
(oracle/_ref), the library's host simplifier with the relative cost, the host instantiation of the INTER_LINEAR resize
against cv2 4.13 (tests/golden/linear_vectors.npz, generator tests/golden/gen_linear_vectors.py), the app's flags,
refusals and FATALs.  The GPU side is tests/test_gpu_eqr_obj.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import eqrmesh_oracle
from tests.golden import gen_linear_vectors

BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")
APP = os.path.join(BIN, "CreateObjFromDisparityEquirect")
REF_APP = "/root/reference/source/conversion/CreateObjFromDisparityEquirect.cpp"


@pytest.fixture(scope="module")
def eqr():
    """The product's binding of include/derp_eqrmesh.h (host hooks only on the CPU)."""
    return capi.EqrMesh(capi.load_cuda())


@pytest.fixture(scope="module")
def eqr_oracle():
    return eqrmesh_oracle.load_oracle()


@pytest.fixture(scope="module")
def eqr_ref():
    lib = eqrmesh_oracle.load_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libeqrmesh_ref.so not built (needs the reference sources)")
    return lib


def room(w, h):
    """A smooth room: disparity of a box around the centre, seen along every equirect ray."""
    theta = (np.arange(w) + 0.5) / w * 2 * np.pi
    phi = (np.arange(h) + 0.5) / h * np.pi
    dx = np.abs(np.sin(phi)[:, None] * np.cos(theta)[None, :]) / 3.0
    dy = np.abs(np.cos(phi))[:, None] / 2.5 * np.ones((1, w))
    dz = np.abs(np.sin(phi)[:, None] * np.sin(theta)[None, :]) / 4.0
    return np.maximum(np.maximum(dx, dy), dz).astype(np.float32)


def jumps(w, h, seed):
    """Depth jumps far beyond the 0.95 tear ratio, and ratios close to it."""
    rng = np.random.RandomState(seed)
    d = room(w, h)
    yy, xx = np.mgrid[0:h, 0:w]
    d[(xx + 2 * yy) % 23 < 8] *= 1.7
    return (d * rng.uniform(0.975, 1.025, d.shape)).astype(np.float32)


def specials(w, h, seed):
    """NaN, 0, +-inf and negative disparities, and disparities below 1 / max_depth (the clamp)."""
    rng = np.random.RandomState(seed)
    d = jumps(w, h, seed)
    vals = np.array([np.nan, 0.0, np.inf, -np.inf, -0.3, 1e-5, 5e-4], np.float32)
    m = rng.uniform(size=d.shape) < 0.15
    d[m] = rng.choice(vals, size=int(m.sum()))
    return d


# (name, w, h, scale, max_depth, tear)
CASES = [("room", 64, 32, 1.0, 700.0, 0.95), ("jumps", 72, 36, 1.0, 700.0, 0.95), ("specials", 48, 24, 1.0, 20.0, 0.95),
         ("specials", 2, 2, 1.0, 700.0, 0.95), ("specials", 3, 2, 1.0, 700.0, 0.95), ("jumps", 31, 17, 1.0, 700.0, 0.9),
         ("specials", 2, 7, 1.0, 1000.0, 0.95), ("room", 40, 20, 1.0, 700.0, 0.0)]
SCALED = [("jumps", 96, 48, 0.5, 700.0, 0.95), ("specials", 101, 53, 0.37, 700.0, 0.95)]


def make(name, w, h, seed=0):
    return {"room": lambda: room(w, h), "jumps": lambda: jumps(w, h, seed), "specials": lambda: specials(w, h, seed)}[name]()


def same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a,
                                                 b.view(np.uint64) if b.dtype == np.float64 else b)


@pytest.mark.parametrize("case", CASES + SCALED)
def test_oracle_equals_reference(eqr_oracle, eqr_ref, case):
    name, w, h, scale, max_depth, tear = case
    d = make(name, w, h)
    ov, of = eqr_oracle.mesh(d, scale=scale, max_depth=max_depth, tear_ratio=tear)
    rv, rf = eqr_ref.mesh(d, scale=scale, max_depth=max_depth, tear_ratio=tear)
    assert same(of, rf) and same(ov, rv)
    assert len(ov) == len(rv) and of.max() < len(ov)
    H = int(np.rint(h * scale)) if scale < 1 else h
    assert len(of) >= 2 * (H - 1)  # at least the wrap faces


def test_vertexes_by_hand(eqr_oracle):
    """2 x 2 at disparity 0.5: depth 2 on the four directions theta = pi / 2, 3 pi / 2, phi = pi / 4, 3 pi / 4; NaN and 0 go to
    max_depth; the two wrap faces follow the quad's faces."""
    d = np.full((2, 2), 0.5, np.float32)
    v, f = eqr_oracle.mesh(d)
    assert np.allclose(np.linalg.norm(v, axis=1), 2.0, rtol=1e-6)
    assert np.array_equal(f[-2:], [[2, 0, 1], [1, 3, 2]])
    d[0, 0], d[1, 1] = np.nan, 0.0
    v, _ = eqr_oracle.mesh(d, max_depth=9.0)
    assert np.allclose(np.linalg.norm(v[[0, 3]], axis=1), 9.0, rtol=1e-6)


def _simplify(lib, name, xyz, idx, triangles, strictness):
    f = getattr(lib.lib, name)
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                  C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    xyz = np.ascontiguousarray(xyz, np.float64)
    idx = np.ascontiguousarray(idx, np.uint32)
    ov, oi = np.empty_like(xyz), np.empty_like(idx)
    nv, nf = C.c_uint64(), C.c_uint64()
    assert f(xyz.ctypes.data, len(xyz), idx.ctypes.data, len(idx), triangles, strictness, ov.ctypes.data, oi.ctypes.data,
             C.byref(nv), C.byref(nf)) == 0
    return ov[:nv.value].copy(), oi[:nf.value].copy()


def cylinder(w, h, seed):
    """A wrapped cylinder (the equirect wrap faces close it) with a little radial noise."""
    rng = np.random.RandomState(seed)
    t = (np.arange(w) + 0.5) / w * 2 * np.pi
    r = 3.0 + rng.uniform(-0.01, 0.01, (h, w))
    xyz = np.stack([r * np.cos(t)[None, :], np.repeat(np.linspace(-1, 1, h)[:, None], w, 1), r * np.sin(t)[None, :]], 2)
    q = (np.arange(h - 1)[:, None] * w + np.arange(w - 1)[None, :]).ravel().astype(np.uint32)
    idx = [np.stack([q + w, q + 1, q], 1), np.stack([q + 1, q + w, q + w + 1], 1)]
    b = (np.arange(h - 1) * w).astype(np.uint32)
    idx += [np.stack([b + w, b, b + w - 1], 1), np.stack([b + w - 1, b + 2 * w - 1, b + w], 1)]
    return xyz.reshape(-1, 3), np.concatenate(idx)


@pytest.mark.parametrize("mesh,target,strictness", [("cyl", 300, 0.8), ("cyl", 50, 1.0), ("torn", 800, 0.8),
                                                    ("torn", 200, 0.5), ("torn", 10 ** 6, 0.8)])
def test_relative_simplifier_equals_reference(eqr_oracle, eqr_ref, mesh, target, strictness):
    """derp_simplify.h with MeshSimplifier's relative cost (isEquiError = false) against the reference's own code."""
    prod = capi.load_cuda()
    if mesh == "cyl":
        xyz, idx = cylinder(40, 20, 3)
    else:
        xyz, idx = eqr_oracle.mesh(specials(60, 30, 4), max_depth=50.0)
    pv, pi = _simplify(prod, "derp_test_simplify_relative", xyz, idx, target, strictness)
    rv, ri = _simplify(eqr_ref, "derp_ref_simplify_relative", xyz, idx, target, strictness)
    assert same(pi, ri) and same(pv, rv)
    if target < len(idx):
        assert len(pi) < len(idx)


@pytest.mark.parametrize("strictness,num_faces", [(0.8, 500), (1.0, 300), (0.8, 10 ** 6)])
def test_reference_simplified_mesh_is_the_product_simplifier(eqr_oracle, eqr_ref, strictness, num_faces):
    """The reference's whole app body (mesh + MeshSimplifier(..., false, 1)) equals the oracle mesh through the library's
    host simplifier: the two halves the GPU path chains."""
    d = jumps(48, 24, 5)
    xyz, idx = eqr_oracle.mesh(d)
    pv, pi = _simplify(capi.load_cuda(), "derp_test_simplify_relative", xyz, idx, num_faces, strictness)
    rv, rf = eqr_ref.mesh(d, num_faces=num_faces, strictness=strictness)
    assert same(pi, rf) and same(pv, rv)


def _resize_host(lib, name, src, scale, dw, dh):
    src = np.ascontiguousarray(src, np.float32)
    out = np.empty((dh, dw), np.float32)
    f = getattr(lib.lib, name)
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
    f(src.ctypes.data, src.shape[1], src.shape[0], scale, out.ctypes.data)
    return out


def test_resize_linear_against_cv2(eqr, eqr_oracle):
    """INTER_LINEAR by factors on floats: the host instantiation of resizeLinearKernel's per-pixel function equals the
    oracle's restatement bit for bit, and both are within 2.5e-7 absolute of cv2 4.13 on (0, 1] data (shape exact)."""
    G = np.load(os.path.join(os.path.dirname(__file__), "golden", "linear_vectors.npz"))
    prod = capi.load_cuda()
    for i, (w, h, f) in enumerate(gen_linear_vectors.CASES):
        want = G["linear_%d" % i]
        src = gen_linear_vectors.source(i, w, h)
        dh, dw = want.shape
        got = _resize_host(prod, "derp_test_resize_linear_host", src, f, dw, dh)
        ora = _resize_host(eqr_oracle, "oracle_resize_linear_f32", src, f, dw, dh)
        assert np.array_equal(got.view(np.uint32), ora.view(np.uint32)), (w, h, f)
        assert np.abs(got - want).max() <= 2.5e-7, (w, h, f, np.abs(got - want).max())


@pytest.mark.parametrize("w,h,scale", [(8, 4, 0.0), (8, 4, -1.0), (8, 4, float("nan")), (1, 8, 1.0), (8, 1, 1.0),
                                       (8, 4, 0.2), (0, 4, 1.0)])
def test_refusals(eqr, eqr_oracle, eqr_ref, w, h, scale):
    """scale <= 0 or NaN (OpenCV throws on the empty size), grids below 2 x 2 — in every library."""
    for lib in (eqr_oracle, eqr_ref, eqr):
        mw, mh = C.c_int(), C.c_int()
        assert lib.lib.derp_equirect_mesh_size(w, h, scale, C.byref(mw), C.byref(mh)) == capi.EINVAL
    for lib in (eqr_ref, eqr):  # the product refuses before it looks for a device
        with pytest.raises(capi.DerpError):
            lib.mesh(np.ones((4, 8), np.float32), strictness=1.5)
    with pytest.raises(capi.DerpError):
        eqr_ref.mesh(np.ones((4, 8), np.float32), strictness=1.5)


def _ref_defines():
    return sorted(re.findall(r"^(DEFINE_\w+\(\w+, .*\);)$", open(REF_APP).read(), re.M))


def test_flag_surface_matches_reference():
    if not os.path.exists(REF_APP):
        pytest.skip("reference sources not present")
    ours = re.findall(r"^(DEFINE_\w+\(\w+, .*\);)$",
                      open(os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host",
                                        "CreateObjFromDisparityEquirect.cpp")).read(), re.M)
    extra = [d for d in ours if d not in _ref_defines()]
    assert sorted(set(ours) - set(extra)) == _ref_defines()
    assert extra == ['DEFINE_int32(gpu, 0, "CUDA device to use");']


def _run(args, tmp_path):
    return subprocess.run([APP] + args, capture_output=True, text=True, cwd=str(tmp_path))


def test_app_checks(tmp_path):
    """The reference's CHECKs: the three required paths and 0 <= strictness <= 1 abort before anything is read."""
    full = ["--input_png_disp=d.png", "--input_png_color=c.png", "--output_obj=o.obj"]
    for drop in range(3):
        p = _run(full[:drop] + full[drop + 1:], tmp_path)
        assert p.returncode != 0 and "Check failed" in p.stderr
    for s in ("-0.1", "1.5"):
        p = _run(full + ["--strictness=" + s], tmp_path)
        assert p.returncode != 0 and "strictness must be between 0 and 1" in p.stderr
    assert not (tmp_path / "o.obj").exists()


def test_app_without_gpu_is_fatal(tmp_path):
    """No CPU fallback: without a device the mesh call fails and the app aborts without writing the OBJ."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    d = (np.ones((8, 16)) * 0.5).astype(np.float32)
    with open(tmp_path / "d.pfm", "wb") as f:
        f.write(b"Pf\n16 8\n-1\n" + d[::-1].tobytes())
    p = _run(["--input_png_disp=d.pfm", "--input_png_color=c.png", "--output_obj=o.obj", "--strictness=0"], tmp_path)
    assert p.returncode != 0 and "derp_equirect_mesh" in p.stderr
    assert not (tmp_path / "o.obj").exists()


@pytest.mark.parametrize("kind", ["gray8", "gray16", "bgr8", "bgr16", "bgra8", "bgra16"])
def test_load_float_matches_cv2(tmp_path, kind):
    """io::loadFloat (the app's reader, loadImage<float> semantics) against cv2: imread, scale to [0, 1], BGR(A)2GRAY.
    The reader is not bit-exact to this chain: it differs in the last bits (up to 2 ulp of values in [0, 1])."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(len(kind))
    dt = np.uint16 if kind.endswith("16") else np.uint8
    ch = {"gray": 1, "bgr": 3, "bgra": 4}[kind[:-2] if kind.endswith("16") else kind[:-1]]
    img = rng.randint(0, np.iinfo(dt).max + 1, (13, 21, ch) if ch > 1 else (13, 21)).astype(dt)
    cv2.imwrite(str(tmp_path / "in.png"), img)
    subprocess.run([os.path.join(BIN, "IoSelfTest"), "--mode=float", "--in=" + str(tmp_path / "in.png"),
                    "--out=" + str(tmp_path / "out.bin")], check=True, capture_output=True)
    got = np.fromfile(str(tmp_path / "out.bin"), np.float32).reshape(13, 21)
    f = cv2.imread(str(tmp_path / "in.png"), cv2.IMREAD_UNCHANGED).astype(np.float32) / np.iinfo(dt).max
    if ch == 3:
        f = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
    elif ch == 4:
        f = cv2.cvtColor(f, cv2.COLOR_BGRA2GRAY)
    assert np.abs(got - f).max() <= 2.5e-7, np.abs(got - f).max()


def test_exports_every_declared_symbol(eqr, eqr_oracle):
    """include/derp_eqrmesh.h: the product and the oracle export every declared entry point, and the binding covers them."""
    hdr = open(os.path.join(capi.ROOT, "include", "derp_eqrmesh.h")).read()
    declared = sorted(re.findall(r"^int (derp_[a-z0-9_]+)\(", hdr, re.M))
    assert declared == capi.EQR_SYMBOLS
    for lib in (eqr, eqr_oracle):
        for name in declared + ["derp_last_error"]:
            assert hasattr(lib.lib, name), (lib.path, name)
