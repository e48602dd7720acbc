import os
"""CPU-only checks of the PRODUCT library (libderp_b200.so): it must load without a GPU, export every
symbol include/derp_b200.h declares, fail loudly on compute calls, and the host instantiations of its
__host__ __device__ building blocks (introselect emulation, minstd skip-ahead, camera) must agree with
libstdc++ / the oracle.  No GPU compute here."""
import ctypes as C
import itertools
import re

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import oracle_hooks as oh


@pytest.fixture(scope="module")
def prod():
    return capi.load_cuda()  # loads on a CPU box: cudart is linked statically


def test_exports_every_declared_symbol(prod, oracle):
    hdr = open(capi.ROOT + "/include/derp_b200.h").read()
    declared = sorted(set(re.findall(r"\b(derp_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 30
    for lib in (prod, oracle):
        for name in declared:
            assert hasattr(lib.lib, name), "%s misses %s" % (lib.path, name)
    assert set(declared) == set(capi.ABI_SYMBOLS), set(declared) ^ set(capi.ABI_SYMBOLS)
    assert prod.backend == "cuda-sm_90a" and oracle.backend == "oracle-cpu"


def test_header_is_plain_c(tmp_path):
    """The boundary is a C ABI: include/derp_b200.h must compile as C99 (no C++ or CUDA types in the signatures) and a C
    program must link against the library with nothing but that header."""
    import subprocess
    src = tmp_path / "cabi.c"
    src.write_text('#include "derp_b200.h"\n#include <stdio.h>\nint main(void) { printf("%s\\n", derp_backend()); '
                   'return derp_bc7_compress(0, 0, 0, 0, 0) == 0; }\n')
    exe = tmp_path / "cabi"
    libdir = os.path.dirname(capi.CUDA_LIB)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", capi.ROOT + "/include", str(src),
                           "-o", str(exe), "-L", libdir, "-lderp_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "cuda-sm_90a"  # bad arguments -> DERP_EINVAL, no CUDA call needed


def test_no_cpu_fallback_without_gpu(prod):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    descs = capi.rig_descs(synth.ring_rig(4, 64, 64))
    with pytest.raises(capi.DerpError) as e:
        capi.Context(prod, descs)
    assert e.value.code == capi.ECUDA


def _robust(prod, a, b, keep):
    f = prod.lib.derp_test_robust_sum
    f.restype = C.c_float
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return f(a.ctypes.data, b.ctypes.data, len(a), keep)


def test_robust_sum_matches_libstdcxx_nth_element(prod, oracle):
    rng = np.random.RandomState(7)
    n_cases = 0
    for n in range(1, 32):
        keep = max(1, n - 2)
        for trial in range(300):
            mode = trial % 4
            if mode == 0:
                a = rng.uniform(0, 1, n)
            elif mode == 1:  # many ties in the key
                a = rng.randint(0, 3, n).astype(np.float64)
            elif mode == 2:  # sorted / reverse sorted (introsort worst cases)
                a = np.sort(rng.uniform(0, 1, n))[:: (1 if trial % 8 < 4 else -1)]
            else:  # organ pipe
                h = np.sort(rng.uniform(0, 1, n))
                a = np.concatenate([h[::2], h[1::2][::-1]])
            b = rng.uniform(0, 1e-3, n) * np.float32(10.0) ** rng.randint(-3, 4, n)
            a32, b32 = a.astype(np.float32), b.astype(np.float32)
            want = oh.nth_element_sum(oracle, a32, b32, keep)
            got = _robust(prod, a32, b32, keep)
            assert np.float32(want).tobytes() == np.float32(got).tobytes(), (n, trial, want, got)
            n_cases += 1
    assert n_cases > 9000


def test_robust_sum_all_permutations_small(prod, oracle):
    base = np.array([0.3, 0.1, 0.7, 0.5, 0.2, 0.9], np.float32)
    bsec = np.array([1e-3, 3e-7, 2.5e-1, 7e-5, 9e-2, 4e-6], np.float32)
    for n in (4, 5, 6):
        for perm in itertools.permutations(range(n)):
            a, b = base[list(perm)], bsec[list(perm)]
            want = oh.nth_element_sum(oracle, a, b, n - 2)
            got = _robust(prod, a, b, n - 2)
            assert np.float32(want).tobytes() == np.float32(got).tobytes()


def _minstd(prod, seed, skip, n, lo, hi):
    f = prod.lib.derp_test_minstd_uniform
    f.restype = None
    f.argtypes = [C.c_uint32, C.c_uint64, C.c_int, C.c_float, C.c_float, C.c_void_p]
    out = np.empty(n, np.float32)
    f(seed, skip, n, lo, hi, out.ctypes.data)
    return out


def test_minstd_stream_matches_libstdcxx(prod, oracle):
    # known answers probed from libstdc++ (SURVEY.md §7): seed(0), U(0.25, 1.75)
    ka = _minstd(prod, 0, 0, 3, 0.25, 1.75)
    assert np.allclose(ka, [0.250011742, 0.447306693, 1.38340807], rtol=0, atol=1e-8)
    for seed in (0, 1, 5, 12345, 2147483647, 2147483646, 4000000000 % (2 ** 32)):
        for lo, hi in ((0.0, 1.0), (1e-4, 2.0), (0.37, 0.370001)):
            ref = oh.minstd_uniform(oracle, seed, 3000, lo, hi)
            got = _minstd(prod, seed, 0, 3000, lo, hi)
            assert np.array_equal(ref, got)
            # skip-ahead == sequential discard
            for skip in (1, 2, 17, 1023, 2999):
                g2 = _minstd(prod, seed, skip, 3000 - skip, lo, hi)
                assert np.array_equal(ref[skip:], g2)


def _prod_sees(prod, desc, pts, normalized):
    f = prod.lib.derp_test_camera_sees
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.CameraDesc), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    pts = np.ascontiguousarray(pts, np.float64)
    pix = np.empty((len(pts), 2))
    seen = np.empty(len(pts), np.uint8)
    prod.check(f(C.byref(desc), int(normalized), pts.ctypes.data, len(pts), pix.ctypes.data, seen.ctypes.data))
    return pix, seen.astype(bool)


def _prod_rig(prod, desc, pix, depth):
    f = prod.lib.derp_test_camera_rig
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.CameraDesc), C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    pix = np.ascontiguousarray(pix, np.float64)
    pts = np.empty((len(pix), 3))
    out = np.empty(len(pix), np.uint8)
    prod.check(f(C.byref(desc), pix.ctypes.data, len(pix), depth, pts.ctypes.data, out.ctypes.data))
    return pts, out.astype(bool)


@pytest.mark.parametrize("kind", ["FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"])
def test_product_camera_matches_oracle_bitwise(prod, oracle, kind):
    rig = synth.ring_rig(6, 640, 480, kind="FTHETA", distortion=[-0.0341, 0.00044, -0.0019])
    cam = dict(rig["cameras"][2])
    cam["type"] = kind
    if kind in ("RECTILINEAR", "ORTHOGRAPHIC"):
        cam["fov"] = 1.2
    cam["principal"] = [322.5, 236.25]
    d = capi.camera_desc_from_json(cam)
    rng = np.random.RandomState(3)
    pts = np.array(cam["origin"]) + rng.normal(size=(4000, 3)) * rng.uniform(0.3, 20, size=(4000, 1))
    for normalized in (False, True):
        p_pix, p_seen = _prod_sees(prod, d, pts, normalized)
        o_pix, o_seen = oh.camera_project(oracle, d, pts, normalized)
        assert np.array_equal(p_seen, o_seen)
        # same operation order, same libm on the host: bit-identical where the point is seen
        assert np.array_equal(p_pix[p_seen], o_pix[o_seen])
    pix = rng.uniform(0, 1, size=(2000, 2)) * np.array([640, 480])
    p_pts, p_out = _prod_rig(prod, d, pix, 7.5)
    o_pts, o_out = oh.camera_unproject(oracle, d, pix, 7.5)
    assert np.array_equal(p_out, o_out)
    assert np.array_equal(p_pts, o_pts)
    f = prod.lib.derp_test_camera_info
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.CameraDesc), C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    rot = np.empty(9)
    dm, cf = C.c_double(), C.c_double()
    prod.check(f(C.byref(d), rot.ctypes.data, C.byref(dm), C.byref(cf)))
    orot, odm, ocf = oh.camera_info(oracle, d)
    assert np.array_equal(rot.reshape(3, 3), orot) and dm.value == odm and cf.value == ocf


def _table(prod, a, b, keep):
    f = prod.lib.derp_test_select_table
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    out = np.zeros(1, np.float32)
    ok = f(a.ctypes.data, b.ctypes.data, len(a), keep, out.ctypes.data)
    return ok, out[0]


def test_table_driven_selection_equals_general_algorithm(prod):
    """derp_select.cuh's permutation-table path, which the cost kernels use for 4..8 sources, against the general
    libstdc++-order algorithm they fall back to: every permutation for n = 4..8, bit-identical fp32 sums; ties / NaNs
    in the first key must be declined."""
    import itertools
    rng = np.random.RandomState(11)
    checked = 0
    for n in range(4, 9):
        keep = n - 2
        perms = itertools.permutations(range(n))  # exhaustive, n = 8 included (40 320 arrangements)
        for perm in perms:
            a = (np.array(perm, np.float32) + 1) * np.float32(0.37) + rng.uniform(0, 0.1)
            b = rng.uniform(0, 3, n).astype(np.float32)  # sums of these depend on the order in the last bit
            ok, got = _table(prod, a, b, keep)
            assert ok == 1
            want = _robust(prod, a, b, keep)
            assert np.float32(got).view(np.uint32) == np.float32(want).view(np.uint32), (n, perm)
            checked += 1
    assert checked == 24 + 120 + 720 + 5040 + 40320
    # declined inputs: equal first keys, NaN, sizes outside 4..8
    a = np.array([0.3, 0.1, 0.3, 0.7, 0.2], np.float32)
    assert _table(prod, a, a, 3)[0] == 0
    a2 = a.copy()
    a2[2] = np.nan
    assert _table(prod, a2, a, 3)[0] == 0
    assert _table(prod, a[:3], a[:3], 1)[0] == 0
    # equal keys are fine when they are not among the first keys
    a3 = np.array([0.5, 0.1, 0.3, 0.7, 0.2], np.float32)
    b3 = np.array([1.0, 1.0, 1.0, 2.0, 2.0], np.float32)
    ok, got = _table(prod, a3, b3, 3)
    assert ok == 1 and np.float32(got) == np.float32(_robust(prod, a3, b3, 3))
