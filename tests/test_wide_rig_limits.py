"""Rigs of 33 to 64 cameras without a GPU: the camera limit of the CUDA library and DerpCLI (64, refused above with
DERP_EINVAL / a CHECK before any device is touched), and the oracle pinned to the reference's own code on a 40-camera
rig, so that the GPU parity tests of tests/test_gpu_wide_rig.py compare against a checker that is itself right there."""
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import ref_digests
from tests.parity_util import both
from tests.test_apps import write_dataset

BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")
HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")
DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_rig_reference_digests.json")


@pytest.fixture
def refcheck(request, monkeypatch):
    """tests/ref_digests.py's refcheck (live against oracle/_ref, else replayed), with this file's digests kept in a
    golden file of their own."""
    from tests import oracle_libs
    monkeypatch.setattr(ref_digests, "PATH", DIGESTS)
    d = ref_digests.Digests("test_wide_rig_limits::" + request.node.name, oracle_libs.load_ref() is None)
    yield d
    d.finish()


def _gpu_present():
    import torch
    return torch.cuda.is_available()


@pytest.fixture(scope="module")
def prod():
    return capi.load_cuda()  # loads on a CPU box: cudart is linked statically


def test_derp_create_refuses_more_than_64_cameras(prod):
    descs = capi.rig_descs(synth.wall_rig(65, 32, 24))
    with pytest.raises(capi.DerpError) as e:
        capi.Context(prod, descs)
    assert e.value.code == capi.EINVAL
    assert "at most 64 cameras" in str(e.value)


def test_derp_create_accepts_64_cameras(prod):
    """64 cameras pass the count check, which comes before the device lookup: without a GPU the next error is the
    missing device."""
    descs = capi.rig_descs(synth.wall_rig(64, 32, 24))
    if _gpu_present():
        capi.Context(prod, descs).close()
        return
    with pytest.raises(capi.DerpError) as e:
        capi.Context(prod, descs)
    assert e.value.code == capi.ECUDA


def _derpcli(tmp_path, num_cams):
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    W = H = 16
    rig = synth.wall_rig(num_cams, W, H)
    colors = synth.random_colors(num_cams, W, H)
    write_dataset(str(tmp_path / "in"), rig, [colors], 1)
    return subprocess.run([os.path.join(BIN, "DerpCLI"), "--input_root=" + str(tmp_path / "in"),
                           "--output_root=" + str(tmp_path / "out"), "--partial_coverage"], capture_output=True, text=True)


def test_derpcli_refuses_65_cameras(tmp_path):
    p = _derpcli(tmp_path, 65)
    assert p.returncode != 0 and "rigs of up to 64 cameras" in p.stderr, p.stderr[-2000:]


def test_derpcli_takes_40_cameras_past_the_limit_check(tmp_path):
    if _gpu_present():
        pytest.skip("GPU present: the end-to-end run is tests/test_gpu_wide_rig.py")
    p = _derpcli(tmp_path, 40)
    assert "rigs of up to 64 cameras" not in p.stderr
    assert p.returncode != 0 and "CUDA" in p.stderr  # the next thing that stops it is the missing GPU


W40, H40 = 48, 36


def _wall40():
    rig = synth.wall_rig(40, W40, H40)
    colors, true_disp = synth.render_rig(rig, W40, H40, scene=synth.Scene(seed=7))
    return rig, colors, true_disp


def _bits(a):
    """Float bits with every NaN mapped to one pattern (the comparisons treat all NaNs as equal)."""
    a = np.ascontiguousarray(a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)


def _pair(oracle, rig):
    from tests import oracle_libs
    ref = oracle_libs.load_ref() or oracle  # replay: the oracle's outputs are checked against the recorded digests
    descs = capi.rig_descs(rig)
    return capi.Context(oracle, descs), capi.Context(ref, descs)


def test_reference_pin_40_cameras_cost_and_brute_force(oracle, refcheck):
    """computeCost on hypothesis maps and brute force (150 candidates, the reference's constant) on a 40-camera wall: up to
    39 sources per cost, destinations on both sides of camera 32."""
    rig, colors, true_disp = _wall40()
    ctxs = _pair(oracle, rig)
    both(ctxs, "level_begin", W40, H40)
    both(ctxs, "set_colors", colors)
    rng = np.random.RandomState(5)
    for d in (3, 36):
        both(ctxs, "reproject", d)
        for disp in (true_disp[d], rng.uniform(1e-4, 2.0, (H40, W40)).astype(np.float32)):
            (oc, of), (rc, rf) = both(ctxs, "eval_cost", d, disp)
            assert refcheck.same(_bits(oc), _bits(rc)) and refcheck.same(_bits(of), _bits(rf))
        oi, ri = both(ctxs, "brute_force", d, num_depths=150)
        assert refcheck.same(oi, ri)
        for o, r in zip(*both(ctxs, "get_disparity", d)):
            assert refcheck.same(_bits(o), _bits(r))


def test_reference_pin_40_cameras_fine_level(oracle, refcheck):
    """One fine level of a 40-camera rig stage by stage: random proposals and ping-pong on destinations below and above
    camera 32, then mismatch handling over every camera, bilateral, median and maskFov."""
    rig, colors, true_disp = _wall40()
    S = len(colors)
    ctxs = _pair(oracle, rig)
    both(ctxs, "level_begin", W40, H40, level=0, num_levels=2, full_width=W40, full_height=H40)
    both(ctxs, "set_colors", colors)
    rng = np.random.RandomState(3)
    for d in range(S):
        start = np.clip(true_disp[d] * rng.uniform(0.85, 1.2, (H40, W40)).astype(np.float32), 1e-4, 2.0).astype(np.float32)
        both(ctxs, "set_disparity", d, start, np.zeros_like(start), np.zeros_like(start))

    def check(dsts):
        for d in dsts:
            o, r = both(ctxs, "get_disparity", d, want_cost=False)
            assert refcheck.same(_bits(o), _bits(r)), d

    for d in (1, 33, 39):
        both(ctxs, "reproject", d)
        both(ctxs, "random_proposals", d, 2)
        check([d])
        both(ctxs, "ping_pong", d, 2)
        check([d])
    both(ctxs, "mismatches")
    check(range(S))
    for d in range(S):
        o, r = both(ctxs, "get_mismatch_mask", d)
        assert refcheck.same(o, r)
    for stage in ("bilateral", "median", "mask_fov"):
        for d in range(S):
            both(ctxs, stage, d)
        check(range(S))
