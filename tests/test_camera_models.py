"""The oracle pinned to the reference's own code on every camera model and FOV cone of the rig format: EQUISOLID and
ORTHOGRAPHIC cameras, FTHETA cameras that see behind themselves or through a cone wider than 180 deg, RECTILINEAR
cameras with a cone, a rig that mixes the four types, and odd sensors whose central ray is the optical axis
(tests/camera_models_util.py).  tests/test_gpu_camera_models.py compares the CUDA library with the oracle on the same
rigs, so this module is what makes the oracle a valid checker there.

Like tests/test_reference_pin.py every comparison is bit for bit (NaN == NaN), live against oracle/_ref when it is
built, otherwise against digests of the reference's outputs recorded with DERP_RECORD_REFERENCE_DIGESTS set, kept in
tests/golden/camera_models_reference_digests.json.  Every stage runs on every rig: the level tables, computeCost on
three disparity maps, brute force at the reference's 150 candidates, the fine-level stages, a two-level processLevel
and upsampleDisparity with the FOV masks of a rescaled camera of each type."""
import os

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import camera_models_util as cm
from tests import oracle_libs, ref_digests
from tests.parity_util import both, same_float_bits

REPLAY = oracle_libs.load_ref() is None
DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "camera_models_reference_digests.json")
NAMES = list(cm.RIGS)
_digests = None


@pytest.fixture(scope="module")
def ref(oracle):
    """The reference's own code, or (replay) the oracle, whose outputs eq_bits checks against the recorded digests."""
    return oracle if REPLAY else oracle_libs.load_ref()


@pytest.fixture(autouse=True)
def reference_digests(request, monkeypatch):
    global _digests
    monkeypatch.setattr(ref_digests, "PATH", DIGESTS)
    _digests = ref_digests.Digests("test_camera_models::" + request.node.name, REPLAY)
    yield
    _digests.finish()


def eq_bits(a, b):
    """a (ours) equals b (the reference's output), bit for bit."""
    if REPLAY:
        return _digests.compare(a, None)
    _digests.compare(a, b)
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        return bool(same_float_bits(a, b).all())
    return bool(np.array_equal(a, b))


def pair(oracle, ref, rig):
    descs = capi.rig_descs(rig)
    return capi.Context(oracle, descs), capi.Context(ref, descs)


def level_colors(name, level):
    """Colours of pyramid level `level`: the scene rendered at that size (the odd sensors do not halve exactly)."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    if level == 0:
        return colors
    return synth.render_rig(rig, W >> level, H >> level, scene=synth.Scene(seed=cm.SCENE_SEED))[0]


@pytest.mark.parametrize("name", NAMES)
def test_tables_cost_and_brute_force(oracle, ref, name):
    """generateFovMasks, computeImageVariance, the warp / colour / bias tables, computeCost on a constant, the true and
    a random disparity map, and brute force with its disparity, cost and confidence."""
    rig, colors, true_disp, W, H = cm.rig_inputs(name)
    S = len(colors)
    ctxs = pair(oracle, ref, rig)
    both(ctxs, "level_begin", W, H)
    both(ctxs, "set_colors", colors)
    masks = []
    for d in range(S):
        o, r = both(ctxs, "get_fov_mask", d)
        assert eq_bits(o, r), ("generateFovMasks", d)
        masks.append(o)
        o, r = both(ctxs, "get_variance", d)
        assert eq_bits(o, r), ("computeImageVariance", d)
    rng = np.random.RandomState(3)
    winners = {}
    for d in cm.DSTS:
        both(ctxs, "reproject", d)
        for s in range(S):
            for getter in ("get_proj_warp", "get_proj_color", "get_proj_bias"):
                o, r = both(ctxs, getter, s)
                assert eq_bits(o, r), (getter, d, s)
        for disp in (np.full((H, W), 0.31, np.float32), true_disp[d], rng.uniform(1e-4, 2.0, (H, W)).astype(np.float32)):
            (oc, of), (rc, rf) = both(ctxs, "eval_cost", d, disp)
            assert eq_bits(oc, rc) and eq_bits(of, rf), ("computeCost", d)
        oi, ri = both(ctxs, "brute_force", d, num_depths=150)
        assert eq_bits(oi, ri), ("winner indices", d)
        winners[d] = oi
        for o, r in zip(*both(ctxs, "get_disparity", d)):
            assert eq_bits(o, r), ("brute-force disparity / cost / confidence", d)
    cm.check_coverage(name, masks, winners)


@pytest.mark.parametrize("name", NAMES)
def test_fine_level_stages(oracle, ref, name):
    """Lanczos upsampling of an oracle brute force, random proposals, ping-pong, mismatches, bilateral, median and
    maskFov, stage by stage; every stage is bit-identical, so no re-synchronisation is needed."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    S = len(colors)
    ctxs = pair(oracle, ref, rig)
    oc = ctxs[0]
    oc.level_begin(W >> 1, H >> 1, level=2, num_levels=3, full_width=W, full_height=H)
    oc.set_colors(level_colors(name, 1))
    coarse = []
    for d in range(S):
        oc.reproject(d)
        oc.brute_force(d, num_depths=150, want_index=False)
        oc.mask_fov(d)
        coarse.append(oc.get_disparity(d, want_cost=False))
    both(ctxs, "level_begin", W, H, level=1, num_levels=3, full_width=W, full_height=H)
    both(ctxs, "set_colors", colors)
    for d in range(S):
        both(ctxs, "upsample_from", d, coarse[d])

    def check(what):
        for d in range(S):
            for o, r in zip(*both(ctxs, "get_disparity", d)):
                assert eq_bits(o, r), (what, d)

    check("upsampleDisparities (Lanczos4)")
    for d in range(S):
        both(ctxs, "reproject", d)
        both(ctxs, "random_proposals", d, 2)
        for o, r in zip(*both(ctxs, "get_disparity", d)):
            assert eq_bits(o, r), ("randomProposals", d)
        both(ctxs, "ping_pong", d, 2)
        for o, r in zip(*both(ctxs, "get_disparity", d)):
            assert eq_bits(o, r), ("pingPong", d)
    both(ctxs, "mismatches")
    check("handleDisparityMismatches")
    for d in range(S):
        o, r = both(ctxs, "get_mismatch_mask", d)
        assert eq_bits(o, r), ("mismatch mask", d)
    for stage in ("bilateral", "median", "mask_fov"):
        for d in range(S):
            both(ctxs, stage, d)
        check(stage)


@pytest.mark.parametrize("name", NAMES)
def test_process_level_two_levels(oracle, ref, name):
    """processLevel itself, two levels coarse to fine with mismatch handling on both, each library on its own."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    S = len(colors)
    ctxs = pair(oracle, ref, rig)
    prev = None
    for level in (1, 0):
        both(ctxs, "level_begin", W >> level, H >> level, level=level, num_levels=2, full_width=W, full_height=H)
        both(ctxs, "set_colors", level_colors(name, level))
        if prev is not None:
            for c, p in zip(ctxs, prev):
                for d in range(S):
                    c.upsample_from(d, p[d])
        both(ctxs, "process_level", num_depths=150, mismatches_start_level=0)
        prev = [[c.get_disparity(d, want_cost=False) for d in range(S)] for c in ctxs]
        for d in range(S):
            assert eq_bits(prev[0][d], prev[1][d]), (level, d)


@pytest.mark.parametrize("name", NAMES)
def test_standalone_upsample(oracle, ref, name):
    """upsampleDisparity (UpsampleDisparityLib.cpp) with the FOV masks of each camera type rescaled to the output size,
    plain and with foreground masks and background disparity."""
    for d, coarse, sizes, (W, H, bg, cmask, fmask) in cm.upsample_cases(name):
        for w, h in sizes:
            assert eq_bits(oracle.upsample_disparity(d, coarse, w, h), ref.upsample_disparity(d, coarse, w, h)), (w, h)
        assert eq_bits(oracle.upsample_disparity(d, coarse, W, H, bg, cmask, fmask, True),
                       ref.upsample_disparity(d, coarse, W, H, bg, cmask, fmask, True))
