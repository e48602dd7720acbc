"""Rigs of 33 to 64 cameras on the GPU: the 64-bit visibility-mask instantiation of every cost kernel against the
oracle, with the tolerance classes of tests/test_gpu_parity.py for the same stages.  Destinations are taken below and
above camera 32, so the destination's own bit and the contributing sources fall in both halves of the mask.  The wall
rigs see the scene's far points from most cameras: a far-only brute force averages more than 32 contributing sources
per cost, which only the selection slots past 32 and the high mask bits can hold."""
import functools
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests.parity_util import both, make_pair, mismatch_fraction, same_float_bits
from tests.test_apps import read_pfm, write_dataset

pytestmark = pytest.mark.gpu

BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")
HOST = os.path.join(capi.ROOT, "facebook360_dep_b200", "csrc", "host")

# name -> (rig maker, width, height, scene seed, destinations)
RIGS = {
    "wall40": (lambda w, h: synth.wall_rig(40, w, h), 64, 48, 7, (5, 36)),
    "wall64": (lambda w, h: synth.wall_rig(64, w, h), 64, 48, 7, (12, 50)),
    "ring48": (lambda w, h: synth.ring_rig(48, w, h, kind="FTHETA"), 80, 64, 12, (3, 40)),
}
WALLS = ["wall40", "wall64"]


@functools.lru_cache(maxsize=4)
def rig_inputs(name):
    make, W, H, seed, dsts = RIGS[name]
    rig = make(W, H)
    colors, true_disp = synth.render_rig(rig, W, H, scene=synth.Scene(seed=seed))
    return rig, colors, true_disp, W, H, dsts


def _begin(name, cuda, oracle, **kw):
    rig, colors, true_disp, W, H, dsts = rig_inputs(name)
    ctxs = make_pair(cuda, oracle, rig)
    both(ctxs, "level_begin", W, H, **kw)
    both(ctxs, "set_colors", colors)
    return ctxs, colors, true_disp, W, H, dsts


@pytest.mark.parametrize("name", list(RIGS))
def test_level_tables(cuda, oracle, name):
    ctxs, colors, _, W, H, dsts = _begin(name, cuda, oracle)
    S = len(colors)
    for d in range(S):
        g, o = both(ctxs, "get_fov_mask", d)
        assert np.array_equal(g, o)
    for s in range(S):
        g, o = both(ctxs, "get_variance", s)
        assert np.array_equal(g.view(np.uint32), o.view(np.uint32)), "variance must be bit-exact"
    for d in dsts:
        both(ctxs, "reproject", d)
        for s in range(S):
            gw, ow = both(ctxs, "get_proj_warp", s)
            # the wall's cameras are parallel: at infinity a source pixel maps to the same destination row, and the
            # coordinate is the fp64 cancellation residue of an exact 0 (~1e-15 px) whose sign and last bits are noise;
            # the mismatch class is counted on the coordinates above that, all of them are held to 1e-3 px below
            resolved = ~(np.abs(ow) < 1e-6)
            assert 1.0 - same_float_bits(gw, ow)[resolved].mean() <= 1e-5
            assert np.array_equal(np.isnan(gw), np.isnan(ow))
            fin = ~np.isnan(ow)
            assert np.abs(gw[fin] - ow[fin]).max(initial=0) <= 1e-3
            gc, oc = both(ctxs, "get_proj_color", s)
            assert (gc != oc).mean() <= 1e-5, "projColor"
            gb, ob = both(ctxs, "get_proj_bias", s)
            assert (gb != ob).mean() <= 2e-5, "projBias"


@pytest.mark.parametrize("name", list(RIGS))
def test_eval_cost(cuda, oracle, name):
    ctxs, _, true_disp, W, H, dsts = _begin(name, cuda, oracle)
    rng = np.random.RandomState(1)
    for d in dsts:
        both(ctxs, "reproject", d)
        for disp in (np.full((H, W), 0.31, np.float32), true_disp[d], rng.uniform(1e-4, 2.0, size=(H, W)).astype(np.float32)):
            (gc, gf), (oc, of) = both(ctxs, "eval_cost", d, disp)
            assert mismatch_fraction(gc, oc) <= 1e-5
            assert mismatch_fraction(gf, of) <= 1e-5
            assert ctxs[0].get_counters() == ctxs[1].get_counters()


def _brute_force_both_modes(ctxs, d, **kw):
    """Oracle brute force, then the CUDA one in plain (1) and filtered (2) mode: winners bit-exact against the oracle,
    the two modes equal bit for bit.  Returns the oracle's (evaluations, source hits) and whether the filtered mode
    completed on its bound list (when more candidates survive the bounds than the list holds it redoes the destination
    with the plain sweep, with the same result)."""
    oi = ctxs[1].brute_force(d, **kw)
    od, oc, of = ctxs[1].get_disparity(d)
    counters = ctxs[1].get_counters()
    out = []
    for mode in (1, 2):
        ctxs[0].set_sweep_mode(mode)
        gi = ctxs[0].brute_force(d, **kw)
        gd, gc, gf = ctxs[0].get_disparity(d)
        assert np.array_equal(gi, oi), (mode, int((gi != oi).sum()))
        assert same_float_bits(gd, od).all() and same_float_bits(gc, oc).all() and same_float_bits(gf, of).all()
        assert ctxs[0].get_counters() == counters, mode
        out.append((gi, gd, gc, gf))
    completed = ctxs[0].sweep_stats()[1] > 0
    ctxs[0].set_sweep_mode(0)
    for a, b in zip(*out):
        assert same_float_bits(a, b).all() if a.dtype == np.float32 else np.array_equal(a, b)
    return counters, completed


@pytest.mark.parametrize("name", list(RIGS))
def test_brute_force_both_sweep_modes(cuda, oracle, name):
    ctxs, _, _, W, H, dsts = _begin(name, cuda, oracle)
    completed = []
    for d in dsts:
        both(ctxs, "reproject", d)
        completed.append(_brute_force_both_modes(ctxs, d, num_depths=48)[1])
    if name == "ring48":
        # on the walls at this size more candidates survive the bounds than the list holds (D / 8 per pixel), so their
        # filtered mode ends in the plain sweep; the ring runs the whole filtered path (bound pass, seed, list, refine)
        # on its 64-bit kernels
        assert all(completed)


@pytest.mark.parametrize("name", WALLS)
def test_more_than_32_sources_per_cost(cuda, oracle, name):
    """Far candidates only: every camera of the wall sees nearly every point, so the average cost has more than 32
    contributing sources and the evaluations use selection slots past 32 and the mask's high word."""
    ctxs, _, _, W, H, dsts = _begin(name, cuda, oracle)
    for d in dsts:
        both(ctxs, "reproject", d)
        (ev, hits), _ = _brute_force_both_modes(ctxs, d, num_depths=40, min_depth_m=2.0)
        assert hits / ev > 32, (d, hits / ev)


@pytest.mark.parametrize("name", list(RIGS))
def test_fine_level_stages(cuda, oracle, name):
    ctxs, colors, true_disp, W, H, dsts = _begin(name, cuda, oracle, level=0, num_levels=2, full_width=None, full_height=None)
    S = len(colors)
    rng = np.random.RandomState(3)
    for d in range(S):
        start = np.clip(true_disp[d] * rng.uniform(0.85, 1.2, (H, W)).astype(np.float32), 1e-4, 2.0).astype(np.float32)
        both(ctxs, "set_disparity", d, start, np.zeros_like(start), np.zeros_like(start))
    for d in dsts:
        both(ctxs, "reproject", d)
        both(ctxs, "random_proposals", d, 2)
        (gd, gc, gf), (od, oc, of) = both(ctxs, "get_disparity", d)
        assert mismatch_fraction(gd, od) <= 2e-5, "random proposals disparity"
        assert mismatch_fraction(gc, oc) <= 2e-5 and mismatch_fraction(gf, of) <= 2e-5
        assert ctxs[0].get_counters() == ctxs[1].get_counters()
        ctxs[0].set_disparity(d, od, oc, of)  # re-synchronise before the next stage
        both(ctxs, "ping_pong", d, 2)
        (gd, gc, gf), (od, oc, of) = both(ctxs, "get_disparity", d)
        assert mismatch_fraction(gd, od) <= 2e-5, "ping-pong disparity"
        assert mismatch_fraction(gc, oc) <= 2e-5
        assert ctxs[0].get_counters() == ctxs[1].get_counters()
        ctxs[0].set_disparity(d, od, oc, of)
    both(ctxs, "mismatches")  # every camera's disparity, every camera's mask
    for d in range(S):
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert mismatch_fraction(gd, od) <= 2e-5
        gm, om = both(ctxs, "get_mismatch_mask", d)
        assert (gm != om).mean() <= 2e-5
        ctxs[0].set_disparity(d, od)
    for d in dsts:
        both(ctxs, "bilateral", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        fin = np.isfinite(od)
        assert np.array_equal(np.isfinite(gd), fin)
        assert (np.abs(gd - od)[fin] <= 2e-6 * np.abs(od)[fin] + 1e-12).all(), "bilateral"
        ctxs[0].set_disparity(d, od)
        both(ctxs, "median", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert same_float_bits(gd, od).all(), "median must be bit-exact"
        both(ctxs, "mask_fov", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert same_float_bits(gd, od).all()


@pytest.mark.parametrize("name", ["wall40", "ring48"])
def test_process_level_two_levels(cuda, oracle, name):
    """Coarse-to-fine over two levels with mismatch handling, each library on its own (no re-synchronisation):
    >= 99.9 % of pixels within 1e-3 relative, like the other end-to-end runs."""
    rig, colors, _, W, H, _ = rig_inputs(name)
    S = len(colors)
    pyr = [colors, [synth.downscale_area(c, 2) for c in colors]]
    ctxs = make_pair(cuda, oracle, rig)
    prev = None
    for level in (1, 0):
        both(ctxs, "level_begin", W >> level, H >> level, level=level, num_levels=2, full_width=W, full_height=H)
        both(ctxs, "set_colors", pyr[level])
        if prev is not None:
            for c, p in zip(ctxs, prev):
                for d in range(S):
                    c.upsample_from(d, p[d])
        both(ctxs, "process_level", num_depths=48, mismatches_start_level=0)
        prev = [[c.get_disparity(d, want_cost=False) for d in range(S)] for c in ctxs]
        good = tot = 0
        for d in range(S):
            g, o = prev[0][d], prev[1][d]
            assert np.array_equal(np.isnan(g), np.isnan(o))
            fin = ~np.isnan(o)
            good += int((np.abs(g - o)[fin] <= 1e-3 * np.abs(o)[fin]).sum())
            tot += int(fin.sum())
        assert good / tot >= 0.999, (level, good / tot)


def test_derpcli_40_cameras_end_to_end(tmp_path, cuda):
    """DerpCLI on a 40-camera rig, two levels: its PFMs equal the run of the same library through the Python binding."""
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    rig, colors, _, W, H, _ = rig_inputs("wall40")
    S = len(colors)
    inp, out = str(tmp_path / "in"), str(tmp_path / "out")
    write_dataset(inp, rig, [colors], 2)
    p = subprocess.run([os.path.join(BIN, "DerpCLI"), "--input_root=" + inp, "--output_root=" + out, "--partial_coverage=true",
                        "--num_depths=48", "--mismatches_start_level=0", "--gpus=1"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    ctx = capi.Context(cuda, capi.rig_descs(rig))
    ctx.level_begin(W // 2, H // 2, level=1, num_levels=2, full_width=W, full_height=H)
    ctx.set_colors([synth.downscale_area(c, 2) for c in colors])
    ctx.process_level(num_depths=48, mismatches_start_level=0)
    c1 = [ctx.get_disparity(d, want_cost=False) for d in range(S)]
    ctx.level_begin(W, H, level=0, num_levels=2, full_width=W, full_height=H)
    ctx.set_colors(colors)
    for d in range(S):
        ctx.upsample_from(d, c1[d])  # the app re-reads the coarser level from its PFM, which is lossless
    ctx.process_level(num_depths=48, mismatches_start_level=0)
    c0 = [ctx.get_disparity(d, want_cost=False) for d in range(S)]
    ctx.close()
    for L, disps in ((1, c1), (0, c0)):
        for d in range(S):
            got = read_pfm(os.path.join(out, "disparity_levels", "level_%d" % L, "cam%d" % d, "000000.pfm"))
            assert np.array_equal(got.view(np.uint32), disps[d].view(np.uint32)), (L, d)
