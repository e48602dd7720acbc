"""Every camera model and FOV cone of the rig format on the GPU: the kernels that build rays, test cones and project
points, against the oracle on the rigs of tests/camera_models_util.py (EQUISOLID, ORTHOGRAPHIC, FTHETA seeing behind
itself or through a cone wider than 180 deg, RECTILINEAR with a cone, the four types mixed in one rig, and odd sensors
whose central ray is the optical axis).  tests/test_camera_models.py pins the oracle to the reference on the same rigs.

The tolerance classes are those of tests/test_gpu_parity.py, unchanged: level tables with FOV masks and variance
bit-exact, warps <= 1e-5 mismatching with the same NaN pattern and |delta| <= 1e-3 px, projected colour <= 1e-5 and
bias <= 2e-5 mismatching; computeCost <= 1e-5 mismatching with equal work counters; brute force in both sweep modes
bit-exact; the fine-level stages re-synchronised between stages, proposals, ping-pong and mismatches <= 2e-5,
bilateral within 2e-6 relative, median and maskFov bit-exact; three levels of processLevel, each library on its own,
>= 99.9 % of pixels within 1e-3 relative; upsampleDisparity bit-exact.  The canopy of ComputeRephotographyErrors
(rephotoPrepKernel: pixelRay and the image circle per vertex) is compared with tests/rephoto_oracle.cpp: winners
bit-exact, disparity colour by check_disparity_colour, colour bit-exact on rigs without ORTHOGRAPHIC cameras.

One tolerance class is new, for the colour and disparity colour of canopies of ORTHOGRAPHIC cameras (a vertex and a
disparity texel both narrow the fp64 point pos + ray * distance to fp32).  Their pixel ray is
sin(asin(r)) / r * (sx, sy) and -cos(asin(r)): the sensor-plane components come out within an fp64 ulp of sx and sy,
which are dyadic ((x + 0.5 - cx) / f), so a vertex pos + ray * fp32 distance lies within an fp64 ulp of an fp32
rounding tie far more often than a generic value does.  libdevice's asin differs from glibc's by one ulp on about a
third of the arguments of these rigs (sin and cos follow; measured on an H100 with CUDA 12.9 and glibc 2.39), and a
one-ulp change of theta flips the fp32 rounding of about 7 % of the ORTHOGRAPHIC vertices of a camera with an
axis-aligned rotation, none of the EQUISOLID ones.  A moved vertex moves the barycentric weights and texture
coordinates of its fragments by an fp32 ulp, so the colour changes far below one RGBA16 step (1 / 65535), while a
wrong winner, texel or mip level changes it by many steps; a disparity texel rounds 1 / |point - centre| to the
nearest step, so a moved point changes it by at most one step.  Measured: at most 0.5 % of a cubemap's pixels differ
in colour, by at most 9e-7.  Required: winners and coverage bit-exact; at most 1 % of colour values differing and
none by a full step; at most 1 % of disparity-colour values differing, none by more than one step.  The depth path's
tables of the same cameras are within their existing class."""
import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import camera_models_util as cm
from tests import rephoto_oracle
from tests.parity_util import both, make_pair, mismatch_fraction, same_float_bits
from tests.test_gpu_filtered_sweep_edges import aligned_constant, binary, check_bounds
from tests.test_gpu_rephoto import STEP, _bgra, _views, check_disparity_colour
from tests.test_gpu_wide_rig import _brute_force_both_modes

pytestmark = pytest.mark.gpu

NAMES = list(cm.RIGS)


def _begin(name, cuda, oracle, **kw):
    rig, colors, true_disp, W, H = cm.rig_inputs(name)
    ctxs = make_pair(cuda, oracle, rig)
    both(ctxs, "level_begin", W, H, **kw)
    both(ctxs, "set_colors", colors)
    return ctxs, colors, true_disp, W, H


def _pyramid(name, levels):
    """Colours of each level, the scene rendered at that size (the odd sensors do not halve exactly)."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    return [colors] + [synth.render_rig(rig, W >> L, H >> L, scene=synth.Scene(seed=cm.SCENE_SEED))[0]
                       for L in range(1, levels)]


@pytest.mark.parametrize("name", NAMES)
def test_level_tables(cuda, oracle, name):
    ctxs, colors, _, W, H = _begin(name, cuda, oracle)
    S = len(colors)
    for d in range(S):
        g, o = both(ctxs, "get_fov_mask", d)
        assert np.array_equal(g, o), ("fov mask", d)
    for s in range(S):
        g, o = both(ctxs, "get_variance", s)
        assert np.array_equal(g.view(np.uint32), o.view(np.uint32)), "variance must be bit-exact"
    for d in cm.DSTS:
        both(ctxs, "reproject", d)
        for s in range(S):
            gw, ow = both(ctxs, "get_proj_warp", s)
            assert mismatch_fraction(gw, ow) <= 1e-5, (d, s)
            assert np.array_equal(np.isnan(gw), np.isnan(ow)), (d, s)
            fin = ~np.isnan(ow)
            assert np.abs(gw[fin] - ow[fin]).max(initial=0) <= 1e-3, (d, s)
            gc, oc = both(ctxs, "get_proj_color", s)
            assert (gc != oc).mean() <= 1e-5, ("projColor", d, s)
            gb, ob = both(ctxs, "get_proj_bias", s)
            assert (gb != ob).mean() <= 2e-5, ("projBias", d, s)


@pytest.mark.parametrize("name", NAMES)
def test_eval_cost(cuda, oracle, name):
    ctxs, _, true_disp, W, H = _begin(name, cuda, oracle)
    rng = np.random.RandomState(1)
    for d in cm.DSTS:
        both(ctxs, "reproject", d)
        for disp in (np.full((H, W), 0.31, np.float32), true_disp[d], rng.uniform(1e-4, 2.0, (H, W)).astype(np.float32)):
            (gc, gf), (oc, of) = both(ctxs, "eval_cost", d, disp)
            assert mismatch_fraction(gc, oc) <= 1e-5, d
            assert mismatch_fraction(gf, of) <= 1e-5, d
            assert ctxs[0].get_counters() == ctxs[1].get_counters(), d


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("num_depths", [48, 150])
def test_brute_force_both_sweep_modes(cuda, oracle, name, num_depths):
    """Plain (1) and filtered (2) sweep: winners, disparity, cost, confidence and counters bit for bit against the
    oracle; the rig's coverage numbers are printed and asserted on the oracle's winners."""
    ctxs, colors, _, W, H = _begin(name, cuda, oracle)
    masks = [ctxs[1].get_fov_mask(d) for d in range(len(colors))]
    winners = {}
    for d in cm.DSTS:
        both(ctxs, "reproject", d)
        _brute_force_both_modes(ctxs, d, num_depths=num_depths)
        winners[d] = ctxs[1].brute_force(d, num_depths=num_depths)
    cm.check_coverage(name, masks, winners)


def _fit(imgs, W, H):
    """64 x 48 content of tests/test_gpu_filtered_sweep_edges.py tiled to W x H (its periods divide 64 and 48)."""
    return [np.ascontiguousarray(np.pad(c, ((0, H - c.shape[0]), (0, W - c.shape[1]), (0, 0)), mode="wrap")) for c in imgs]


@pytest.mark.parametrize("name", NAMES)
def test_lower_bound_never_exceeds_cost(cuda, name):
    """derp_debug_lower_bound: no bound of the filtered sweep exceeds the exact cost, on the rendered scene, on aligned
    constant content and on a 2-px checkerboard."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    S = len(colors)
    ctx = capi.Context(cuda, capi.rig_descs(rig))
    ctx.level_begin(W, H)
    for content in ("rendered", "const_mid", "checker2"):
        for d in cm.DSTS:
            if content == "rendered":
                ctx.set_colors(colors)
            elif content == "const_mid":
                ctx.set_colors(_fit(aligned_constant(S, d, 40000, 32768), W, H))
            else:
                ctx.set_colors(_fit(binary(S, "checker2"), W, H))
            ctx.reproject(d)
            check_bounds(cuda, ctx, "%s/%s" % (name, content), d)
    ctx.close()


@pytest.mark.parametrize("name", NAMES)
def test_fine_level_stages(cuda, oracle, name):
    ctxs, colors, true_disp, W, H = _begin(name, cuda, oracle, level=0, num_levels=2)
    S = len(colors)
    rng = np.random.RandomState(3)
    for d in range(S):
        start = np.clip(true_disp[d] * rng.uniform(0.85, 1.2, (H, W)).astype(np.float32), 1e-4, 2.0).astype(np.float32)
        both(ctxs, "set_disparity", d, start, np.zeros_like(start), np.zeros_like(start))
    for d in range(S):
        both(ctxs, "reproject", d)
        both(ctxs, "random_proposals", d, 2)
        (gd, gc, gf), (od, oc, of) = both(ctxs, "get_disparity", d)
        assert mismatch_fraction(gd, od) <= 2e-5, ("random proposals disparity", d)
        assert mismatch_fraction(gc, oc) <= 2e-5 and mismatch_fraction(gf, of) <= 2e-5, d
        assert ctxs[0].get_counters() == ctxs[1].get_counters(), d
        ctxs[0].set_disparity(d, od, oc, of)  # re-synchronise before the next stage
        both(ctxs, "ping_pong", d, 2)
        (gd, gc, gf), (od, oc, of) = both(ctxs, "get_disparity", d)
        assert mismatch_fraction(gd, od) <= 2e-5, ("ping-pong disparity", d)
        assert mismatch_fraction(gc, oc) <= 2e-5, d
        assert ctxs[0].get_counters() == ctxs[1].get_counters(), d
        ctxs[0].set_disparity(d, od, oc, of)
    both(ctxs, "mismatches")
    for d in range(S):
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert mismatch_fraction(gd, od) <= 2e-5, ("mismatches", d)
        gm, om = both(ctxs, "get_mismatch_mask", d)
        assert (gm != om).mean() <= 2e-5, d
        ctxs[0].set_disparity(d, od)
    for d in range(S):
        both(ctxs, "bilateral", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        fin = np.isfinite(od)
        assert np.array_equal(np.isfinite(gd), fin), d
        assert (np.abs(gd - od)[fin] <= 2e-6 * np.abs(od)[fin] + 1e-12).all(), ("bilateral", d)
        ctxs[0].set_disparity(d, od)
        both(ctxs, "median", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert same_float_bits(gd, od).all(), ("median must be bit-exact", d)
        both(ctxs, "mask_fov", d)
        gd, od = both(ctxs, "get_disparity", d, want_cost=False)
        assert same_float_bits(gd, od).all(), ("maskFov", d)


@pytest.mark.parametrize("name", NAMES)
def test_process_level_three_levels(cuda, oracle, name):
    """Coarse to fine over three levels with mismatch handling, each library on its own (no re-synchronisation): the
    fine-level FOV masks of the upsampling and every stage in between."""
    rig, colors, _, W, H = cm.rig_inputs(name)
    S = len(colors)
    pyr = _pyramid(name, 3)
    ctxs = make_pair(cuda, oracle, rig)
    prev = None
    for level in (2, 1, 0):
        both(ctxs, "level_begin", W >> level, H >> level, level=level, num_levels=3, full_width=W, full_height=H)
        both(ctxs, "set_colors", pyr[level])
        if prev is not None:
            for c, p in zip(ctxs, prev):
                for d in range(S):
                    c.upsample_from(d, p[d])
        both(ctxs, "process_level", num_depths=48, mismatches_start_level=1)
        prev = [[c.get_disparity(d, want_cost=False) for d in range(S)] for c in ctxs]
        good = tot = 0
        for d in range(S):
            g, o = prev[0][d], prev[1][d]
            assert np.array_equal(np.isnan(g), np.isnan(o)), (level, d)
            fin = ~np.isnan(o)
            good += int((np.abs(g - o)[fin] <= 1e-3 * np.abs(o)[fin]).sum())
            tot += int(fin.sum())
        assert good / tot >= 0.999, (level, good / tot)


@pytest.mark.parametrize("name", NAMES)
def test_standalone_upsample(cuda, oracle, name):
    for d, coarse, sizes, (W, H, bg, cmask, fmask) in cm.upsample_cases(name):
        for w, h in sizes:
            g = cuda.upsample_disparity(d, coarse, w, h)
            o = oracle.upsample_disparity(d, coarse, w, h)
            assert same_float_bits(g, o).all(), (d.type, w, h)
        g = cuda.upsample_disparity(d, coarse, W, H, bg, cmask, fmask, True)
        o = oracle.upsample_disparity(d, coarse, W, H, bg, cmask, fmask, True)
        assert same_float_bits(g, o).all(), d.type


@pytest.fixture(scope="module")
def rcuda():
    return capi.Rephoto(capi.load_cuda())


@pytest.fixture(scope="module")
def roracle():
    return rephoto_oracle.load()


def check_colour(g, o, what, exact):
    """Colour cubemap, GPU against checker: bit-exact, or (canopies of ORTHOGRAPHIC cameras, see the module docstring)
    at most 1 % of values differing and none by a full RGBA16 step."""
    assert np.array_equal(g[..., 3] > 0, o[..., 3] > 0), what
    diff = np.abs(g - o)
    count, err = int((diff > 0).sum()), float(diff.max())
    print(what, "colour: %d of %d values differ, max |cuda - oracle| %.3g" % (count, diff.size, err))
    if exact:
        assert count == 0, (what, count, err)
    else:
        assert count <= 0.01 * diff.size and err < 1 / 65535, (what, count, err)


def check_disparity(g, o, what, exact):
    """Disparity cubemap: check_disparity_colour, or (canopies of ORTHOGRAPHIC cameras) the same NaN pattern, at most
    1 % of values differing and none by more than one RGBA16 step."""
    assert np.array_equal(g[..., 3] > 0, o[..., 3] > 0), what
    if exact:
        check_disparity_colour(g, o, what)
        return
    nan = np.isnan(o)
    assert np.array_equal(np.isnan(g), nan), what
    diff = np.abs(g - o)[~nan]
    count, err = int((diff > 0).sum()), float(diff.max()) if diff.size else 0.0
    print(what, "disparity colour: %d of %d values differ, max |cuda - oracle| %.3g" % (count, diff.size, err))
    assert count <= 0.01 * diff.size and err <= STEP, (what, count, err)


@pytest.mark.parametrize("name", ["equisolid", "fisheye_full", "ortho", "mixed"])
def test_rephoto_cubemaps(rcuda, roracle, name):
    """The canopies of ComputeRephotographyErrors: each camera's own and the other cameras', rendered to a cubemap at
    the camera's centre.  Winners bit for bit; colour bit for bit unless a canopy of an ORTHOGRAPHIC camera is drawn;
    disparity colour by check_disparity_colour."""
    rig, colors, true_disp, W, H = cm.rig_inputs(name)
    types = cm.camera_types(name)
    bgra = [_bgra(c) for c in colors]
    for i in cm.DSTS:
        (gc, gd, gw), (rc, rd, rw) = _views(rcuda, rig, true_disp, bgra, i)
        (oc, od, ow), (qc, qd, qw) = _views(roracle, rig, true_disp, bgra, i)
        assert np.array_equal(gw, ow) and np.array_equal(rw, qw), (name, i, int((gw != ow).sum()), int((rw != qw).sum()))
        assert (rw >= 0).any(axis=0).mean() > 0.1, (name, i)
        others = [t for j, t in enumerate(types) if j != i]
        check_colour(gc, oc, (name, i, "own"), types[i] != "ORTHOGRAPHIC")
        check_colour(rc, qc, (name, i, "others"), "ORTHOGRAPHIC" not in others)
        check_disparity(gd, od, (name, i, "own"), types[i] != "ORTHOGRAPHIC")
        check_disparity(rd, qd, (name, i, "others"), "ORTHOGRAPHIC" not in others)
