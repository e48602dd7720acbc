"""Rephotography on the GPU: derp_rephoto_cubemap / derp_rephoto_score against the CPU oracle, the score's ordering over
disparity maps of known quality, and ComputeRephotographyErrors end to end after DerpCLI.  Everything is seeded."""
import json
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import rephoto_oracle

pytestmark = pytest.mark.gpu
BIN = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin")


@pytest.fixture(scope="module")
def rcuda():
    """include/derp_rephoto.h on the product library (no fallback: a missing library or symbol fails)."""
    return capi.Rephoto(capi.load_cuda())


@pytest.fixture(scope="module")
def roracle():
    return rephoto_oracle.load()


def _bgra(img_u16):
    h, w = img_u16.shape[:2]
    return np.concatenate([img_u16.astype(np.float32) * np.float32(1 / 65535), np.ones((h, w, 1), np.float32)], -1)


def _scene(rig, W):
    colors, disps = synth.render_rig(rig, W, W, scene=synth.Scene(seed=11))
    return [_bgra(c) for c in colors], disps


def _views(lib, rig, disps, bgra, i):
    """(reference, rendered) colour cubemaps and winners of camera i, as ComputeRephotographyErrors forms them."""
    cams = rig["cameras"]
    ctr = np.array(cams[i]["origin"], np.float32)
    others = [j for j in range(len(cams)) if j != i]
    W = disps[0].shape[0]
    ref = lib.rephoto_cubemap(capi.rig_descs({"cameras": [cams[i]]}), [disps[i]], [bgra[i]], ctr, W,
                              want_disparity=True, want_winners=True)
    ren = lib.rephoto_cubemap(capi.rig_descs({"cameras": [cams[j] for j in others]}), [disps[j] for j in others],
                              [bgra[j] for j in others], ctr, W, want_disparity=True, want_winners=True)
    return ref, ren


STEP = 1 / 65535 + 1e-6  # one RGBA16 step


def check_disparity_colour(g, o, what):
    """Disparity colour, GPU against checker.  Its texel 1 / |world - centre| starts from the fp64 camera ray, whose
    sin / cos / atan may differ by an ulp between libdevice and glibc.  Both sides round the distance to fp32 first
    (DisparityColor.h: float distance = 1.0 / disparity), which absorbs such an ulp except at an fp32 rounding
    boundary, so a texel lands one RGBA16 step apart only rarely.  The blend is a convex combination of texels, so a
    value can differ by at most that step.  Requires NaN at the same places, at most a few differing values in 10^6 and
    none by more than one step."""
    nan = np.isnan(o)
    assert np.array_equal(np.isnan(g), nan), what
    diff = np.abs(g - o)[~nan]
    count, err = int((diff > 0).sum()), float(diff.max()) if diff.size else 0.0
    print(what, "disparity colour: %d of %d values differ, max |cuda - oracle| %.3g" % (count, diff.size, err))
    assert count <= 3e-6 * diff.size, (what, count, diff.size)
    assert err <= STEP, (what, err)


def _score(lib, ref, ren, method="MSSIM", radius=1):
    mask = (ref[0][..., 3] > 0).astype(np.uint8)
    return lib.rephoto_score(ref[0][..., :3], ren[0][..., :3], mask, method, radius)


@pytest.mark.parametrize("case", ["ring16_128", "ring16_512", "wall8_rect_256"])
def test_cubemaps_and_scores_match_oracle(rcuda, roracle, case):
    if case.startswith("ring"):
        W = int(case.split("_")[1])
        rig = synth.ring_rig(16, W, W, kind="FTHETA")
        cams = (0, 5) if W == 128 else (3,)
    else:
        W = 256
        rig = synth.wall_rig(8, W, W, kind="RECTILINEAR")
        cams = (2,)
    bgra, disps = _scene(rig, W)
    for i in cams:
        (gc, gd, gw), (rc, rd, rw) = _views(rcuda, rig, disps, bgra, i)
        (oc, od, ow), (qc, qd, qw) = _views(roracle, rig, disps, bgra, i)
        # coverage and every canopy's surviving primitive: same rules, same fp32/fp64 arithmetic -> bit for bit
        assert np.array_equal(gw, ow) and np.array_equal(rw, qw), (case, i, int((gw != ow).sum()), int((rw != qw).sum()))
        assert (rw >= 0).any(axis=0).mean() > (0.5 if case.startswith("ring") else 0.1)
        for g, o in ((gc, oc), (rc, qc)):
            # colour: the same RGBA16 texels, weights and fp32 sums -> the same bits
            assert np.array_equal(g[..., 3] > 0, o[..., 3] > 0)
            assert np.array_equal(g, o), (case, i, float(np.abs(g - o).max()))
        for g, o in ((gd, od), (rd, qd)):
            assert np.array_equal(g[..., 3] > 0, o[..., 3] > 0)
            check_disparity_colour(g, o, (case, i))
        for method in ("MSSIM", "NCC"):
            for radius in (1, 2):
                sg, ag = _score(rcuda, (gc,), (rc,), method, radius)
                so, ao = _score(roracle, (gc,), (rc,), method, radius)  # same inputs: the score alone
                assert np.array_equal(np.isnan(sg), np.isnan(so))
                fin = ~np.isnan(so)
                assert np.abs(sg - so)[fin].max() <= 1e-6
                assert np.abs(ag - ao).max() <= 1e-6, (ag, ao)


def _derpcli_disparities(tmp_path, rig, colors, W):
    """DerpCLI over a 3-level pyramid of the frame; returns the finest level's disparities and the output root."""
    inp, out = str(tmp_path / "in"), str(tmp_path / "out")
    os.makedirs(os.path.join(inp, "rigs"), exist_ok=True)
    json.dump(rig, open(os.path.join(inp, "rigs", "rig_calibrated.json"), "w"))
    for L in range(3):
        for cam, img in zip(rig["cameras"], colors):
            d = os.path.join(inp, "video", "color_levels", "level_%d" % L, cam["id"])
            os.makedirs(d, exist_ok=True)
            assert cv2.imwrite(os.path.join(d, "000000.png"), img if L == 0 else synth.downscale_area(img, 1 << L))
    subprocess.run([os.path.join(BIN, "DerpCLI"), "--input_root=" + inp, "--output_root=" + out, "--first=000000",
                    "--last=000000", "--partial_coverage=true", "--num_depths=64", "--gpus=1"], check=True,
                   capture_output=True)
    lvl0 = os.path.join(out, "disparity_levels", "level_0")
    disps = []
    for cam in rig["cameras"]:
        with open(os.path.join(lvl0, cam["id"], "000000.pfm"), "rb") as f:
            f.readline()
            w, h = map(int, f.readline().split())
            f.readline()
            disps.append(np.frombuffer(f.read(), np.float32).reshape(h, w).copy())
    return inp, lvl0, disps


def test_score_orders_disparity_quality_and_app_end_to_end(rcuda, tmp_path):
    """Ground truth scores higher than DerpCLI's estimate, which scores higher than a constant disparity; then the app
    on DerpCLI's output writes the log line the reference's test parses and the 5-panel plot."""
    W, S = 128, 8
    rig = synth.ring_rig(S, W, W, kind="FTHETA")
    colors, gt = synth.render_rig(rig, W, W, scene=synth.Scene(seed=5))
    bgra = [_bgra(c) for c in colors]
    inp, lvl0, est = _derpcli_disparities(tmp_path, rig, colors, W)
    const = [np.full((W, W), 1 / 3.0, np.float32) for _ in range(S)]
    means = {}
    for name, disps in (("ground_truth", gt), ("derpcli", est), ("constant", const)):
        s = [_score(rcuda, *_views(rcuda, rig, disps, bgra, i))[1] for i in range(S)]
        means[name] = float(np.mean(s))
    print("rephotography MSSIM, 8-camera FTHETA ring at 128^2:", json.dumps(means))
    assert means["ground_truth"] > means["derpcli"] > means["constant"], means
    out = str(tmp_path / "rephoto_out")
    logs = str(tmp_path / "logs")
    os.makedirs(logs)
    subprocess.run([os.path.join(BIN, "ComputeRephotographyErrors"), "--rig=" + inp + "/rigs/rig_calibrated.json",
                    "--color=" + inp + "/video/color_levels/level_0", "--disparity=" + lvl0, "--output=" + out,
                    "--first=000000", "--last=000000", "--log_dir=" + logs], check=True, capture_output=True)
    # scripts/test/test_derp_cli.py: the last line of <log_dir>/ComputeRephotographyErrors.INFO
    lines = open(os.path.join(logs, "ComputeRephotographyErrors.INFO")).read().strip().split("\n")
    m = re.search(r"TOTAL average MSSIM: R (\S+)%, G (\S+)%, B (\S+)%", lines[-1])
    assert m, lines[-1]
    total = np.mean([float(v) for v in m.groups()])
    assert abs(total / 100 - means["derpcli"]) < 1e-3, (total, means)
    plot = cv2.imread(os.path.join(out, "rephoto", "cam3", "000000.png"), cv2.IMREAD_UNCHANGED)
    assert plot is not None and plot.shape == (6 * W, 5 * W, 3) and plot.dtype == np.uint8
