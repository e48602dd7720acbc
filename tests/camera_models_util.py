"""Rigs of every camera model and FOV cone the rig format allows, for the depth path and the canopy.

Each rig is a ring of 6 cameras (synth.ring_rig) whose type, focal, fov and distortion are then set per camera:

  name            type                          fov            focal (px at W = 64)   reaches
  equisolid       EQUISOLID                     none (-1)      W / 4                  rays past 90 deg, theta = pi at r > 2
  equisolid_cone  EQUISOLID                     1.4            W / 4                  positive general cone, image circle
  ortho           ORTHOGRAPHIC                  none (0)       W / 2                  "is behind" cone, r > 1 clamp
  ortho_cone      ORTHOGRAPHIC                  1.2            W / 2                  general cone
  fisheye_full    FTHETA, golden distortion     none (-1)      W / pi                 points behind sources, distMax clamp
  fisheye_wide    FTHETA, golden distortion     1.9 (cos < 0)  W / pi                 negative-cosine cone
  rect_cone       RECTILINEAR                   0.9            hfov 100 deg           rectilinear general cone
  mixed           FTHETA, RECTILINEAR, EQUISOLID, ORTHOGRAPHIC alternating, no fov    per-source type divergence

The odd-size variants (65 x 49) put the central pixel's ray exactly on the optical axis, the squaredNorm == 0 branch
of sensorToCamera.  "Golden distortion" is the one of the reference's 16-camera test rig (synth.sphere_rig), whose
distMax is about 1.9 rad.

check_coverage measures what each rig is for, so that the tests can assert a rig still reaches its branches."""
import functools
import math

import numpy as np

from facebook360_dep_b200 import capi, synth

GOLDEN_DISTORTION = [-0.03413328161902581, 0.0004374554953464843, -0.0018843963208481174]
NUM_CAMS = 6
DSTS = (0, 1, 2, 3)  # the destinations of the per-destination stages: every type of the mixed rig
SCENE_SEED = 42

# type -> (focal at width W, distortion)
_INTRINSICS = {
    "EQUISOLID": (lambda W: W / 4.0, None),
    "ORTHOGRAPHIC": (lambda W: W / 2.0, None),
    "FTHETA": (lambda W: W / math.pi, GOLDEN_DISTORTION),
    "RECTILINEAR": (lambda W: (W / 2.0) / math.tan(math.radians(100.0) / 2.0), None),
}
_MIXED = ["FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"]

# name -> (types of the cameras, fov or None, width, height, whether the cone excludes part of each sensor)
RIGS = {
    "equisolid": ("EQUISOLID", None, 64, 48, False),
    "equisolid_cone": ("EQUISOLID", 1.4, 64, 48, True),
    "ortho": ("ORTHOGRAPHIC", None, 64, 48, False),
    "ortho_cone": ("ORTHOGRAPHIC", 1.2, 64, 48, True),
    "fisheye_full": ("FTHETA", None, 64, 48, False),
    "fisheye_wide": ("FTHETA", 1.9, 64, 48, True),
    "rect_cone": ("RECTILINEAR", 0.9, 64, 48, True),
    "mixed": (_MIXED, None, 64, 48, False),
    "equisolid_odd": ("EQUISOLID", None, 65, 49, False),
    "ortho_odd": ("ORTHOGRAPHIC", None, 65, 49, False),
}

# name -> (least share of FOV pixels whose ray is more than 90 deg off the optical axis, least share of FOV pixels
# that get a brute-force winner): a little under what the rigs reach, so that a change to the builder that empties
# a branch fails instead of passing silently
MINIMA = {
    "equisolid": (0.40, 0.90),
    "equisolid_cone": (0.0, 0.90),
    "ortho": (0.0, 0.90),
    "ortho_cone": (0.0, 0.90),
    "fisheye_full": (0.15, 0.90),
    "fisheye_wide": (0.07, 0.90),
    "rect_cone": (0.0, 0.65),
    "mixed": (0.10, 0.90),
    "equisolid_odd": (0.40, 0.90),
    "ortho_odd": (0.0, 0.90),
}


def camera_types(name):
    types = RIGS[name][0]
    return [types] * NUM_CAMS if isinstance(types, str) else [types[i % len(types)] for i in range(NUM_CAMS)]


def make_rig(name):
    """The rig JSON dict of `name`."""
    _, fov, W, H, _ = RIGS[name]
    rig = synth.ring_rig(NUM_CAMS, W, H, kind="FTHETA")
    for cam, kind in zip(rig["cameras"], camera_types(name)):
        focal, dist = _INTRINSICS[kind]
        f = focal(W)
        cam["type"] = kind
        cam["focal"] = [f, -f]
        cam.pop("fov", None)
        cam.pop("distortion", None)
        if fov is not None:
            cam["fov"] = fov
        if dist is not None:
            cam["distortion"] = list(dist)
    return rig


@functools.lru_cache(maxsize=16)
def rig_inputs(name):
    """(rig, colours, true disparities, W, H) of `name`, rendered with synth.render_rig."""
    _, _, W, H, _ = RIGS[name]
    rig = make_rig(name)
    colors, true_disp = synth.render_rig(rig, W, H, scene=synth.Scene(seed=SCENE_SEED))
    return rig, colors, true_disp, W, H


def past_90_share(rig, fov_masks):
    """Share of FOV pixels, over all cameras, whose ray is more than 90 deg off its camera's optical axis."""
    past = tot = 0
    for cam, m in zip(rig["cameras"], fov_masks):
        H, W = m.shape
        _, _, theta = synth.pixel_rays(cam, W, H)
        inside = np.asarray(m) != 0
        past += int(((theta.numpy() > math.pi / 2) & inside).sum())
        tot += int(inside.sum())
    return past / max(1, tot)


def check_coverage(name, fov_masks, winners):
    """Asserts that `name` still reaches its branches and prints its coverage numbers.  `fov_masks` are every camera's
    FOV masks, `winners` {destination: brute-force winner indices}."""
    rig = rig_inputs(name)[0]
    fov_share = float(np.mean([np.mean(np.asarray(m) != 0) for m in fov_masks]))
    past = past_90_share(rig, fov_masks)
    won = sum(int(((winners[d] >= 0) & (fov_masks[d] != 0)).sum()) for d in winners)
    inside = sum(int((fov_masks[d] != 0).sum()) for d in winners)
    win_share = won / max(1, inside)
    print("%s coverage: rays past 90 deg %.1f %%, winners %.1f %%, FOV mask %.1f %%"
          % (name, 100 * past, 100 * win_share, 100 * fov_share))
    min_past, min_win = MINIMA[name]
    assert past >= min_past, (name, past)
    assert win_share >= min_win, (name, win_share)
    if RIGS[name][4]:
        assert fov_share < 1, name
    else:
        assert fov_share == 1, name


def upsample_cases(name):
    """(camera desc, coarse map, [(out w, out h)], masked-call inputs) for one camera of each type of the rig."""
    rig, _, _, W, H = rig_inputs(name)
    types = camera_types(name)
    rng = np.random.RandomState(2)
    cw, ch = W // 2, H // 2
    for i in sorted({types.index(t) for t in types}):
        d = capi.camera_desc_from_json(rig["cameras"][i])
        coarse = rng.uniform(1e-4, 2, (ch, cw)).astype(np.float32)
        coarse[3:6, 7:9] = np.nan
        sizes = ((W, H), (W + 7, H + 5), (cw, ch))
        cmask = (rng.uniform(size=(ch, cw)) > 0.3).astype(np.uint8)
        fmask = (rng.uniform(size=(H, W)) > 0.2).astype(np.uint8)
        bg = rng.uniform(0.01, 0.02, (H, W)).astype(np.float32)
        yield d, coarse, sizes, (W, H, bg, cmask, fmask)
