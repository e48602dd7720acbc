"""RigSimulator on the GPU (include/derp_rigsim.h) against the checker, the reference's own RigSimulator.cpp compiled by
oracle/rigsim.mk: 0 differing bits in the fp32 colour and depth planes of every render, and the share of rays whose sky
texel the host resolved."""
import ctypes as C
import math

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import rigsim_util as ru
from tests import sweep_util as su

pytestmark = pytest.mark.gpu

SCENES = ["icosahedron", "cube", "ground_plane"]
_LIBM = C.CDLL("libm.so.6")
_LIBM.sinf.restype = _LIBM.cosf.restype = C.c_float
_LIBM.sinf.argtypes = _LIBM.cosf.argtypes = [C.c_float]


@pytest.fixture(scope="module")
def sim():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return capi.RigSim(capi.load_cuda())


@pytest.fixture(scope="module")
def ref():
    r = ru.load_ref()
    if r is None:
        pytest.skip("the RigSimulator checker (oracle/rigsim.mk) is not built")
    return r


def _share(sim, label):
    host, rays = sim.last_host_rays()
    print("%s: %d of %d rays resolved on the host (%.4f %%)" % (label, host, rays, 100.0 * host / max(rays, 1)))
    assert host <= 0.01 * rays
    return host, rays


def _scenes(sim, ref, scene, seed=3, **kw):
    ref.build(scene, seed=seed, **kw)
    sim.srand(seed)
    return sim.scene(scene, **kw)


def _assert_same(a, b, what):
    diff = int((ru.bits(a) != ru.bits(b)).sum())
    assert diff == 0, "%s: %d differing words" % (what, diff)


def _rig(kind):
    if kind == "pinhole_ring":
        return ru.ring_descs(5, 40, 36, kind="RECTILINEAR")
    if kind == "ftheta_ring":
        return ru.ring_descs(3, 36, 30)
    if kind == "golden_small":  # rig_from_json on the reference's 16-camera test rig at 84 x 54
        descs = su.rig("golden", 16, 0, 0, scale=1 / 40)
        for d in descs:
            d.resolution[0], d.resolution[1] = round(d.resolution[0]), round(d.resolution[1])
        return descs
    raise ValueError(kind)


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("kind", ["pinhole_ring", "ftheta_ring"])
@pytest.mark.parametrize("aas", [1, 2, 3])
def test_cameras_match_reference(sim, ref, scene, kind, aas):
    h = _scenes(sim, ref, scene)
    sky = ru.skybox(96, 48, seed=aas)
    descs = _rig(kind)
    ref.set_render(sky, aas=aas)
    got = sim.render_cameras(h, descs, sky, aas=aas)
    _share(sim, "%s %s aas %d" % (scene, kind, aas))
    for i, d in enumerate(descs):
        img, dep = ref.render_camera(d)
        _assert_same(got[i][0], img, "camera %d colour" % i)
        _assert_same(got[i][1], dep, "camera %d depth" % i)
    sim.destroy(h)


@pytest.mark.parametrize("aas", [1, 2])
def test_golden_rig_and_marble_match_reference(sim, ref, aas):
    h = _scenes(sim, ref, "icosahedron", seed=11, red_triangle=True, min_icosahedron_dist=20.0,
                max_icosahedron_dist=60.0, min_icosahedron_radius=2.0, max_icosahedron_radius=8.0)
    sky = ru.skybox(128, 64, seed=5)
    descs = _rig("golden_small")
    ref.set_render(sky, aas=aas, marble=True, marble_scale=0.37)
    got = sim.render_cameras(h, descs, sky, aas=aas, marble=True, marble_scale=0.37)
    _share(sim, "golden rig marble aas %d" % aas)
    for i, d in enumerate(descs):
        img, dep = ref.render_camera(d)
        _assert_same(got[i][0], img, "camera %d colour" % i)
        _assert_same(got[i][1], dep, "camera %d depth" % i)
    sim.destroy(h)


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("stereo", [False, True])
@pytest.mark.parametrize("aas", [1, 2, 3])
def test_equirects_match_reference(sim, ref, scene, stereo, aas):
    h = _scenes(sim, ref, scene, seed=aas)
    sky = ru.skybox(80, 40, seed=7)
    ref.set_render(sky, aas=aas, interpupillary_radius=3.2)
    a, b = sim.render_equirect(h, 48, 24, sky, stereo=stereo, aas=aas)
    _share(sim, "%s %s aas %d" % (scene, "stereo" if stereo else "mono", aas))
    ra, rb = ref.render_equirect(48, 24, stereo=stereo)
    _assert_same(a, ra, "first plane")
    _assert_same(b, rb, "second plane")
    sim.destroy(h)


def test_scene_without_triangles_matches_reference(sim, ref):
    """--num_random_icosahedrons 0: the BVH is one empty leaf with a NaN centre, every ray sees the sky."""
    h = _scenes(sim, ref, "icosahedron", seed=1, num_random_icosahedrons=0)
    sky = ru.skybox(64, 32, seed=3)
    ref.set_render(sky, aas=2)
    descs = ru.ring_descs(2, 32, 24)
    got = sim.render_cameras(h, descs, sky, aas=2)
    for i, d in enumerate(descs):
        img, dep = ref.render_camera(d)
        _assert_same(got[i][0], img, "colour")
        _assert_same(got[i][1], dep, "depth")
    a, b = sim.render_equirect(h, 32, 16, sky, aas=2)
    ra, rb = ref.render_equirect(32, 16)
    _assert_same(a, ra, "equirect colour")
    _assert_same(b, rb, "equirect 1 / depth")
    sim.destroy(h)


def test_device_resident_outputs(sim, ref):
    import torch
    h = _scenes(sim, ref, "icosahedron", seed=2)
    sky = ru.skybox(64, 32, seed=2)
    descs = ru.ring_descs(2, 32, 24)
    ref.set_render(sky, aas=2)
    bgr = [torch.empty((24, 32, 3), dtype=torch.float32, device="cuda") for _ in descs]
    dep = [torch.empty((24, 32), dtype=torch.float32, device="cuda") for _ in descs]
    sim.render_cameras(h, descs, sky, outs=([t.data_ptr() for t in bgr], [t.data_ptr() for t in dep]), aas=2)
    torch.cuda.synchronize()
    for i, d in enumerate(descs):
        img, depth = ref.render_camera(d)
        _assert_same(bgr[i].cpu().numpy(), img, "colour")
        _assert_same(dep[i].cpu().numpy(), depth, "depth")
    sim.destroy(h)


def _mono_rays(W, H, xs, ys):
    """renderMonoEquirect's fp32 rays at supersamples (xs, ys) of a W x H plane, with the C library's sinf / cosf."""
    rays = np.zeros((len(xs), 6), np.float32)
    for k, (x, y) in enumerate(zip(xs, ys)):
        theta = float(np.float32(2.0 * math.pi * float(np.float32(1.0) - np.float32(x + np.float32(0.5)) / np.float32(W))))
        phi = float(np.float32(math.pi * float(np.float32(y + np.float32(0.5))) / float(np.float32(H))))
        sp, cp, st, ct = _LIBM.sinf(phi), _LIBM.cosf(phi), _LIBM.sinf(theta), _LIBM.cosf(theta)
        rays[k, 3:] = [np.float32(sp) * np.float32(ct), np.float32(sp) * np.float32(st), cp]
    return rays


def test_full_size_mono_equirect_by_sampled_rays(sim, ref):
    """The default mono_eqr (3080 x 1540, default icosahedron scene) against traceRayToGetColor on 4000 sampled rays."""
    h = _scenes(sim, ref, "icosahedron", seed=1)
    sky = ru.skybox(1024, 512, seed=9)
    ref.set_render(sky)
    img, inv = sim.render_equirect(h, 3080, 1540, sky)
    _share(sim, "mono_eqr 3080 x 1540")
    rng = np.random.default_rng(4)
    xs, ys = rng.integers(0, 3080, 4000), rng.integers(0, 1540, 4000)
    want = ref.trace(_mono_rays(3080, 1540, xs, ys))
    _assert_same(img[ys, xs], np.float32(255.0) * want[:, :3], "colour")
    _assert_same(inv[ys, xs], np.clip(np.float32(1.0) / want[:, 3], np.float32(0), np.float32(1)), "1 / depth")
    sim.destroy(h)


def test_full_size_camera_matches_reference(sim, ref):
    """A 2048 x 2048 FTHETA camera of the 16-camera ring, the whole image through the checker."""
    h = _scenes(sim, ref, "icosahedron", seed=1)
    sky = ru.skybox(1024, 512, seed=10)
    d = ru.ring_descs(16, 2048, 2048)[3]
    ref.set_render(sky)
    got = sim.render_cameras(h, [d], sky)
    _share(sim, "FTHETA 2048 x 2048")
    img, dep = ref.render_camera(d)
    _assert_same(got[0][0], img, "colour")
    _assert_same(got[0][1], dep, "depth")
    sim.destroy(h)


@pytest.mark.parametrize("stereo", [False, True])
def test_ceiling_matches_reference(sim, ref, stereo):
    """Equirects and cameras with the ceiling on (and marble), against the reference's own ceiling code."""
    h = _scenes(sim, ref, "cube", seed=6)
    sky = ru.skybox(64, 32, seed=6)
    c = ru.CEILING
    opts = dict(ceiling=ru.ceiling_image(), ceiling_position=c["position"], ceiling_width=c["width"],
                ceiling_depth=c["depth"], marble=True, marble_scale=0.2)
    ref.set_render(sky, aas=2, marble=True, marble_scale=0.2)
    ref.set_ceiling(ru.ceiling_image(), c["position"], c["width"], c["depth"])
    try:
        a, b = sim.render_equirect(h, 64, 32, sky, stereo=stereo, aas=2, **opts)
        ra, rb = ref.render_equirect(64, 32, stereo=stereo)
        descs = ru.ring_descs(2, 32, 24)
        got = sim.render_cameras(h, descs, sky, aas=2, **opts)
        want = [ref.render_camera(d) for d in descs]
    finally:
        ref.clear_ceiling()
    _assert_same(a, ra, "first plane")
    _assert_same(b, rb, "second plane")
    for (gi, gd), (wi, wd) in zip(got, want):
        _assert_same(gi, wi, "camera colour")
        _assert_same(gd, wd, "camera depth")
    sim.destroy(h)


def test_area_kernel_matches_cv2(sim):
    """The render's INTER_AREA kernel alone on tests/golden/rigsim_vectors.npz (cv2 4.13): 3 and 1 channels, factors
    2-4, FLT_MAX whose sums overflow to inf, and inf."""
    import os
    z = np.load(os.path.join(ru.ROOT, "tests", "golden", "rigsim_vectors.npz"))
    for cn in (3, 1):
        for k in (2, 3, 4):
            _assert_same(sim.area(z["src_c%d" % cn], k), z["dst_c%d_k%d" % (cn, k)], "cn %d k %d" % (cn, k))
        _assert_same(sim.area(z["src_c%d" % cn], 1), z["src_c%d" % cn], "copy")


# ---- the app end to end ------------------------------------------------------------------------------------------
APP_FLAGS = dict(num_cams_in_ring=3, ftheta_width=40, ftheta_height=32, ftheta_image_circle_radius=20,
                 pinhole_width=32, pinhole_height=24, eqr_width=48, eqr_height=24)
MODES = ["mono_eqr", "stereo_eqr", "pinhole_ring", "ftheta_ring", "dodecahedron", "icosahedron", "rig_from_json"]


def _app(args):
    import os
    import subprocess
    exe = os.path.join(ru.ROOT, "facebook360_dep_b200", "bin", "RigSimulator")
    r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-800:]
    return r


def _check_cameras(ref, descs, ids, out):
    for d, cid in zip(descs, ids):
        img, dep = ref.render_camera(d)
        assert np.array_equal(ru.read_png8(str(out / (cid + ".png"))), ru.to_u8(img)), cid
        assert np.array_equal(ru.read_png8(str(out / (cid + "_depth.png"))), ru.to_u8(dep)), cid
        _assert_same(ru.read_pfm(str(out / (cid + "_depth.pfm"))), dep, "pfm")


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("mode", MODES)
def test_app_matches_reference(sim, ref, tmp_path, mode, scene):
    """Decoded PNGs and PFMs of every --mode and --scene against the reference's planes under imwrite's 8-bit
    conversion; the camera modes' rigs are the reference's own, written at full precision."""
    import json
    sky = ru.skybox(64, 32, seed=11)
    ru.write_skybox(str(tmp_path / "sky.png"), sky)
    ref.build(scene, seed=1)  # the app never seeds: glibc's initial state is srand(1)
    ref.set_render(sky, aas=2)
    args = ["--mode=" + mode, "--scene=" + scene, "--skybox_path=" + str(tmp_path / "sky.png"),
            "--anti_alias_supersample=2"] + ["--%s=%s" % kv for kv in APP_FLAGS.items()]
    if mode == "mono_eqr":
        _app(args + ["--dest_mono=" + str(tmp_path / "m.png"), "--dest_mono_depth=" + str(tmp_path / "d.png")])
        a, b = ref.render_equirect(48, 24)
        assert np.array_equal(ru.read_png8(str(tmp_path / "m.png")), ru.to_u8(a))
        assert np.array_equal(ru.read_png8(str(tmp_path / "d.png")), ru.to_u8(b * np.float32(255)))
        return
    if mode == "stereo_eqr":
        _app(args + ["--dest_%s=%s" % (k, tmp_path / (k + ".png")) for k in ("left", "right", "stereo")])
        a, b = ref.render_equirect(48, 24, stereo=True)
        assert np.array_equal(ru.read_png8(str(tmp_path / "left.png")), ru.to_u8(a))
        assert np.array_equal(ru.read_png8(str(tmp_path / "right.png")), ru.to_u8(b))
        assert np.array_equal(ru.read_png8(str(tmp_path / "stereo.png")), ru.to_u8(np.concatenate([a, b])))
        return
    out = tmp_path / "cams"
    if mode == "rig_from_json":
        from facebook360_dep_b200 import synth
        rig = synth.ring_rig(2, 36, 28, kind="FTHETA")
        json.dump(rig, open(tmp_path / "rig.json", "w"))
        args.append("--rig_in=" + str(tmp_path / "rig.json"))
    else:
        ref.save_rig(mode, str(tmp_path / "rig.json"), digits=0,
                     **{k: v for k, v in APP_FLAGS.items() if k in ru.RIG_FLAGS})
        rig = json.load(open(tmp_path / "rig.json"))
    r = _app(args + ["--dest_cam_images=" + str(out)])
    assert "------ rendering camera %d" % (len(rig["cameras"]) - 1) in r.stderr
    _check_cameras(ref, capi.rig_descs(rig), [c["id"] for c in rig["cameras"]], out)


def test_app_noise_on_one_camera(sim, ref, tmp_path):
    """--noise_amplitude on a one-camera rig: the noise draws continue the rand() stream after the scene, in the
    reference's per-pixel order (deterministic with one camera; with more the reference draws from racing threads)."""
    import json
    from facebook360_dep_b200 import synth
    sky = ru.skybox(64, 32, seed=12)
    ru.write_skybox(str(tmp_path / "sky.png"), sky)
    rig = synth.ring_rig(1, 40, 30, kind="FTHETA")
    json.dump(rig, open(tmp_path / "rig.json", "w"))
    ref.build("icosahedron", seed=1)
    ref.set_render(sky, aas=2, noise_amplitude=7.5)
    try:
        _app(["--mode=rig_from_json", "--rig_in=" + str(tmp_path / "rig.json"), "--skybox_path=" +
              str(tmp_path / "sky.png"), "--anti_alias_supersample=2", "--noise_amplitude=7.5",
              "--dest_cam_images=" + str(tmp_path / "cams")])
        _check_cameras(ref, capi.rig_descs(rig), [c["id"] for c in rig["cameras"]], tmp_path / "cams")
    finally:
        ref.set_render(sky)
