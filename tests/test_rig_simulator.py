"""RigSimulator's host half (include/derp_rigsim.h) against the checker, the reference's own RigSimulator.cpp compiled
by oracle/rigsim.mk, without a GPU: the scene triangles and the flattened BVH bit for bit, the rand() stream position
they leave, the per-ray code (DERP_HD, run on the host) on random and adversarial rays, the checker's INTER_AREA against
cv2, and the overloads the reference resolves."""
import math
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import rigsim_util as ru

SCENES = ["icosahedron", "cube", "ground_plane"]


@pytest.fixture(scope="module")
def sim():
    return capi.RigSim(capi.load_cuda())


@pytest.fixture(scope="module")
def ref():
    r = ru.load_ref()
    if r is None:
        pytest.skip("the RigSimulator checker (oracle/rigsim.mk) is not built")
    return r


def test_abi_is_exported(sim):
    for name in capi.RIGSIM_SYMBOLS:
        assert hasattr(sim.lib, name), name
    header = open(os.path.join(ru.ROOT, "include", "derp_rigsim.h")).read()
    for name in capi.RIGSIM_SYMBOLS:
        assert name + "(" in header, name


SCENE_CASES = [
    ("icosahedron", {}),
    ("icosahedron", dict(red_triangle=True)),
    ("icosahedron", dict(num_random_icosahedrons=7, min_icosahedron_dist=3.0, max_icosahedron_dist=9.5,
                         min_icosahedron_radius=0.5, max_icosahedron_radius=1.25, red_triangle=True)),
    ("icosahedron", dict(num_random_icosahedrons=1000, max_icosahedron_dist=400.0)),
    ("icosahedron", dict(num_random_icosahedrons=0)),
    ("cube", {}),
    ("cube", dict(red_triangle=True)),  # the flag only changes the icosahedron scene
    ("ground_plane", {}),
]


@pytest.mark.parametrize("seed", [1, 12345])
@pytest.mark.parametrize("scene,kw", SCENE_CASES)
def test_scene_and_bvh_match_reference(sim, ref, scene, kw, seed):
    want = ref.build(scene, seed=seed, **kw)
    want_next = ref.rand()
    sim.srand(seed)
    h = sim.scene(scene, **kw)
    got = sim.scene_arrays(h)
    got_next = sim.rand()
    sim.destroy(h)
    assert ru.same_scene(got, want)
    assert got_next == want_next, "the rand() stream is left at a different position"
    tris, nodes, leaf = got
    assert nodes[0]["escape"] == len(nodes)
    assert sorted(leaf.tolist()) == list(range(len(tris)))
    if scene == "icosahedron" and kw.get("num_random_icosahedrons", 250) >= 250:
        empty = np.isnan(nodes["center"]).any(axis=1)
        assert empty.sum() > 0, "the default scene has empty clusters (shared v0, strict <)"
        assert (nodes["count"][empty] == 0).all()


def test_ground_plane_distance(sim):
    """--ground_plane_dist_m sets the plane's height.  (The reference keeps the vertices in a function-local static,
    so in one process only its first scene's distance counts; the app builds one scene per process, and the checker
    is compared at the default above.)"""
    sim.srand(1)
    h = sim.scene("ground_plane", ground_plane_dist_m=0.3)
    tris, nodes, leaf = sim.scene_arrays(h)
    sim.destroy(h)
    assert (tris["v0"][:, 2] == np.float32(-0.3)).all() and len(tris) == 2 and leaf.tolist() == [0, 1]


def _random_rays(rng, n, spread):
    o = (rng.normal(0, 1, (n, 3)) * rng.choice(spread, (n, 1))).astype(np.float32)
    d = rng.normal(0, 1, (n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([o, d.astype(np.float32)], 1)


def _sky_boundary_rays(cols, rows):
    """Directions whose sky sample lies within a few float steps of a column or row boundary, and the poles."""
    out = []
    a = -math.pi + 2 * math.pi * np.arange(cols + 1) / cols
    for da in (-2e-7, -6e-8, 0.0, 6e-8, 2e-7):
        for z in (0.3, -0.7, 0.999):
            r = math.sqrt(1 - z * z)
            out.append(np.stack([np.cos(a + da) * r, np.sin(a + da) * r, np.full_like(a, z)], 1))
    phi = math.pi * np.arange(rows + 1) / rows
    for dp in (-2e-7, -6e-8, 0.0, 6e-8, 2e-7):
        out.append(np.stack([np.sin(phi + dp) * 0.6, np.sin(phi + dp) * 0.8, np.cos(phi + dp)], 1))
    out.append(np.array([[0, 0, 1], [0, 0, -1], [0, -0.0, -1], [-1, -0.0, 0], [-1, 0, 0], [1e-30, -1e-30, 1]]))
    d = np.concatenate(out).astype(np.float32)
    return np.concatenate([np.zeros_like(d), d], 1)


def _grazing_rays(tris, rng, n=4000):
    """Rays from just off a triangle's plane along one of its edges, through its vertices and across its edges: the
    near-parallel test (a * a < 0.0001f) and the barycentric and distance rejections decide these."""
    rays = []
    for t in tris[rng.integers(0, len(tris), n)]:
        v0, e1, e2, nrm = (t[k].astype(np.float64) for k in ("v0", "e1", "e2", "normal"))
        kind = rng.integers(0, 4)
        if kind == 0:  # along an edge, in the plane
            o, d = v0 - 0.5 * e1, e1
        elif kind == 1:  # at a vertex or an edge midpoint, from a point above the plane
            p = v0 + rng.choice([0.0, 0.5, 1.0]) * e1 + rng.choice([0.0, 0.5]) * e2
            o = p + nrm * rng.uniform(0.1, 5)
            d = p - o
        elif kind == 2:  # almost parallel to the plane
            o = v0 + nrm * 1e-3 - e1
            d = e1 + nrm * rng.uniform(-1e-4, 1e-4) * np.linalg.norm(e1)
        else:  # from the triangle's own plane, backwards
            o = v0 + 0.25 * e1 + 0.25 * e2
            d = -nrm + rng.normal(0, 1e-3, 3)
        rays.append(np.concatenate([o, d / np.linalg.norm(d)]))
    return np.array(rays, np.float32)


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("marble", [False, True])
def test_host_trace_matches_reference(sim, ref, scene, marble):
    rng = np.random.default_rng(17)
    tris, _, _ = ref.build(scene, seed=9)
    sim.srand(9)
    h = sim.scene(scene)
    sky = ru.skybox(97, 53, seed=3)
    ref.set_render(sky, marble=marble, marble_scale=0.1)
    rays = np.concatenate([_random_rays(rng, 20000, [0, 0.3, 30, 300]), _sky_boundary_rays(97, 53),
                           _grazing_rays(tris, rng)])
    want = ref.trace(rays)
    got = sim.trace_host(h, rays, sky, marble=marble, marble_scale=0.1)
    sim.destroy(h)
    bad = (ru.bits(got) != ru.bits(want)).any(axis=1)
    assert not bad.any(), "%d of %d rays differ, first %s" % (bad.sum(), len(rays), rays[bad][0].tolist())
    assert (want[:, 3] < 3e38).sum() > 1000 or scene == "cube"


def test_host_trace_with_empty_clusters_and_marble_scale(sim, ref):
    """Rays aimed at the centres of the default scene's icosahedrons, through the NaN spheres of its empty clusters."""
    tris, nodes, _ = ref.build("icosahedron", seed=4)
    sim.srand(4)
    h = sim.scene("icosahedron")
    assert np.isnan(nodes["center"]).any()
    centres = tris["v0"].reshape(-1, 20, 3).mean(axis=1)
    d = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    rays = np.concatenate([np.zeros_like(d), d], 1).astype(np.float32)
    sky = ru.skybox(40, 20, seed=1)
    for scale in (0.1, 1.7, 0.003):
        ref.set_render(sky, marble=True, marble_scale=scale)
        want = ref.trace(rays)
        got = sim.trace_host(h, rays, sky, marble=True, marble_scale=scale)
        assert (want[:, 3] < 3e38).all()
        assert np.array_equal(ru.bits(got), ru.bits(want))
    sim.destroy(h)


def test_ceiling_on_the_host(sim):
    """The ceiling's hit, its texel and its depth, and a ray that misses it (a plain restatement of the mixed
    double / float arithmetic of RigSimulator.cpp:205-220; the checker cannot load a ceiling image)."""
    sim.srand(1)
    h = sim.scene("ground_plane")
    sky = ru.skybox(8, 4, seed=2)
    ceil = ru.skybox(5, 3, seed=4)
    opts = dict(ceiling=ceil, ceiling_position=2.0, ceiling_width=4.0, ceiling_depth=3.0)
    rays = np.float32([[0, 0, 0, 0.3, -0.2, 0.9327379], [0, 0, 0, 0.9, 0.1, 0.4242641], [0, 0, 0, 0, 0, -1]])
    out = sim.trace_host(h, rays, sky, **opts)
    o, d = rays[0, :3], rays[0, 3:]
    depth = np.float32((2.0 - float(o[2])) / float(d[2]))
    p = o + depth * d
    s, t = np.float32(float(p[0]) / 4.0 + 0.5), np.float32(float(p[1]) / 3.0 + 0.5)
    texel = ceil[int(t * np.float32(3)), int(s * np.float32(5))]
    assert out[0, 3] == depth
    assert np.array_equal(out[0, :3], texel.astype(np.float32) / np.float32(255))
    assert out[1, 3] == np.finfo(np.float32).max  # outside the ceiling's width: the sky
    assert abs(out[2, 3] - 1.70) < 1e-5  # the ground below
    sim.destroy(h)


def test_checker_area_resize_matches_cv2(ref):
    """The checker's INTER_AREA (oracle/rigsimshim) against cv2 4.13, with FLT_MAX sums that overflow to inf."""
    z = np.load(os.path.join(ru.ROOT, "tests", "golden", "rigsim_vectors.npz"))
    for cn in (3, 1):
        for k in (2, 3, 4):
            assert np.array_equal(ru.bits(ref.area(z["src_c%d" % cn], k)), ru.bits(z["dst_c%d_k%d" % (cn, k)])), (cn, k)


def test_reference_overloads_are_pinned():
    """The reference's sky texel calls the float acosf and atan2f and its equirect directions float sincosf (the
    product's kernel and host tables assume these); its stereo eyes call double sincos."""
    obj = os.path.join(ru.ROOT, "oracle", "_ref", "rigsim_app.o")
    if not os.path.exists(obj):
        pytest.skip("the RigSimulator checker (oracle/rigsim.mk) is not built")
    undefined = set(subprocess.run(["nm", "-u", obj], capture_output=True, text=True, check=True).stdout.split())
    for name in ("acosf", "atan2f", "sincosf", "sincos"):
        assert name in undefined, name
    assert "acos" not in undefined and "sin" not in undefined and "cos" not in undefined


def test_refusals(sim):
    sim.srand(1)
    h = sim.scene("cube")
    sky = ru.skybox(8, 4)
    with pytest.raises(capi.DerpError, match="anti_alias_supersample"):
        sim.trace_host(h, np.zeros((1, 6), np.float32), sky, aas=0)
    with pytest.raises(capi.DerpError, match="skybox"):
        sim.trace_host(h, np.zeros((1, 6), np.float32), np.zeros((0, 4, 3), np.uint8))
    bad = capi.RigsimSceneParams(7, 1, 0, 0, 1, 2, 1, 2, 1)
    out = capi.C.c_void_p()
    assert sim.lib.derp_rigsim_scene_create(capi.C.byref(bad), capi.C.byref(out)) != 0
    assert b"unknown scene" in sim.lib.derp_last_error()
    sim.destroy(h)


# ---- the app (csrc/host/RigSimulator.cpp) -----------------------------------------------------------------------------
HOST = os.path.join(ru.ROOT, "facebook360_dep_b200", "csrc", "host")
APP = os.path.join(ru.ROOT, "facebook360_dep_b200", "bin", "RigSimulator")
RIG_MODES = ["pinhole_ring", "ftheta_ring", "dodecahedron", "icosahedron"]


@pytest.fixture(scope="module")
def app():
    subprocess.check_call(["make", "-C", HOST], stdout=subprocess.DEVNULL)
    return APP


def _app_defines():
    import re
    src = open(os.path.join(HOST, "RigSimulator.cpp")).read()
    return {m.group(2): [m.group(1), m.group(3).strip().strip('"'), re.sub(r'"\s*"', "", m.group(4)).strip().strip('"')]
            for m in re.finditer(r'DEFINE_(\w+)\(\s*(\w+)\s*,\s*("[^"]*"|[^,]*?)\s*,\s*((?:"[^"]*"\s*)+)\)', src)}


def test_flag_surface_matches_reference(app):
    """The reference's DEFINE_ lines (RigSimulator.cpp:46-121, tests/golden/rigsim_flags.json) plus --gpu."""
    import json
    want = json.load(open(os.path.join(ru.ROOT, "tests", "golden", "rigsim_flags.json")))
    found = _app_defines()
    assert found.pop("gpu") == ["int32", "0", "CUDA device to use"]
    assert found == want
    h = subprocess.run([app, "--help"], capture_output=True, text=True)
    for flag in want:
        assert "-" + flag + " " in h.stdout, flag


def _run(app, args, cwd=None):
    return subprocess.run([app] + args, capture_output=True, text=True, timeout=300, cwd=cwd)


def test_refusals(app, tmp_path):
    sky = str(tmp_path / "sky.png")
    ru.write_skybox(sky, ru.skybox(8, 4))
    cases = [
        ([], "Check failed"),  # --mode is required
        (["--mode=mono_eqr"], "PNG only"),  # the default res/skybox.jpg: no JPEG decoder
        (["--mode=mono_eqr", "--skybox_path=" + str(tmp_path / "sky.jpg")], "PNG only"),
        (["--mode=mono_eqr", "--skybox_path=" + str(tmp_path / "missing.png")], "failed to load image"),
        (["--mode=mono_eqr", "--skybox_path=" + sky, "--anti_alias_supersample=0"], "anti_alias_supersample"),
        (["--mode=mono_eqr", "--skybox_path=" + sky, "--dest_mono=m.jpg", "--dest_mono_depth=d.png"], "PNG only"),
        (["--mode=mono_eqr", "--skybox_path=" + sky, "--ceiling_path=" + str(tmp_path / "c.jpg")], "PNG only"),
        (["--mode=mono_eqr", "--skybox_path=" + sky], "dest_mono"),
        (["--mode=stereo_eqr", "--skybox_path=" + sky, "--dest_left=l.png"], "dest_right"),
        (["--mode=unknown", "--skybox_path=" + sky], "unexpected mode"),
        (["--mode=pinhole_ring", "--skybox_path=" + sky, "--scene=sphere"], "unexpected scene"),
        (["--mode=rig_from_json", "--skybox_path=" + sky], "rig_in"),
    ]
    for args, msg in cases:
        r = _run(app, args, cwd=str(tmp_path))
        assert r.returncode != 0, args
        assert msg in r.stderr, (args, r.stderr[-400:])


def test_fatal_without_gpu(app, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    sky = str(tmp_path / "sky.png")
    ru.write_skybox(sky, ru.skybox(8, 4))
    r = _run(app, ["--mode=mono_eqr", "--skybox_path=" + sky, "--dest_mono=" + str(tmp_path / "m.png"),
                   "--dest_mono_depth=" + str(tmp_path / "d.png"), "--eqr_width=8", "--eqr_height=4"])
    assert r.returncode != 0 and "derp_rigsim_render_equirect" in r.stderr
    assert not os.path.exists(tmp_path / "m.png")
    assert "building BVH" in r.stderr


RIG_CASES = [{}, dict(num_cams_in_ring=5, rig_radius=0.5, ftheta_width=64, ftheta_height=48,
                      ftheta_image_circle_radius=30, ftheta_image_circle_fov=190.0, pinhole_width=40, pinhole_height=30,
                      pinhole_fov_horizontal=100.0, pinhole_aspect_ratio=1.5, top_cam_vertical_offset=2.5)]


@pytest.mark.parametrize("mode", RIG_MODES)
@pytest.mark.parametrize("case", range(len(RIG_CASES)))
def test_rig_out_matches_reference(app, ref, tmp_path, mode, case):
    """--rig_out against Camera::saveRig of the reference's own rig builders: the same cameras, keys and values at
    --rig_out's 10 decimals (folly's FIXED mode)."""
    import json
    kw = RIG_CASES[case]
    sky = str(tmp_path / "sky.png")
    ru.write_skybox(sky, ru.skybox(8, 4))
    ref.save_rig(mode, str(tmp_path / "ref.json"), **kw)
    r = _run(app, ["--mode=" + mode, "--skybox_path=" + sky, "--rig_out=" + str(tmp_path / "app.json")] +
             ["--%s=%s" % (k, v) for k, v in kw.items()])
    assert r.returncode == 0, r.stderr[-400:]
    got = json.load(open(tmp_path / "app.json"))["cameras"]
    want = json.load(open(tmp_path / "ref.json"))["cameras"]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert set(a) == set(b)
        for k, v in b.items():
            if isinstance(v, list):
                assert np.abs(np.array(a[k], float) - np.array(v, float)).max() <= 0.6e-10, (k, a[k], v)
            else:
                assert a[k] == v, k


@pytest.mark.parametrize("scene", SCENES)
def test_host_trace_with_ceiling_matches_reference(sim, ref, scene):
    """The ceiling's mixed double / float arithmetic (RigSimulator.cpp:205-220) against the reference, with rays aimed
    at its edges and through it from below and above."""
    rng = np.random.default_rng(23)
    ref.build(scene, seed=2)
    sim.srand(2)
    h = sim.scene(scene)
    sky = ru.skybox(31, 17, seed=4)
    ceil = ru.ceiling_image()
    c = ru.CEILING
    ref.set_render(sky)
    ref.set_ceiling(ceil, c["position"], c["width"], c["depth"])
    try:
        edges = []
        for s in np.linspace(-0.5, 0.5, 51):
            for t in np.linspace(-0.5, 0.5, 31):
                p = np.array([s * c["width"], t * c["depth"], c["position"]]) * (1 + rng.normal(0, 1e-7, 3))
                edges.append(np.concatenate([[0, 0, 0], p / np.linalg.norm(p)]))
        rays = np.concatenate([_random_rays(rng, 20000, [0, 0.3, 3, 30]), np.array(edges, np.float32)])
        want = ref.trace(rays)
        got = sim.trace_host(h, rays, sky, ceiling=ceil, ceiling_position=c["position"], ceiling_width=c["width"],
                             ceiling_depth=c["depth"])
    finally:
        ref.clear_ceiling()
    sim.destroy(h)
    assert (want[:, 3] < 3e38).sum() > 1000
    bad = (ru.bits(got) != ru.bits(want)).any(axis=1)
    assert not bad.any(), "%d of %d rays differ, first %s" % (bad.sum(), len(rays), rays[bad][0].tolist())
