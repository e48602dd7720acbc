"""The canopy rasteriser (csrc/derp_rephoto.cuh) and the rephotography score at the inputs where such kernels go wrong,
against the CPU checker and against references the checker does not share:

  - non-square and odd meshes, textures, mip chains, cube edges, equirect heights and viewports; deep minification;
    colour coarser than the mesh; the production shapes of SimpleMeshRenderer's defaults
  - DerpCLI-like disparities: NaN outside the image circle and in holes, +-0, negative, +inf, denormals, a far band and
    a near region inside the near plane, with a vertex exactly on it
  - visibility against an fp64 z-buffer, the equirect resample against an fp64 restatement of GL §8.13, and the score
    against cv2 at edge shapes and radii

Everything is seeded."""
import time

import numpy as np
import pytest

from facebook360_dep_b200 import capi, synth
from tests import canopy_oracle
from tests import oracle_hooks as oh
from tests.test_gpu_rephoto import check_disparity_colour
from tests.test_rephoto import EDGE_CASES, check_score_vs_cv2, edge_case

pytestmark = pytest.mark.gpu
NEAR = 0.1  # CanopyScene's kNearZ


@pytest.fixture(scope="module")
def gcuda():
    return capi.Canopy(capi.load_cuda())


@pytest.fixture(scope="module")
def goracle():
    return canopy_oracle.load()


@pytest.fixture(scope="module")
def rcuda():
    return capi.Rephoto(capi.load_cuda())


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.time()
    yield
    print("\n%s: %.1f s wall" % (request.node.name, time.time() - t0))


def _bgra(img_u16):
    h, w = img_u16.shape[:2]
    return np.concatenate([img_u16.astype(np.float32) * np.float32(1 / 65535), np.ones((h, w, 1), np.float32)], -1)


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _render_both(libs, descs, disps, bgra, pos, projection, size, matrix=None, **kw):
    """(colour, colour winners, disparity colour, disparity winners) of each library, the colour and the disparity
    colour as two calls (their textures differ in size, so each is a raster of its own)."""
    out = []
    for lib in libs:
        k = dict(projection=projection, size=size, matrix=matrix, want_winners=True, **kw)
        c, _, wc = lib.render(descs, disps, bgra, pos, want_disparity=False, **k)
        _, d, wd = lib.render(descs, disps, bgra, pos, want_color=False, want_disparity=True, **k)
        out.append((c, wc, d, wd))
    return out


def _check_against_checker(out, what, min_cover=0.05):
    (gc, gwc, gd, gwd), (oc, owc, od, owd) = out
    assert np.array_equal(gwc, owc) and np.array_equal(gwd, owd), (what, int((gwc != owc).sum()), int((gwd != owd).sum()))
    assert (gwc >= 0).any(axis=0).mean() > min_cover, what
    assert _same(gc, oc), (what, float(np.nanmax(np.abs(gc - oc))))
    assert np.array_equal(gd[..., 3] > 0, od[..., 3] > 0), what
    check_disparity_colour(gd, od, what)


# ---- 1. shapes: non-square, odd, mip chains through 1 x k levels, GPU against checker ---------------------------------
VIEWS = {
    "cube33": ("cubemap", (33, 33)),
    "cube41": ("cubemap", (41, 41)),
    "equirect41": ("equirect", (82, 41)),
    "persp75x43": ("perspective", (75, 43)),
}


def _mip_chain(w, h):
    out = [(w, h)]
    while w > 1 or h > 1:
        w, h = max(1, w // 2), max(1, h // 2)
        out.append((w, h))
    return out


@pytest.mark.parametrize("view", sorted(VIEWS))
@pytest.mark.parametrize("texture", ["dense168x108", "coarse45x29", "minify1000x450"])
def test_shapes_match_checker(gcuda, goracle, texture, view):
    """An 84 x 54 mesh of a sphere_rig (FTHETA image circles, off-centre principal points, roll) with colour at another
    aspect: denser (168 x 108: mips 84 x 54, 42 x 27, 21 x 13, 10 x 6, 5 x 3, 2 x 1), coarser than the mesh (45 x 29:
    magnification, lambda < 0) or far denser than the view (1000 x 450 into 33-pixel faces: lambda >= 3 everywhere,
    the deepest levels and GL_REPEAT's wrap).  Odd cube edges, an odd equirect height and an odd W != H viewport."""
    mw, mh = 84, 54
    cw, ch = {"dense168x108": (168, 108), "coarse45x29": (45, 29), "minify1000x450": (1000, 450)}[texture]
    chain = _mip_chain(cw, ch)
    assert any(w % 2 and h % 2 and min(w, h) > 1 for w, h in chain) and any(min(w, h) == 1 < max(w, h) for w, h in chain)
    rig = synth.sphere_rig(6, 168, 108, radius=0.2)
    scene = synth.Scene(seed=13)
    colors, _ = synth.render_rig(rig, cw, ch, scene=scene)
    _, disps = synth.render_rig(rig, mw, mh, scene=scene, noise=False)
    bgra = [_bgra(c) for c in colors]
    descs = capi.rig_descs(rig)
    pos = np.float32([0.012, -0.021, 0.007])
    projection, size = VIEWS[view]
    matrix = capi.snapshot_matrix(pos, [0.3, 0.9, 0.1], [0, 0, 1], 100.0, *size) if projection == "perspective" else None
    out = _render_both((gcuda, goracle), descs, disps, bgra, pos, projection, size, matrix)
    _check_against_checker(out, (texture, view))


# ---- 2. DerpCLI-like disparities and the near plane ------------------------------------------------------------------
def _unit_rays(oracle, desc, w, h):
    """fp64 camera origin and pixel-centre rays (camera.rig at depth 0 and 1) of the camera rescaled to w x h"""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    pix = np.stack([xx.ravel() + 0.5, yy.ravel() + 0.5], -1)
    o, outside = oh.camera_unproject(oracle, desc, pix, 0.0)
    p1, _ = oh.camera_unproject(oracle, desc, pix, 1.0)
    return o, p1 - o, outside.reshape(h, w)


def _vertices64(oracle, goracle, cam, disp, ipd):
    """fp64 canopy vertices: camera.rig(pixel, 1.0f / disparity), minus canopyVS' eye offset (the checker's fp32
    eye(), pinned against fp64 by test_eye_offset_matches_fp64) when ipd != 0; NaN where the vertex is not finite."""
    h, w = disp.shape
    assert cam["resolution"] == [w, h]  # the mesh is the camera at its own resolution
    o, r, _ = _unit_rays(oracle, capi.rig_descs({"cameras": [cam]})[0], w, h)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        dist = (np.float32(1) / disp.astype(np.float32)).astype(np.float64).ravel()
        p = o + r * dist[:, None]
    if ipd != 0:
        p32 = np.ascontiguousarray(p, np.float32)
        e = np.zeros((len(p), 2), np.float32)
        f = goracle.lib.oracle_canopy_eye
        f.restype = None
        f.argtypes = [np.ctypeslib.ctypes.c_void_p, np.ctypeslib.ctypes.c_int, np.ctypeslib.ctypes.c_float,
                      np.ctypeslib.ctypes.c_void_p]
        f(p32.ctypes.data, len(p32), ipd, e.ctypes.data)
        p = p.copy()
        p[:, :2] -= e.astype(np.float64)
    p[~np.isfinite(p).all(1)] = np.nan
    return p


def _face_matrices64(center):
    """createCubemapTexture's projection * view per face in fp64: frustum(-n, n, -n, n, n) (far at infinity) times the
    face's rotation and translate(-center)"""
    table = [((1, 0, 0), (0, 0, -1), (0, -1, 0)), ((-1, 0, 0), (0, 0, 1), (0, -1, 0)), ((0, 1, 0), (1, 0, 0), (0, 0, 1)),
             ((0, -1, 0), (1, 0, 0), (0, 0, -1)), ((0, 0, 1), (1, 0, 0), (0, -1, 0)), ((0, 0, -1), (-1, 0, 0), (0, -1, 0))]
    P = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, -2 * NEAR], [0, 0, -1, 0]], np.float64)
    out = []
    for fwd, right, up in table:
        R = np.array([right, up, -np.asarray(fwd)], np.float64)
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = -R @ np.asarray(center, np.float64)
        out.append(P @ T)
    return out


def _strip_triangles(mw, mh):
    """vertex ids of the strip's triangles in primitive order: prim = (y * (mw - 1) + x) * 2 + k"""
    y, x = np.mgrid[0:mh - 1, 0:mw - 1]
    t0 = np.stack([y * mw + x, (y + 1) * mw + x, y * mw + x + 1], -1)
    t1 = np.stack([(y + 1) * mw + x, y * mw + x + 1, (y + 1) * mw + x + 1], -1)
    return np.stack([t0, t1], 2).reshape(-1, 3)


def _clip_near(poly):
    """Sutherland-Hodgman against z >= -w in fp64"""
    out = []
    for i in range(len(poly)):
        a, b = poly[i], poly[(i + 1) % len(poly)]
        da, db = a[2] + a[3], b[2] + b[3]
        if da >= 0:
            out.append(a)
        if (da >= 0) != (db >= 0):
            out.append(a + (b - a) * (da / (da - db)))
    return out


def _candidates(clip):
    """per triangle (T, 3, 4 clip coordinates): finite and not outside one side plane; and straddling the near plane"""
    fin = np.isfinite(clip).all((1, 2))
    x, y, w = clip[..., 0], clip[..., 1], clip[..., 3]
    with np.errstate(invalid="ignore"):
        rej = (x > w).all(1) | (x < -w).all(1) | (y > w).all(1) | (y < -w).all(1)
        inside = clip[..., 2] + clip[..., 3] >= 0
    cand = fin & ~rej & inside.any(1)
    return cand, cand & ~inside.all(1)


def _zbuffer64(clip, W, H, edge_eps=1e-4, tie_eps=1e-6):
    """The nearest triangle at every pixel centre of a W x H viewport, in fp64: near-plane clip, perspective divide,
    coverage by the clipped polygon's edges, window depth by the polygon's plane.  Returns (winner, ambiguous): pixels
    within edge_eps px of any polygon's edge, or whose two nearest depths are within tie_eps, are ambiguous."""
    win = np.full((H, W), -1, np.int64)
    best = np.full((H, W), np.inf)
    second = np.full((H, W), np.inf)
    amb = np.zeros((H, W), bool)
    cand, _ = _candidates(clip)
    for t in np.nonzero(cand)[0]:
        poly = _clip_near(list(clip[t]))
        if len(poly) < 3:
            continue
        q = np.array(poly)
        X = q[:, 0] / q[:, 3] * (W / 2) + W / 2
        Y = q[:, 1] / q[:, 3] * (H / 2) + H / 2
        Z = q[:, 2] / q[:, 3] * 0.5 + 0.5
        x0, x1 = max(0, int(np.ceil(X.min() - 0.5 - edge_eps))), min(W - 1, int(np.floor(X.max() - 0.5 + edge_eps)))
        y0, y1 = max(0, int(np.ceil(Y.min() - 0.5 - edge_eps))), min(H - 1, int(np.floor(Y.max() - 0.5 + edge_eps)))
        if x0 > x1 or y0 > y1:
            continue
        area = 0.5 * np.sum(X * np.roll(Y, -1) - np.roll(X, -1) * Y)
        if area == 0:
            continue
        s = 1.0 if area > 0 else -1.0
        py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.float64) + 0.5
        inside = np.ones(px.shape, bool)
        near_edge = np.zeros(px.shape, bool)
        dists = []
        for i in range(len(q)):
            j = (i + 1) % len(q)
            ex, ey = X[j] - X[i], Y[j] - Y[i]
            L = np.hypot(ex, ey)
            if L == 0:
                continue
            d = s * (ex * (py - Y[i]) - ey * (px - X[i])) / L  # > 0 inside
            dists.append(d)
            inside &= d > 0
        dmin = np.min(dists, 0)
        near_edge = (np.abs(np.stack(dists)) < edge_eps).any(0) & (dmin > -edge_eps)
        amb[y0:y1 + 1, x0:x1 + 1] |= near_edge
        # window depth: the plane through the polygon (three vertices spanning the largest area)
        k = max(((0, i, i + 1) for i in range(1, len(q) - 1)),
                key=lambda c: abs((X[c[1]] - X[c[0]]) * (Y[c[2]] - Y[c[0]]) - (X[c[2]] - X[c[0]]) * (Y[c[1]] - Y[c[0]])))
        A = np.array([[X[i], Y[i], 1.0] for i in k])
        a, b, c = np.linalg.solve(A, Z[list(k)])
        z = np.clip(a * px + b * py + c, 0, 1)
        cov = inside & ~near_edge
        sub_b, sub_s, sub_w = best[y0:y1 + 1, x0:x1 + 1], second[y0:y1 + 1, x0:x1 + 1], win[y0:y1 + 1, x0:x1 + 1]
        nearer = cov & (z < sub_b)
        sub_s[nearer] = sub_b[nearer]
        sub_s[cov & ~nearer] = np.minimum(sub_s[cov & ~nearer], z[cov & ~nearer])
        sub_b[nearer] = z[nearer]
        sub_w[nearer] = t
    amb |= (second - best) < tie_eps
    return win, amb


def _view_winners(winners, views, W, H):
    """GPU winners in the output layout (views stacked, each top row first) -> [view, window row, column]"""
    return winners.reshape(views, H, W)[:, ::-1, :]


def _derpcli_like(rng, disp, outside):
    """NaN outside the image circle (maskFovKernel) and in interior holes; +-0, negative, +inf and denormal values; a
    far band; a near region (d in [10, 40]: 2.5 - 10 cm from the camera)"""
    d = disp.copy()
    h, w = d.shape
    d[outside] = np.nan
    for _ in range(4):
        y, x = rng.randint(h // 4, 3 * h // 4), rng.randint(w // 4, 3 * w // 4)
        d[y:y + 2, x:x + 3] = np.nan
    specials = np.float32([0.0, -0.0, -0.3, -2.0, np.inf, 1e-40, -1e-41, np.float32(1.4e-45)])
    idx = rng.choice(h * w, 60, replace=False)
    d.ravel()[idx] = specials[np.arange(60) % len(specials)]
    d[:, w // 3: w // 3 + 3] = 1e-6  # far band: 10^6 m
    y0, x0 = h // 2, 2 * w // 3
    d[y0 - 4:y0 + 4, x0 - 5:x0 + 5] = rng.uniform(10, 40, (8, 10)).astype(np.float32)
    d[outside] = np.nan
    return d


def _axis_camera(position, mw, mh):
    """A RECTILINEAR camera at the render position looking along +x whose centre pixel lies on its optical axis (odd
    sensor, principal at the centre): its ray is exactly (1, 0, 0), so disparity 10 puts that vertex at x = 0.1f, on
    the +X face's near plane (z + w == 0 exactly in fp32).  Its left, right, upper and lower neighbours lie just behind
    the plane (d = 12), the rest in front (d = 2): triangles with a vertex on the plane and one on each side.  A focal
    length of 3 px spreads neighbouring rays 18 degrees apart, so that such triangles cover pixel centres."""
    cam = {"version": 1, "type": "RECTILINEAR", "id": "axis", "origin": [float(v) for v in position],
           "forward": [1.0, 0.0, 0.0], "up": [0.0, 0.0, 1.0], "right": [0.0, -1.0, 0.0], "resolution": [mw, mh],
           "focal": [3.0, -3.0]}
    d = np.full((mh, mw), 2.0, np.float32)
    cy, cx = mh // 2, mw // 2
    d[cy, cx - 1] = d[cy, cx + 1] = d[cy - 1, cx] = d[cy + 1, cx] = 12.0
    d[cy, cx] = 10.0
    return cam, d


@pytest.mark.parametrize("shader,blend,ipd", [("svd", True, 0.0), ("on_screen", False, 0.0), ("svd", False, 0.032),
                                              ("on_screen", True, -0.032)])
def test_derpcli_like_disparities_and_near_plane(gcuda, goracle, oracle, shader, blend, ipd):
    """Five FTHETA cameras 6 cm from the centre with DerpCLI-like disparities, plus the axis camera of _axis_camera, as
    a cubemap and a perspective view from a centre on the +X axis's plane x = 0: GPU against checker.  At ipd 0 the
    near-plane path must have run: triangles of the fp64 mesh that straddle z = -w of a view (and are not trivially
    rejected) win pixels on the GPU."""
    mw, mh = 65, 41
    pos = np.float32([0.0, -0.013, 0.004])
    rig = synth.sphere_rig(5, 65, 41, radius=0.06, seed=5)
    scene = synth.Scene(seed=21)
    colors, disps = synth.render_rig(rig, mw, mh, scene=scene)
    rng = np.random.RandomState(9)
    disps = [_derpcli_like(rng, d, _unit_rays(oracle, capi.rig_descs({"cameras": [c]})[0], mw, mh)[2])
             for d, c in zip(disps, rig["cameras"])]
    axis, dax = _axis_camera(pos, mw, mh)
    rig["cameras"].append(axis)
    disps.append(dax)
    colors.append(colors[0])
    bgra = [_bgra(c) for c in colors]
    descs = capi.rig_descs(rig)
    snap = capi.snapshot_matrix(pos, [0.9, -0.3, 0.2], [0, 0, 1], 110.0, 57, 39)
    kw = dict(ipd=ipd, alpha_blend=blend, shader=shader)
    won = {}
    for projection, size, matrix in (("cubemap", (37, 37), None), ("perspective", (57, 39), snap)):
        out = _render_both((gcuda, goracle), descs, disps, bgra, pos, projection, size, matrix, **kw)
        _check_against_checker(out, (shader, blend, ipd, projection), min_cover=0.2)
        if ipd != 0:
            continue
        mats = _face_matrices64(pos) if projection == "cubemap" else [snap.astype(np.float64)]
        W, H = size
        gw = out[0][1]
        tris = _strip_triangles(mw, mh)
        n = 0
        for ci, (cam, d) in enumerate(zip(rig["cameras"], disps)):
            p = _vertices64(oracle, goracle, cam, d, ipd)
            ph = np.concatenate([p, np.ones((len(p), 1))], 1)
            vw = _view_winners(gw[ci], len(mats), W, H)
            for v, M in enumerate(mats):
                clip = (ph @ M.T)[tris]
                _, straddle = _candidates(clip)
                won_px = vw[v][vw[v] >= 0]
                n += int(straddle[won_px].sum())
        won[projection] = n
    if ipd == 0:
        print("pixels won by triangles straddling the near plane:", won)
        assert won["cubemap"] > 0 and won["perspective"] > 0, won


# ---- 3. visibility against an fp64 z-buffer ---------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["cube", "perspective", "cube_ipd"])
def test_winners_match_fp64_zbuffer(gcuda, goracle, oracle, case):
    """Small RECTILINEAR rigs (no image circle, so no alpha test): every pixel's winning primitive is the nearest
    triangle of the fp64 mesh covering the pixel centre, except within 1e-4 px of an edge or 1e-6 of a depth tie."""
    mw, mh = 25, 17
    rig = synth.wall_rig(3, 25, 17, kind="RECTILINEAR", hfov_deg=100.0)
    _, disps = synth.render_rig(rig, mw, mh, scene=synth.Scene(seed=3), noise=False)
    bgra = [np.ones((mh, mw, 4), np.float32)] * 3
    descs = capi.rig_descs(rig)
    pos = np.float32([0.05, 0.011, -0.006])
    ipd = 0.032 if case == "cube_ipd" else 0.0
    if case == "perspective":
        size, matrix = (41, 29), capi.snapshot_matrix(pos, [1, 0.2, -0.1], [0, 0, 1], 120.0, 41, 29)
        mats = [matrix.astype(np.float64)]
    else:
        size, matrix = (33, 33), None
        mats = _face_matrices64(pos)
    W, H = size
    _, _, gw = gcuda.render(descs, disps, bgra, pos, "perspective" if matrix is not None else "cubemap", size, matrix,
                            ipd=ipd, want_winners=True)
    tris = _strip_triangles(mw, mh)
    compared = 0
    for ci, (cam, d) in enumerate(zip(rig["cameras"], disps)):
        p = _vertices64(oracle, goracle, cam, d, ipd)
        ph = np.concatenate([p, np.ones((len(p), 1))], 1)
        vw = _view_winners(gw[ci], len(mats), W, H)
        for v, M in enumerate(mats):
            ref, amb = _zbuffer64((ph @ M.T)[tris], W, H)
            ok = ~amb
            bad = ok & (vw[v] != ref)
            assert not bad.any(), (case, ci, v, int(bad.sum()), np.argwhere(bad)[:5].tolist())
            compared += int((ok & (ref >= 0)).sum())
    print(case, "covered pixels compared with the fp64 z-buffer:", compared)
    assert compared > (2000 if case != "perspective" else 500)


# ---- 4. the equirect resample against an fp64 restatement of GL §8.13 -------------------------------------------------
# GL §8.13 table 8.19: major axis, sc and tc of each face (faces +X, -X, +Y, -Y, +Z, -Z), as (axis index, sign)
GL_FACES = [((0, 1), (2, -1), (1, -1)), ((0, -1), (2, 1), (1, -1)), ((1, 1), (0, 1), (2, 1)),
            ((1, -1), (0, 1), (2, -1)), ((2, 1), (0, 1), (1, -1)), ((2, -1), (0, -1), (1, -1))]


def _face_of(d):
    """GL §8.13's face of direction(s) d (..., 3), ties of |x|, |y|, |z| going to x, then y"""
    a = np.abs(d)
    fx = (a[..., 0] >= a[..., 1]) & (a[..., 0] >= a[..., 2])
    fy = ~fx & (a[..., 1] >= a[..., 2])
    axis = np.where(fx, 0, np.where(fy, 1, 2))
    comp = np.take_along_axis(d, axis[..., None], -1)[..., 0]
    return 2 * axis + (comp < 0)


def _face_st(d, f):
    """(s, t) of directions d on faces f: s = (sc / |ma| + 1) / 2, t = (tc / |ma| + 1) / 2"""
    s = np.empty(d.shape[:-1])
    t = np.empty(d.shape[:-1])
    for k, ((ma, _), (sa, ss), (ta, ts)) in enumerate(GL_FACES):
        m = f == k
        mag = np.abs(d[m][:, ma])
        s[m] = (ss * d[m][:, sa] / mag + 1) / 2
        t[m] = (ts * d[m][:, ta] / mag + 1) / 2
    return s, t


def _texel_point(f, i, j, e):
    """The centre of texel (i, j) of face f (GL rows: j = 0 at the bottom) on the unit cube; a texel one past an edge
    is folded over that edge onto the adjacent face (the cube unfolded: same distance along the edge)."""
    out = np.zeros(np.shape(f) + (3,))
    a = (2 * np.asarray(i, np.float64) + 1) / e - 1
    b = (2 * np.asarray(j, np.float64) + 1) / e - 1
    for k, ((ma, ms), (sa, ss), (ta, ts)) in enumerate(GL_FACES):
        m = f == k
        out[m, ma] = ms
        out[m, sa] = ss * a[m]
        out[m, ta] = ts * b[m]
    over = np.abs(out) > 1
    fold = over.any(-1)
    # the overflowing coordinate becomes +-1 and the old major axis loses the overflow
    for k, ((ma, ms), _, _) in enumerate(GL_FACES):
        m = fold & (f == k)
        excess = (np.abs(out[m]) - 1).max(-1)
        out[m, ma] = ms * (1 - excess)
    out = np.where(over, np.sign(out), out)
    return out


def _lookup(cube, e, f, i, j):
    """texel values (..., 4) of face f, (i, j) in GL's bottom-up rows of the stacked top-row-first layout, with texels
    past an edge taken from the adjacent face"""
    p = _texel_point(f, i, j, e)
    g = _face_of(p)
    s, t = _face_st(p, g)
    ii = np.clip(np.floor(s * e).astype(np.int64), 0, e - 1)
    jj = np.clip(np.floor(t * e).astype(np.int64), 0, e - 1)
    return cube.reshape(6, e, e, 4)[g, e - 1 - jj, ii]


def equirect64(cube, e):
    """equirectFS over an unpremultiplied cube (6 e x e, faces stacked, each top row first): the 2e x e equirect, row 0
    at latitude +pi/2, in fp64.  GL_LINEAR at level 0 with seamless filtering (GL §8.13.1): a texel past one edge
    comes from the adjacent face, one past a corner is the mean of the footprint's other three.  NaN propagates.
    Also returns the footprint's spread (max - min texel per channel) and where the sample lies on a texel-centre row or column (u or v within 1e-6 of an integer): there the
    footprint's second texel has weight 0, and rounding in fp32 or fp64 picks the neighbour on either side, so whether
    a NaN there reaches the sample is not defined by the direction alone."""
    y, x = np.mgrid[0:e, 0:2 * e].astype(np.float64)
    lon = (1 - (x + 0.5) / (2 * e)) * 2 * np.pi
    lat = -((y + 0.5) / e - 0.5) * np.pi
    d = np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], -1)
    f = _face_of(d)
    s, t = _face_st(d, f)
    u, v = s * e - 0.5, t * e - 0.5
    i0, j0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    a, b = (u - i0)[..., None], (v - j0)[..., None]
    cube = cube.astype(np.float64)
    tex, out_i, out_j = [], [], []
    for dj in (0, 1):
        for di in (0, 1):
            i, j = i0 + di, j0 + dj
            out_i.append((i < 0) | (i >= e))
            out_j.append((j < 0) | (j >= e))
            tex.append(_lookup(cube, e, f, i, j))
    tex = np.stack(tex)
    corner = np.stack(out_i) & np.stack(out_j)
    for k in range(4):
        m = corner[k]
        others = [o for o in range(4) if o != k]
        tex[k][m] = (tex[others[0]][m] + tex[others[1]][m] + tex[others[2]][m]) / 3
    on_centre = (np.abs(u - np.round(u)) < 1e-6) | (np.abs(v - np.round(v)) < 1e-6)
    with np.errstate(invalid="ignore"):
        spread = tex.max(0) - tex.min(0)
    out = ((1 - a) * (1 - b) * tex[0] + a * (1 - b) * tex[1]) + ((1 - a) * b * tex[2] + a * b * tex[3])
    return out, on_centre, spread


def _check_equirect(gcuda, descs, disps, bgra, pos, e, what):
    cube = gcuda.render(descs, disps, bgra, pos, "cubemap", (e, e))[0]
    eq = gcuda.render(descs, disps, bgra, pos, "equirect", (2 * e, e))[0]
    ref, on_centre, spread = equirect64(cube, e)
    nan = np.isnan(ref)
    # NaN exactly where the fp64 resample has NaN, except where a weight-0 texel decides (equirect64)
    moot = on_centre[..., None] & (nan != np.isnan(eq))
    assert moot.any(-1).sum() <= max(4, 0.01 * e * e)  # a few samples on the symmetry lines of the directions
    assert np.array_equal(np.isnan(eq) | moot, nan | moot), (what, int((np.isnan(eq) != nan).sum()))
    fin = ~nan & ~np.isnan(eq)
    # fp32 rounding of the weights and trig: 1e-5, plus the fp32 texel coordinate s * e - 0.5, a few ulps of e (2^-21 e
    # texels) off the fp64 one, times the footprint's spread
    excess = np.abs(eq - ref) - spread * (e * 2.0 ** -21)
    err, worst = float(np.abs(eq - ref)[fin].max()), float(excess[fin].max())
    print(what, "equirect: max |cuda - fp64| %.3g (%.3g beyond the coordinate term) over %d values, %.1f%% NaN, "
          "%d samples' NaN decided by a weight-0 texel" % (err, worst, fin.sum(), 100 * nan.mean(), moot.any(-1).sum()))
    assert worst <= 1e-5, (what, err, worst)
    return cube, nan


@pytest.mark.parametrize("e", [2, 3, 7, 40, 41])
def test_equirect_matches_fp64_resample(gcuda, e):
    """Three cameras of a wall rig cover part of the sphere, so NaN (uncovered) texels sit next to covered ones across
    the seams and corners of the cube; the GPU's equirect equals the fp64 resample of the GPU's own cubemap."""
    W = 32
    rig = synth.wall_rig(3, W, W, kind="FTHETA")
    colors, disps = synth.render_rig(rig, W, W, scene=synth.Scene(seed=17))
    bgra = [_bgra(c) for c in colors]
    cube, nan = _check_equirect(gcuda, capi.rig_descs(rig), disps, bgra, np.float32([0.03, 0.0, 0.01]), e, e)
    cnan = np.isnan(cube[..., 0]).reshape(6, e, e)
    assert cnan.any() and (~cnan).any()
    if e >= 7:  # uncovered texels on a face edge next to covered ones on the same edge
        edges = np.concatenate([cnan[:, 0], cnan[:, -1], cnan[:, :, 0], cnan[:, :, -1]], 1)
        assert (edges.any(1) & ~edges.all(1)).any()


# ---- 5. SimpleMeshRenderer's default shapes ---------------------------------------------------------------------------
def test_production_shapes_match_checker_and_fp64_resample(gcuda, goracle):
    """--width 3072 (1536^2 faces), a 2048^2 colour texture and a 1024^2 mesh, two cameras: GPU against checker in
    the equirect, and the GPU's equirect against the fp64 resample of its 1536^2 cubemap."""
    mw = 1024
    rig = synth.sphere_rig(2, 2048, 2048, radius=0.33)
    scene = synth.Scene(seed=29)
    colors, _ = synth.render_rig(rig, 2048, 2048, scene=scene, device="cuda")
    _, disps = synth.render_rig(rig, mw, mw, scene=scene, noise=False, device="cuda")
    bgra = [_bgra(c) for c in colors]
    descs = capi.rig_descs(rig)
    pos = np.float32([0.004, -0.002, 0.001])
    out = _render_both((gcuda, goracle), descs, disps, bgra, pos, "equirect", (3072, 1536))
    _check_against_checker(out, "production", min_cover=0.3)
    _check_equirect(gcuda, descs, disps, bgra, pos, 1536, "production")


# ---- 6. the score against cv2 at edge shapes -------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["MSSIM", "NCC"])
@pytest.mark.parametrize("radius", [1, 2, 4, 5, 31])
@pytest.mark.parametrize("case", EDGE_CASES)
def test_score_edge_shapes_match_cv2(rcuda, case, method, radius):
    """derp_rephoto_score directly against cv2 (tests/golden/rephoto_edge_vectors.npz), test_score_matches_cv2's
    tolerance: odd non-square and cubemap-layout images, kernels wider than the image, 1-pixel dimensions, NaN inputs
    inside the mask and an empty mask."""
    x, y, mask, ref, ref_avg = edge_case(case, method, radius)
    score, avg = rcuda.rephoto_score(x, y, mask, method, radius)
    check_score_vs_cv2(score, avg, ref, ref_avg, mask)
