"""The device's interval proofs, probed directly (derp_test_* hooks): the libm bounds they rest on against mpmath and
the host, and their decisions on boxes around boundary points against the host twins at the boxes' corners, centres
and interior points.

A proof that is off by an ulp is wrong only next to a decision boundary, where whole-output comparisons on ordinary
rigs almost never look.  Every family builds its points on such boundaries and asserts both that decided boxes agree
with the host everywhere in the box and that the family yields decided and undecided boxes alike."""
import math

import mpmath
import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests import interval_util as iu

pytestmark = pytest.mark.gpu
BOX_ULPS = (0, 1, 16, 1024)


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return capi.load_cuda()


@pytest.fixture(scope="module")
def ra(cuda):
    return capi.RigAnalysis(cuda)


# ---- libm premises ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["sin", "cos", "atan", "asin", "atan2", "atan2f", "acosf", "atan2Pos"])
def test_math_premises(ra, fn):
    """Device within CUDA's documented bound of the exact value, host within the budget, and the host's value inside
    the interval the proofs widen the device's value to."""
    a, b = iu.adversarial(fn)
    out = ra.math(fn, a, b)
    dev, lo, hi = out[:, 0], out[:, 1], out[:, 2]
    h = iu.host(fn, a, b)
    ed, eh = iu.ulp_errors(fn, a, b, dev), iu.ulp_errors(fn, a, b, h)
    print("%s: %d arguments, device max %.3f ulp, host max %.3f ulp" % (fn, len(a), ed.max(), eh.max()), end="")
    if fn in iu.FLOAT:
        print(", max device-host distance %d float steps" % iu.float_steps(dev, h).max(), end="")
    else:
        print(", max device-host distance %d double steps" % np.abs(dev.view(np.int64) - h.view(np.int64)).max(), end="")
    print()
    assert ed.max() <= iu.DEVICE_ULPS[fn], (a[ed.argmax()], None if b is None else b[ed.argmax()], ed.max())
    if fn == "atan2Pos":
        return  # the sweep's own atan2 (its value only: no proof widens it)
    assert eh.max() <= iu.HOST_ULPS
    inside = (lo <= h) & (h <= hi)
    assert inside.all(), (a[~inside][:4], h[~inside][:4], dev[~inside][:4])


def test_acosf_exhaustive(ra):
    """Every float in [-1, 1]: the device's and glibc's acosf against acos in double, and glibc's value inside the
    device value's widenF."""
    st = ra.acosf_exhaustive()
    print("acosf over [-1, 1]: device max %.4f ulp, host max %.4f ulp, max distance %d float steps, %d outside"
          % (st["device_ulps"], st["host_ulps"], st["steps"], st["outside"]))
    assert st["device_ulps"] <= 2 + 2 ** -20
    assert st["host_ulps"] <= iu.HOST_ULPS
    assert st["outside"] == 0


# ---- exact sees ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"])
def test_exact_sees_bit_identical(cuda, ra, kind):
    """Camera::sees on points is IEEE arithmetic for these types: the device's pixel bits equal the host's
    (-fmad=false), with distortion clamped at distMax."""
    rng = np.random.default_rng(11)
    cams = [iu.camera(kind), iu.camera(kind, distortion=(-0.08, 0.01, -0.001)),
            iu.camera(kind, distortion=(0.3, -0.2, 0.05), fov=1.2)]
    for c in cams:
        pts = rng.normal(size=(20000, 3)) * 3
        pd, sd = ra.sees_device(c, pts)
        ph, sh = iu.host_sees(cuda, c, pts)
        assert np.array_equal(sd, sh)
        assert np.array_equal(pd.view(np.int64), ph.view(np.int64))


# ---- decided boxes ------------------------------------------------------------------------------------------------
def _rotation(cuda, desc):
    return iu.camera_info(cuda, desc)[0]


def _check_boxes(ra, cuda, desc, pts, rng):
    """seesIv on boxes around pts against the host at 17 points per box, and where seen, the exact pixel row of the
    box's centre inside the device's interval; returns (decided, undecided)."""
    nd = nu = 0
    for k in BOX_ULPS:
        boxes = iu.boxes_around(pts, k)
        dec, py = ra.sees_iv(desc, boxes)
        samples = iu.box_samples(boxes, rng)
        pix, seen = iu.host_sees(cuda, desc, samples.reshape(-1, 3))
        seen, hy = seen.reshape(len(boxes), -1), pix[:, 1].reshape(len(boxes), -1)
        for i in np.nonzero(dec >= 0)[0]:
            assert (seen[i] == bool(dec[i])).all(), (k, boxes[i], dec[i], seen[i])
            if dec[i] == 1:
                assert ((py[i, 0] <= hy[i]) & (hy[i] <= py[i, 1])).all(), (k, boxes[i], py[i], hy[i])
                e = iu.exact_py(cuda, desc, samples[i, 8])
                assert e is not None and py[i, 0] <= e <= py[i, 1], (k, boxes[i], py[i], e)
        nd += int((dec >= 0).sum())
        nu += int((dec < 0).sum())
    return nd, nu


@pytest.mark.parametrize("kind,fov,dist", iu.SEES_CAMERAS)
def test_sees_iv_decided_boxes(cuda, ra, kind, fov, dist):
    """Sensor edges, the FOV cone (cosFov -1, 0, > 0 and < 0), the optical axis and behind a wide FTHETA."""
    rng = np.random.default_rng(5)
    desc = iu.camera(kind, fov=fov, distortion=dist)
    pts = np.vstack([iu.edge_points(cuda, desc, d, rng) for d in (0.7, 3.0)])
    nd, nu = _check_boxes(ra, cuda, desc, pts, rng)
    print("%s fov %s: %d decided, %d undecided boxes" % (kind, fov, nd, nu))
    assert nd > 0 and nu > 0


def _exact_rig_point(desc, rot, x, y, r, depth):
    """cam.rig({x + .5, y + .5}, depth) in exact arithmetic from the shared IEEE sx, sy, norm and undistort's r."""
    sx = (x + 0.5 - (desc.principal[0] if desc.has_principal else desc.resolution[0] / 2)) / desc.focal[0]
    sy = (y + 0.5 - (desc.principal[1] if desc.has_principal else desc.resolution[1] / 2)) / desc.focal[1]
    sq = sx * sx + sy * sy
    if sq == 0:
        u = [mpmath.mpf(0), mpmath.mpf(0), mpmath.mpf(-1)]
    else:
        norm, r = mpmath.mpf(math.sqrt(sq)), mpmath.mpf(r)
        if desc.type == capi.CAM_FTHETA:
            th = r
        elif desc.type == capi.CAM_RECTILINEAR:
            th = mpmath.atan(r)
        elif desc.type == capi.CAM_EQUISOLID:
            th = 2 * mpmath.asin(r / 2) if r <= 2 else mpmath.mpf(3.14159265358979323846)
        else:
            th = mpmath.asin(r) if r <= 1 else mpmath.mpf(3.14159265358979323846 / 2)
        f = mpmath.sin(th) / norm
        u = [f * sx, f * sy, -mpmath.cos(th)]
    return [desc.origin[k] + (rot[0][k] * u[0] + rot[1][k] * u[1] + rot[2][k] * u[2]) * mpmath.mpf(depth)
            for k in range(3)]


RIG_POINT_CAMERAS = [("FTHETA", 20.0, (-0.06, 0.008, 0), False), ("RECTILINEAR", 20.0, (-0.06, 0.008, 0), False),
                     ("EQUISOLID", 20.0, (-0.06, 0.008, 0), False), ("ORTHOGRAPHIC", 20.0, (-0.06, 0.008, 0), False),
                     ("EQUISOLID", 7.5, (0, 0, 0), True), ("ORTHOGRAPHIC", 15.0, (0, 0, 0), True)]


@pytest.mark.parametrize("kind,focal,dist,axis", RIG_POINT_CAMERAS)
def test_rig_point_iv_holds_host_and_exact(cuda, ra, kind, focal, dist, axis):
    """rigPointIv's intervals hold the host's rig point and the exact chain from undistort's result.

    The axis-aligned cameras (forward -z at the origin, principal (16.5, 11.5)) put pixel (31, 11) at sensor radius
    15 / 15 = 1 (ORTHOGRAPHIC: theta = asin(1)) or 15 / 7.5 = 2 (EQUISOLID: theta = 2 asin(1)).  There the exact chain
    gives cos(theta) = 0 or sin(theta) = 0 while the device's theta is pi / 2 or pi rounded, so only theta's own
    widening (eTheta) keeps the exact world coordinate, which depends on that one factor alone, in the interval."""
    if axis:
        desc = iu.camera(kind, focal=(focal, focal), res=(33, 23), forward=(0, 0, -1), up=(0, 1, 0), origin=(0, 0, 0))
    else:
        desc = iu.camera(kind, distortion=dist, focal=(focal, focal + 1), res=(33, 24))
    rot = _rotation(cuda, desc)
    W, H = int(desc.resolution[0]), int(desc.resolution[1])
    pix = np.array([(x, y) for y in range(H) for x in range(W)], np.int32)
    for depth in (0.37, 5.0):
        iv = ra.rig_point_iv(desc, pix, depth)
        hp = iu.host_rig(cuda, desc, pix + 0.5, depth)
        assert ((iv[:, 0:6:2] <= hp) & (hp <= iv[:, 1:6:2])).all()
        for i in range(len(pix)):
            e = _exact_rig_point(desc, rot, pix[i, 0], pix[i, 1], iv[i, 6], depth)
            for k in range(3):
                assert iv[i, 2 * k] <= e[k] <= iv[i, 2 * k + 1], (kind, pix[i], k)


def _eqr_points(W, H, depth, rows=None):
    """Points whose exact direction lies on texel edges u W = j, v H = i (and, for decided boxes, texel centres), on
    the poles, the seam and theta = 0."""
    pts = []
    for i in ([v / 2 for v in range(2 * H + 1)] if rows is None else rows):
        phi = mpmath.pi * mpmath.mpf(i) / H
        for j in [v / 2 for v in range(2 * W + 1)]:
            th = -2 * mpmath.pi * mpmath.mpf(j) / W
            pts.append([float(mpmath.sin(phi) * mpmath.cos(th) * depth), float(mpmath.sin(phi) * mpmath.sin(th) * depth),
                        float(mpmath.cos(phi) * depth)])
    for y in (0.0, -0.0, 1e-300, -1e-300, 1e-45, -1e-45):
        pts += [[-depth, y, 0.3], [depth, y, -0.2], [-1e-3, y, depth]]
    pts += [[0.0, 0.0, depth], [0.0, 0.0, -depth], [1e-9, 0, depth], [1e-9, -1e-9, -depth]]
    # |z| > 1 after the float depth: only where float(norm) is subnormal (float(2e-45) = 1.4e-45, so z = 1.43); above
    # that range sqrt(w * w) = |w| and the float rounding of norm cannot push |z| past 1 + 2^-24
    pts += [[0.0, 0.0, 2.0e-45], [1e-46, 0.0, -2.1e-45], [0.0, 3e-46, 2.2e-45], [0.0, 0.0, 2.9e-45]]
    pts += list(np.random.default_rng(W * H).normal(size=(64, 3)) * depth)  # away from every edge, mostly
    return np.array(pts)


@pytest.mark.parametrize("W,H", [(1, 1), (7, 5), (64, 32), (4096, 2048)])
def test_eqr_index_proven_decided_boxes(cuda, W, H):
    sv = capi.SweepView(cuda)
    rng = np.random.default_rng(9)
    nd = nu = 0
    for depth in (1.0, 2.7):
        pts = _eqr_points(min(W, 96), min(H, 48), depth) if W < 4096 else _eqr_points(W // 64, H // 64, depth)
        if W >= 4096:  # every column edge (and centre) on the rows next to the poles, and every row edge
            pts = np.vstack([pts, _eqr_points(W, H, depth, rows=[1, H - 1]), _eqr_points(4, H, depth)])
        for k in BOX_ULPS:
            boxes = iu.boxes_around(pts, k)
            got = sv.eqr_index(boxes, W, H, proven=True)
            samples = iu.box_samples(boxes, rng)
            host = sv.eqr_index(samples.reshape(-1, 3), W, H).reshape(len(boxes), -1)
            for i in np.nonzero(got != -2)[0]:
                assert (host[i] == got[i]).all(), (W, H, k, boxes[i], got[i], host[i])
            nd += int((got != -2).sum())
            nu += int((got == -2).sum())
    print("eqrIndexProven %dx%d: %d decided, %d undecided boxes" % (W, H, nd, nu))
    assert nd > 0 and nu > 0


def _sky_dirs(rows, cols):
    """Float directions on row and column edges, the seam and the binade crossings of phi and atan2."""
    d = []
    ths = [mpmath.mpf(2) * mpmath.pi * j / cols - mpmath.pi for j in range(cols + 1)] + \
          [mpmath.mpf(s) for s in (0.5, 1, 2, -0.5, -1, -2)]
    phis = [mpmath.pi * i / rows for i in range(rows + 1)] + [mpmath.mpf(s) for s in (0.5, 1, 2)]
    for phi in phis:
        for th in ths:
            d.append([float(mpmath.sin(phi) * mpmath.cos(th)), float(mpmath.sin(phi) * mpmath.sin(th)),
                      float(mpmath.cos(phi))])
    d = np.array(d, np.float32)
    seam = np.array([[-1, 0, 0.2], [-1, -0.0, 0.2], [-1, 1e-45, -0.3], [-1, -1e-45, 0.1]], np.float32)
    return np.vstack([d, seam])


@pytest.mark.parametrize("rows,cols", [(1, 1), (9, 17), (512, 1024)])
def test_sky_texel_decided(cuda, rows, cols):
    rs = capi.RigSim(cuda)
    base = _sky_dirs(min(rows, 64), min(cols, 128))
    nd = nu = 0
    for k in BOX_ULPS:
        d = base.copy()
        for _ in range(min(k, 16)):  # k float steps along each component (1024: a 1024-ulp offset)
            d = np.nextafter(d, np.float32(np.inf))
        if k == 1024:
            d = (base + np.spacing(np.abs(base)) * 1024).astype(np.float32)
        got = rs.sky_texel(d, rows, cols)
        host = rs.sky_texel(d, rows, cols, host=True)
        dec = got[:, 0] >= 0
        assert np.array_equal(got[dec], host[dec]), (k, d[dec][np.any(got[dec] != host[dec], 1)][:4])
        nd += int(dec.sum())
        nu += int((~dec).sum())
    print("skyTexelDevice %dx%d: %d decided, %d undecided" % (rows, cols, nd, nu))
    assert nd > 0 and nu > 0


def test_proven_count_timing(cuda, ra):
    """Cameras with equal and adjacent float t, and more than 32 seeing cameras (timing list full: host)."""
    rng = np.random.default_rng(13)
    same = [iu.camera("FTHETA", fov=2.0, res=(200, 100), focal=(60.0, 60.0)) for _ in range(3)]
    near = [iu.camera("FTHETA", fov=2.0, res=(200, 100), focal=(60.0, 60.0), origin=(0.1, -0.2, 0.05 + 1e-9 * i))
            for i in range(3)]
    many = [iu.camera("FTHETA" if i % 2 else "RECTILINEAR", res=(200, 100), focal=(60.0, 60.0),
                      forward=(1, 0.2 + 1e-3 * i, -0.1)) for i in range(36)]
    total_dec = total_und = 0
    # pixel rows whose t = row / 100 lies halfway between two floats: the device must leave them to the host
    t = rng.uniform(0.2, 0.8, 500).astype(np.float32)
    rows = (t.astype(np.float64) + np.nextafter(t, np.float32(1)).astype(np.float64)) / 2 * 100
    for rig in (same, near, same + near, many):
        pts = np.vstack([np.array([[3.0, 0.6, -0.3]]) + rng.normal(size=(3000, 3)) * 0.8,
                         iu.host_rig(cuda, rig[0], np.stack([rng.uniform(0, 200, 500), rows], 1), 2.0)])
        c, t = ra.proven_count(rig, pts)
        hc, ht = ra.proven_count(rig, pts, host=True)
        dec = c >= 0
        assert np.array_equal(c[dec], hc[dec])
        assert np.array_equal(t[dec].view(np.uint32), ht[dec].view(np.uint32))
        if rig is many:
            assert (c[hc > 32] == -1).all() and (hc > 32).any()
        total_dec += int(dec.sum())
        total_und += int((~dec).sum())
    print("provenCount: %d decided, %d undecided points" % (total_dec, total_und))
    assert total_dec > 0 and total_und > 0


def test_proven_count_t_at_float_midpoints(cuda, ra):
    """An FTHETA camera whose t = py / res lies halfway between two floats, next to a RECTILINEAR camera (exact
    sees) whose t is the lower of the two: minTimingDiff is 0 or one float step depending on how the host rounds the
    FTHETA camera's t, so a device that decided that t from one end of its interval would differ."""
    rng = np.random.default_rng(17)
    a = iu.camera("FTHETA", fov=2.0, res=(200, 100), focal=(60.0, 60.0))
    t = rng.uniform(0.3, 0.7, 300).astype(np.float32)
    mid = (t.astype(np.float64) + np.nextafter(t, np.float32(1)).astype(np.float64)) / 2
    pts = iu.host_rig(cuda, a, np.stack([rng.uniform(80, 120, len(t)), mid * 100], 1), 2.0)
    decided, host_diffs = 0, set()
    for p, tk in zip(pts, t):
        b = iu.camera("RECTILINEAR", res=(200, 100), focal=(60.0, 60.0))
        pix, _ = iu.host_sees(cuda, b, p[None])
        b.has_principal = 1
        b.principal[0], b.principal[1] = 100.0, 50.0 + (float(tk) * 100 - pix[0, 1])
        pix, seen = iu.host_sees(cuda, b, p[None])
        assert seen[0] and np.float32(pix[0, 1] / 100) == tk
        c, tm = ra.proven_count([a, b], p[None])
        hc, ht = ra.proven_count([a, b], p[None], host=True)
        assert hc[0] == 2
        host_diffs.add(float(ht[0]) > 0)
        if c[0] >= 0:
            decided += 1
            assert c[0] == 2 and tm.view(np.uint32)[0] == ht.view(np.uint32)[0], (p, tk, tm, ht)
    print("t at float midpoints: %d of %d points decided" % (decided, len(t)))
    assert host_diffs == {False, True}  # the host rounds both ways over the set


def test_camera_mode_on_sensor_edges_matches_checker(tmp_path):
    """RigAnalyzer's camera mode through the public entry point on a rig whose pixel centres land on the other
    cameras' sensor edges: cameras 1 and 2 are camera 0 with the principal point half a pixel off, so camera 0's last
    column and row project to x = res and y = res of camera 1 (outside) and its first to x = 0, y = 0 of camera 2
    (inside).  0 differences from the checker, and some pixels resolved on the host."""
    import json

    import torch
    from tests import riganalyzer_util as ru
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    ref = ru.load_ref()
    if ref is None:
        pytest.skip("the RigAnalyzer checker (oracle/riganalyzer.mk) is not built")
    lib = capi.RigAnalysis(capi.load_cuda())
    cams = []
    for i, shift in enumerate((0.0, 0.5, -0.5)):
        d = iu.camera("FTHETA", res=(96, 64), focal=(40.0, 40.0))
        d.has_principal = 1
        d.principal[0], d.principal[1] = 48.0 + shift, 32.0 + shift
        cams.append(iu.desc_json(d, "cam%d" % i))
    path = ru.write_rig(tmp_path / "edges.json", {"cameras": cams})
    descs = ru.descs_of(path)
    for distance in (2.0, 1e4):
        got = lib.camera(descs, 0, distance)
        host = lib.last_host_points()
        ref.set_flags(["--overlap_distance=%r" % distance])
        assert ref.lib.ref_ra_save(2, path.encode(), str(tmp_path / "c.ppm").encode(), b"cam0") == 0
        want = ru.read_ppm(tmp_path / "c.ppm")[1]
        print("camera mode on sensor edges at %g: %d of %d pixels on the host" % (distance, host, got.size))
        assert np.array_equal(got, want)
        assert host > 0
