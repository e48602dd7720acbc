"""Shared by the interval-proof tests: adversarial argument sets for the math functions the device's proofs widen,
their exact values and ulp distances with mpmath, the C library's functions through ctypes, and the cameras and box
construction of the decided-box tests."""
import ctypes as C
import math

import mpmath
import numpy as np

from facebook360_dep_b200 import capi

mpmath.mp.prec = 200
LIBM = C.CDLL("libm.so.6")
for _n in ("sin", "cos", "atan", "asin", "acos"):
    getattr(LIBM, _n).restype, getattr(LIBM, _n).argtypes = C.c_double, [C.c_double]
LIBM.atan2.restype, LIBM.atan2.argtypes = C.c_double, [C.c_double, C.c_double]
LIBM.acosf.restype, LIBM.acosf.argtypes = C.c_float, [C.c_float]
LIBM.atan2f.restype, LIBM.atan2f.argtypes = C.c_float, [C.c_float, C.c_float]

# CUDA C++ Programming Guide maximum ulp errors (atan2Pos: derp_camera.cuh's bound), and derp_interval.cuh's host budget
DEVICE_ULPS = {"sin": 2, "cos": 2, "atan": 2, "asin": 2, "atan2": 2, "acosf": 2, "atan2f": 3, "atan2Pos": 2}
HOST_ULPS = 2
FLOAT = {"acosf", "atan2f"}
TWO_ARGS = {"atan2", "atan2f", "atan2Pos"}
EXACT = {"sin": mpmath.sin, "cos": mpmath.cos, "atan": mpmath.atan, "asin": mpmath.asin, "atan2": mpmath.atan2,
         "acosf": mpmath.acos, "atan2f": mpmath.atan2, "atan2Pos": mpmath.atan2}


def host(fn, a, b=None):
    """The C library's fn over the arguments (float functions on the arguments narrowed to float)."""
    if fn == "acosf":
        return np.array([LIBM.acosf(float(np.float32(x))) for x in a])
    if fn in ("atan2f",):
        return np.array([LIBM.atan2f(float(np.float32(y)), float(np.float32(x))) for y, x in zip(a, b)])
    if fn in ("atan2", "atan2Pos"):
        return np.array([LIBM.atan2(y, x) for y, x in zip(a, b)])
    f = getattr(LIBM, fn)
    return np.array([f(x) for x in a])


def exact_atan2(y, x):
    """atan2 with IEEE signed zeros (mpmath has no -0): +-0 or +-pi on the x axis, +-pi / 2 on the y axis."""
    if y == 0:
        return mpmath.mpf(0) if math.copysign(1, x) > 0 else math.copysign(1, y) * mpmath.pi
    return mpmath.atan2(mpmath.mpf(y), mpmath.mpf(x))


def ulp_of(e, single):
    """The ulp of the exact value e (mpf): 2^(floor(log2 |e|) - p + 1), at least the format's least subnormal."""
    lo = -149 if single else -1074
    if e == 0:
        return mpmath.ldexp(1, lo)
    ex = int(mpmath.floor(mpmath.log(abs(e), 2)))
    return mpmath.ldexp(1, max(ex - (23 if single else 52), lo))


def ulp_errors(fn, a, b, values):
    """|value - exact| in ulps of the exact value, per argument."""
    single = fn in FLOAT
    out = np.empty(len(values))
    for i, v in enumerate(values):
        x = float(np.float32(a[i])) if single else float(a[i])
        if fn in TWO_ARGS:
            y = float(np.float32(b[i])) if single else float(b[i])
            e = exact_atan2(x, y)
        else:
            e = EXACT[fn](mpmath.mpf(x))
        out[i] = float(abs(mpmath.mpf(float(v)) - e) / ulp_of(e, single))
    return out


def _around(v, k, dtype=np.float64):
    """v and its k nearest neighbours on each side in dtype."""
    v = dtype(v)
    out = [v]
    lo = hi = v
    for _ in range(k):
        lo, hi = np.nextafter(lo, dtype(-np.inf)), np.nextafter(hi, dtype(np.inf))
        out += [lo, hi]
    return out


def _inverse_points(inv, targets, k, dtype):
    """Arguments whose exact result is each target: inv(target) rounded to dtype, with k neighbours each side."""
    out = []
    for t in targets:
        out += _around(float(inv(mpmath.mpf(t))), k, dtype)
    return out


def adversarial(fn, seed=7):
    """(a, b) argument arrays where the functions go wrong: binade crossings of the result, cos near pi / 2, tiny and
    huge arguments, asin near 1, atan2 on the axes and next to the branch cut."""
    rng = np.random.default_rng(seed)
    dt = np.float32 if fn in FLOAT else np.float64
    crossings = [2.0 ** -e for e in range(1, 12)] + [1.0, 2.0]
    if fn in ("sin", "cos"):
        a = [0.0, 5e-324, 1e-300, 1e-10, math.pi, math.pi / 2, math.pi / 4]
        for k in range(1, 9):  # the argument at multiples of pi / 2 (theta runs over [0, pi] in the proofs)
            a += _around(float(mpmath.pi * k / 2), 8)
        inv = mpmath.asin if fn == "sin" else mpmath.acos
        a += _inverse_points(inv, [t for t in crossings if t <= 1], 6, dt)
        a += list(rng.uniform(0, math.pi, 1500)) + list(rng.uniform(-10, 10, 300))
        return np.array(a, np.float64), None
    if fn == "atan":
        a = [0.0, 5e-324, 1e-300, 1e-16, 1.0, 1.6e16, 1.6331239353195370e16, 1e300]
        a += list(np.geomspace(1e-20, 1.6e16, 1500))
        a += _inverse_points(mpmath.tan, [t for t in crossings if t < 1.57], 6, dt)
        return np.array(a, np.float64), None
    if fn == "asin":
        a = _around(1.0, 40) + _around(-1.0, 40) + [0.0, 5e-324, 1e-300, 1e-10, 0.5]
        a += _inverse_points(mpmath.sin, [t for t in crossings if t < 1.57], 6, dt)
        a += list(rng.uniform(-1, 1, 1500))
        return np.array([x for x in a if abs(x) <= 1], np.float64), None
    if fn == "acosf":
        a = _around(1.0, 40, dt) + _around(-1.0, 40, dt) + _around(0.0, 6, dt)
        a += _inverse_points(mpmath.cos, [t for t in crossings + [3.0] if t < 3.1415], 8, dt)
        a += list(rng.uniform(-1, 1, 1500).astype(dt))
        return np.array([x for x in a if abs(x) <= 1], np.float64), None
    # atan2 (y, x) pairs: axes, the cut, binade crossings of the result and random directions
    ys, xs = [], []
    mags = [1.0, 3.5, 1e-30, 1e30] if dt is np.float64 else [1.0, 3.5, 1e-20, 1e20]
    tiny = [5e-324, 1e-300] if dt is np.float64 else [1.4e-45, 1e-40]
    for m in mags:
        for y, x in [(0.0, m), (-0.0, m), (0.0, -m), (-0.0, -m), (m, 0.0), (-m, 0.0), (m, -0.0), (0.0, 0.0),
                     (-0.0, -0.0)] + [(s * t, -m) for t in tiny for s in (1, -1)] + [(s * t, m) for t in tiny for s in (1, -1)]:
            ys.append(y)
            xs.append(x)
    for t in crossings + [-c for c in crossings] + [math.pi / 2 + 0.5, -math.pi / 2 - 0.5, 3.0, -3.0]:
        for m in (1.0, 7.3):
            c, s = mpmath.cos(t) * m, mpmath.sin(t) * m
            for y in _around(float(s), 4, dt):
                ys.append(y)
                xs.append(dt(float(c)))
    ang = rng.uniform(-math.pi, math.pi, 1500)
    r = rng.uniform(0.01, 100, 1500)
    ys += list((r * np.sin(ang)).astype(dt))
    xs += list((r * np.cos(ang)).astype(dt))
    y, x = np.array(ys, np.float64), np.array(xs, np.float64)
    if fn == "atan2Pos":  # its argument y is a norm, y >= 0; at the origin the sweep divides 0 by xy = 0 either way
        y = np.abs(y)
        keep = (y != 0) | (x != 0)
        y, x = y[keep], x[keep]
    return y, x


def float_steps(a, b):
    """The distance in float steps between float32 arrays a and b (their ordered bit patterns)."""
    def key(v):
        i = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(key(a) - key(b))


# ---- cameras ------------------------------------------------------------------------------------------------------
def camera(kind, fov=None, distortion=(0.0, 0.0, 0.0), res=(64, 48), focal=(30.0, 30.0), forward=(1, 0.2, -0.1),
           up=(0, 0, 1), origin=(0.1, -0.2, 0.05)):
    d = capi.CameraDesc()
    d.type = capi.CAM_TYPES[kind]
    f = np.array(forward, float)
    f /= np.linalg.norm(f)
    u = np.array(up, float)
    u = u - f * f.dot(u)
    u /= np.linalg.norm(u)
    r = np.cross(f, u)
    for k, v in (("origin", origin), ("forward", f), ("up", u), ("right", r)):
        for i in range(3):
            getattr(d, k)[i] = float(v[i])
    for i in range(2):
        d.resolution[i] = float(res[i])
        d.focal[i] = float(focal[i])
    for i in range(3):
        d.distortion[i] = float(distortion[i])
    if fov is not None:
        d.has_fov = 1
        d.fov = float(fov)
    return d


def _fn(lib, name, args):
    f = getattr(lib, name)
    f.restype, f.argtypes = C.c_int, args
    return f


def host_sees(lib, desc, pts):
    """derp::sees on the host (derp_test_camera_sees): (pixel [n, 2], seen [n])."""
    f = _fn(lib.lib, "derp_test_camera_sees", [C.POINTER(capi.CameraDesc), C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_void_p])
    p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    pix, seen = np.empty((len(p), 2)), np.empty(len(p), np.uint8)
    lib.check(f(C.byref(desc), 0, p.ctypes.data, len(p), pix.ctypes.data, seen.ctypes.data))
    return pix, seen.astype(bool)


def host_rig(lib, desc, pix, depth):
    """cam.rig(pix, depth) on the host (derp_test_camera_rig): [n, 3]."""
    f = _fn(lib.lib, "derp_test_camera_rig", [C.POINTER(capi.CameraDesc), C.c_void_p, C.c_int, C.c_double,
                                              C.c_void_p, C.c_void_p])
    p = np.ascontiguousarray(pix, np.float64).reshape(-1, 2)
    out, outside = np.empty((len(p), 3)), np.empty(len(p), np.uint8)
    lib.check(f(C.byref(desc), p.ctypes.data, len(p), depth, out.ctypes.data, outside.ctypes.data))
    return out


def camera_info(lib, desc):
    """(rotation [3, 3] rows right, up, backward, distMax, cosFov) as the library builds them."""
    f = _fn(lib.lib, "derp_test_camera_info", [C.POINTER(capi.CameraDesc), C.c_void_p, C.c_void_p, C.c_void_p])
    rot, dm, cf = np.empty(9), C.c_double(), C.c_double()
    lib.check(f(C.byref(desc), rot.ctypes.data, C.byref(dm), C.byref(cf)))
    return rot.reshape(3, 3), dm.value, cf.value


def boxes_around(pts, ulps):
    """Boxes [n, 6] of +-ulps ulps around each point (per coordinate)."""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    sp = np.spacing(np.abs(p)) * ulps
    b = np.empty((len(p), 6))
    b[:, 0::2], b[:, 1::2] = p - sp, p + sp
    return b


def box_samples(boxes, rng, interior=8):
    """[n, 9 + interior, 3]: each box's 8 corners, its centre and random interior points."""
    b = np.asarray(boxes).reshape(-1, 3, 2)
    n = len(b)
    corners = np.array([[(k >> j) & 1 for j in range(3)] for k in range(8)])
    out = np.empty((n, 9 + interior, 3))
    for j in range(3):
        lo, hi = b[:, j, 0][:, None], b[:, j, 1][:, None]
        out[:, :8, j] = np.where(corners[None, :, j] == 1, hi, lo)
        out[:, 8, j] = 0.5 * lo[:, 0] + 0.5 * hi[:, 0]
        out[:, 9:, j] = lo + (hi - lo) * rng.random((n, interior))
    return out


def desc_json(desc, cam_id="cam0"):
    """The rig-JSON camera of a CameraDesc (the inverse of capi.camera_desc_from_json), for the checkers."""
    kind = {v: k for k, v in capi.CAM_TYPES.items()}[desc.type]
    c = {"version": 1, "type": kind, "id": cam_id, "resolution": list(desc.resolution), "focal": list(desc.focal),
         "distortion": list(desc.distortion)}
    for k in ("origin", "forward", "up", "right"):
        c[k] = list(getattr(desc, k))
    if desc.has_principal:
        c["principal"] = list(desc.principal)
    if desc.has_fov:
        c["fov"] = desc.fov
    return c


def edge_points(lib, desc, depth, rng):
    """Rig points on the sensor edges x = 0, x = res, y = 0, y = res, on the FOV cone and the optical axis."""
    W, H = desc.resolution[0], desc.resolution[1]
    cx, cy = (desc.principal[0], desc.principal[1]) if desc.has_principal else (W / 2, H / 2)
    t = rng.uniform(0, 1, 40)
    pix = np.concatenate([np.stack([np.zeros(40), t * H], 1), np.stack([np.full(40, W), t * H], 1),
                          np.stack([t * W, np.zeros(40)], 1), np.stack([t * W, np.full(40, H)], 1), [[cx, cy]]])
    pts = host_rig(lib, desc, pix, depth)
    rot, _, cos_fov = camera_info(lib, desc)
    fwd, up, right = -rot[2], rot[1], rot[0]
    origin = np.array(desc.origin[:])
    if cos_fov > -1:
        s = math.sqrt(max(0.0, 1 - cos_fov * cos_fov))
        for a in np.linspace(0, 2 * np.pi, 24, endpoint=False):
            v = cos_fov * fwd + s * (math.cos(a) * up + math.sin(a) * right)
            pts = np.vstack([pts, origin + v * depth])
    return np.vstack([pts, origin + fwd * depth, origin - fwd * depth])  # the optical axis, ahead and behind


SEES_CAMERAS = [("FTHETA", None, (0, 0, 0)), ("FTHETA", 2.6, (-0.05, 0.004, 0)), ("FTHETA", 1.2, (0, 0, 0)),
                ("FTHETA", math.pi, (0.02, 0, 0)), ("RECTILINEAR", None, (-0.1, 0.02, 0)),
                ("RECTILINEAR", 0.9, (0, 0, 0)), ("EQUISOLID", 2.2, (0, 0, 0)), ("ORTHOGRAPHIC", None, (-0.05, 0, 0))]


def exact_py(lib, desc, p):
    """Camera::sees' pixel row of the point p in exact arithmetic (mpmath): Camera.h:301-341 with exact atan2, sqrt,
    products and quotients; None where the chain is undefined (the optical axis)."""
    rot, dist_max, _ = camera_info(lib, desc)
    mp = mpmath.mpf
    v = [mp(float(p[k])) - mp(desc.origin[k]) for k in range(3)]
    cx, cy, cz = [sum(mp(rot[r][k]) * v[k] for k in range(3)) for r in range(3)]
    d = [mp(x) for x in desc.distortion]

    def factor(r2):
        return 1 + r2 * (d[0] + r2 * (d[1] + r2 * d[2]))

    if desc.type == capi.CAM_ORTHOGRAPHIC:
        n = mpmath.sqrt(cx * cx + cy * cy + cz * cz) if cz < 0 else mpmath.sqrt(cx * cx + cy * cy)
        if n == 0:
            return None
        py = cy / n
        sy = factor((cx / n) ** 2 + py * py) * py
    else:
        xy = mpmath.sqrt(cx * cx + cy * cy)
        if xy == 0:
            return None
        if desc.type == capi.CAM_FTHETA:
            r = mpmath.atan2(xy, -cz)
        elif desc.type == capi.CAM_RECTILINEAR:
            r = xy / -cz if -cz > 0 else mp(16331239353195370.0)
        else:
            r = 2 * mpmath.sqrt((1 + cz / mpmath.sqrt(cx * cx + cy * cy + cz * cz)) / 2)
        r = min(mp(dist_max), r) if math.isfinite(dist_max) else r
        sy = factor(r * r) * r / xy * cy
    principal = desc.principal[1] if desc.has_principal else desc.resolution[1] / 2
    return mp(desc.focal[1]) * sy + mp(principal)
