"""Shared inputs of the RigSimulator tests: the checker (the reference's own RigSimulator.cpp, oracle/rigsim.mk), a
seeded skybox, rigs and rays, and the comparison of scenes.  The checker is None when it has not been built."""
import ctypes as C
import os

import numpy as np

from facebook360_dep_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "librigsim_ref.so")

SCENE_DEFAULTS = dict(num_random_icosahedrons=250, min_icosahedron_dist=100.0, max_icosahedron_dist=250.0,
                      min_icosahedron_radius=20.0, max_icosahedron_radius=50.0, red_triangle=False,
                      ground_plane_dist_m=1.70)


class Ref:
    """ctypes binding of oracle/ref_bridge_rigsim.cpp."""

    def __init__(self, path=REF_LIB):
        L = self.lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        d, i, f, v = C.c_double, C.c_int, C.c_float, C.c_void_p
        L.ref_rigsim_build.argtypes = [C.c_char_p, i, d, d, d, d, i, d, C.c_uint]
        L.ref_rigsim_triangles.argtypes = [v]
        L.ref_rigsim_bvh.argtypes = [C.POINTER(i), C.POINTER(i), v, v, v]
        L.ref_rigsim_set_render.argtypes = [i, i, d, d, d]
        L.ref_rigsim_set_skybox.argtypes = [v, i, i]
        L.ref_rigsim_trace.argtypes = [v, i, v]
        L.ref_rigsim_render_camera.argtypes = [C.POINTER(capi.CameraDesc), v, v]
        L.ref_rigsim_render_mono.argtypes = [i, i, v, v]
        L.ref_rigsim_render_stereo.argtypes = [i, i, v, v]
        L.ref_rigsim_area.argtypes = [v, i, i, i, i, v]
        L.ref_rigsim_set_ceiling.argtypes = [v, i, i, d, d, d]
        L.ref_rigsim_clear_ceiling.argtypes = []
        L.ref_rigsim_save_rig.argtypes = [C.c_char_p, C.c_char_p, i, d, i, i, i, d, i, i, d, d, d, i]
        self._sky = None

    def build(self, scene="icosahedron", seed=1, **kw):
        p = dict(SCENE_DEFAULTS, **kw)
        n = self.lib.ref_rigsim_build(scene.encode(), p["num_random_icosahedrons"], p["min_icosahedron_dist"],
                                      p["max_icosahedron_dist"], p["min_icosahedron_radius"],
                                      p["max_icosahedron_radius"], int(p["red_triangle"]), p["ground_plane_dist_m"], seed)
        assert n >= 0
        tris = np.zeros(max(n, 1), capi.RIGSIM_TRIANGLE)
        self.lib.ref_rigsim_triangles(tris.ctypes.data)
        nn, nl = C.c_int(), C.c_int()
        self.lib.ref_rigsim_bvh(C.byref(nn), C.byref(nl), None, None, None)
        nodes = np.zeros(nn.value, capi.RIGSIM_NODE)
        sph = np.zeros((nn.value, 4), np.float32)
        idx = np.zeros((nn.value, 3), np.int32)
        leaf = np.zeros(max(nl.value, 1), np.int32)
        self.lib.ref_rigsim_bvh(C.byref(nn), C.byref(nl), sph.ctypes.data, idx.ctypes.data, leaf.ctypes.data)
        nodes["center"], nodes["radius"] = sph[:, :3], sph[:, 3]
        nodes["first"], nodes["count"], nodes["escape"] = idx[:, 0], idx[:, 1], idx[:, 2]
        return tris[:n], nodes, leaf[:nl.value]

    def rand(self):
        return int(self.lib.ref_rigsim_rand())

    def set_render(self, skybox, aas=1, marble=False, marble_scale=0.1, noise_amplitude=0.0,
                   interpupillary_radius=3.2):
        self._sky = np.ascontiguousarray(skybox, np.uint8)
        self.lib.ref_rigsim_set_skybox(self._sky.ctypes.data, self._sky.shape[1], self._sky.shape[0])
        self.lib.ref_rigsim_set_render(aas, int(marble), marble_scale, noise_amplitude, interpupillary_radius)

    def trace(self, rays):
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        out = np.empty((len(r), 4), np.float32)
        self.lib.ref_rigsim_trace(r.ctypes.data, len(r), out.ctypes.data)
        return out

    def render_camera(self, desc):
        h, w = int(desc.resolution[1]), int(desc.resolution[0])
        img, dep = np.empty((h, w, 3), np.float32), np.empty((h, w), np.float32)
        assert self.lib.ref_rigsim_render_camera(C.byref(desc), img.ctypes.data, dep.ctypes.data) == 0
        return img, dep

    def render_equirect(self, w, h, stereo=False):
        a = np.empty((h, w, 3), np.float32)
        b = np.empty((h, w, 3) if stereo else (h, w), np.float32)
        (self.lib.ref_rigsim_render_stereo if stereo else self.lib.ref_rigsim_render_mono)(w, h, a.ctypes.data,
                                                                                          b.ctypes.data)
        return a, b

    def area(self, src, k):
        s = np.ascontiguousarray(src, np.float32)
        cn = 1 if s.ndim == 2 else s.shape[2]
        out = np.empty((s.shape[0] // k, s.shape[1] // k) + s.shape[2:], np.float32)
        self.lib.ref_rigsim_area(s.ctypes.data, s.shape[1], s.shape[0], cn, k, out.ctypes.data)
        return out

    def set_ceiling(self, image, position, width, depth):
        """--ceiling_*; the reference loads its ceiling image once per process, so the first image given stays."""
        self._ceil = np.ascontiguousarray(image, np.uint8)
        self.lib.ref_rigsim_set_ceiling(self._ceil.ctypes.data, self._ceil.shape[1], self._ceil.shape[0], position,
                                        width, depth)

    def clear_ceiling(self):
        self.lib.ref_rigsim_clear_ceiling()

    def save_rig(self, mode, path, digits=10, **kw):
        """main's rig of a camera --mode, written by Camera::saveRig(path, rig, {}, digits) (0: shortest round-trip
        doubles); kw: the app's flags."""
        f = dict(RIG_FLAGS, **kw)
        assert self.lib.ref_rigsim_save_rig(mode.encode(), path.encode(), f["num_cams_in_ring"], f["rig_radius"],
                                            f["ftheta_width"], f["ftheta_height"], f["ftheta_image_circle_radius"],
                                            f["ftheta_image_circle_fov"], f["pinhole_width"], f["pinhole_height"],
                                            f["pinhole_fov_horizontal"], f["pinhole_aspect_ratio"],
                                            f["top_cam_vertical_offset"], digits) == 0


# The rig flags of RigSimulator.cpp:46-121 at their defaults
RIG_FLAGS = dict(num_cams_in_ring=14, rig_radius=0.218, ftheta_width=300, ftheta_height=400,
                 ftheta_image_circle_radius=250, ftheta_image_circle_fov=166.667, pinhole_width=512, pinhole_height=512,
                 pinhole_fov_horizontal=77.7, pinhole_aspect_ratio=1.0, top_cam_vertical_offset=13.0)
CEILING = dict(position=3.0, width=40.0, depth=25.0)


def ceiling_image():
    """The one ceiling image every ceiling test uses (the reference keeps the first one it loads)."""
    return skybox(50, 30, seed=8)


def load_ref():
    return Ref() if os.path.exists(REF_LIB) else None


def skybox(w=64, h=32, seed=0):
    """A seeded 8-bit BGR skybox whose every texel differs from its neighbours (a wrong texel changes the colour)."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def ring_descs(n, w, h, kind="FTHETA", radius=0.218):
    return capi.rig_descs(synth.ring_rig(n, w, h, kind=kind, radius=radius))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_scene(a, b):
    """(triangles, nodes, leaf indices) equal bit for bit (NaN centres of empty clusters included)."""
    ta, na, la = a
    tb, nb, lb = b
    return (ta.tobytes() == tb.tobytes() and na.tobytes() == nb.tobytes() and np.array_equal(la, lb))


def write_skybox(path, bgr):
    """An 8-bit RGBA PNG of a B, G, R image (alpha 255), which the app reads as imread(IMREAD_COLOR) does."""
    from tests import sweep_util as su
    su.write_png(path, np.concatenate([bgr, np.full(bgr.shape[:2] + (1,), 255, np.uint8)], 2))


def read_png8(path):
    """Decoder of the 8-bit grey or RGB PNGs the app writes (non-interlaced, filter 0 rows): grey [h, w] or B, G, R."""
    import struct
    import zlib
    data = open(path, "rb").read()
    pos, idat, w, h, cn = 8, b"", 0, 0, 0
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        t, d = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if t == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", d[:10])
            assert depth == 8 and ctype in (0, 2)
            cn = 1 if ctype == 0 else 3
        elif t == b"IDAT":
            idat += d
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + cn * w)
    assert (raw[:, 0] == 0).all()
    img = raw[:, 1:].reshape(h, w, cn)
    return img[..., 0].copy() if cn == 1 else img[..., ::-1].copy()


def to_u8(v):
    """imwrite's conversion of a float image to 8 bits: saturate_cast<uchar> (round half to even, NaN / inf -> 0)."""
    v = np.asarray(v, np.float32)
    ok = np.isfinite(v) & (v > -2147483648.0) & (v < 2147483648.0)
    return np.clip(np.where(ok, np.rint(np.where(ok, v, 0)), 0), 0, 255).astype(np.uint8)


def read_pfm(path):
    data = open(path, "rb").read()
    parts = data.split(b"\n", 3)
    w, h = map(int, parts[1].split())
    return np.frombuffer(parts[3], np.float32).reshape(h, w)
