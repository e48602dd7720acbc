"""Shared inputs of the ProjectEquirectsToCameras / ProjectCamerasToEquirects tests: rigs of every camera model, the
checker library, 1-pixel checkerboard masks and the 8-bit grey PNG reader."""
import json
import os

import numpy as np

from facebook360_dep_b200 import capi, synth
from tests import sweep_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libeqrproject_ref.so")
KINDS = ["FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"]


def load_ref():
    """The checker (oracle/eqrproject.mk), or None when it has not been built."""
    return capi.SweepView(REF_LIB) if os.path.exists(REF_LIB) else None


def rig_json(kind, n, w, h):
    if kind == "golden":
        return json.load(open(su.GOLDEN_RIG))
    if kind == "RECTILINEAR":
        return synth.ring_rig(n, w, h, kind="RECTILINEAR", hfov_deg=100.0)
    if kind == "poles":  # cameras looking straight up and down, the principal point on a pixel corner and a centre
        r = synth.ring_rig(2, w, h, kind="FTHETA")
        for c, s in zip(r["cameras"], (1.0, -1.0)):
            c["forward"], c["up"], c["right"] = [0.0, 0.0, s], [1.0, 0.0, 0.0], [0.0, s, 0.0]
        r["cameras"][1]["principal"] = [w / 2 + 0.5, h / 2 + 0.5]
        return r
    return synth.ring_rig(n, w, h, kind=kind)


def rig(kind, n=4, w=40, h=30):
    return capi.rig_descs(rig_json(kind, n, w, h))


def rescaled_to_width(ref, descs, width):
    """The reference's own rescaleCameras at --width (ref_eqrproject_rescale of the checker)."""
    import ctypes as C
    out = (capi.CameraDesc * len(descs))()
    fn = ref.lib.ref_eqrproject_rescale
    fn.restype, fn.argtypes = C.c_int, [C.POINTER(capi.CameraDesc), C.c_int, C.c_int, C.POINTER(capi.CameraDesc)]
    assert fn(descs, len(descs), width, out) == 0
    return out


def checkerboards(n, base=(64, 32)):
    """One 1-pixel checkerboard per camera, of a different size each (any index disagreement flips a pixel)."""
    out = []
    for i in range(n):
        w, h = base[0] + 2 * i, base[1] + i
        yy, xx = np.mgrid[0:h, 0:w]
        out.append(((xx + yy + i) % 2).astype(np.uint8))
    return out


def read_png_gray8(path):
    """Decoder of 8-bit grey, non-interlaced PNGs with filter 0 rows (what io::writePng8Gray writes)."""
    import struct
    import zlib
    data = open(path, "rb").read()
    pos, idat, w, h = 8, b"", 0, 0
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        t, d = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if t == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", d[:10])
            assert depth == 8 and ctype == 0
        elif t == b"IDAT":
            idat += d
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].copy()


def write_png_gray8(path, img):
    import struct
    import zlib
    h, w = img.shape
    raw = b"".join(b"\x00" + img[y].tobytes() for y in range(h))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))
