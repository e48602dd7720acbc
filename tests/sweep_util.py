"""Shared inputs of the sweep-view tests: rigs as the apps hold them and float BGRA images with real alpha."""
import json
import os

import numpy as np

from facebook360_dep_b200 import capi, synth

GOLDEN_RIG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sweep_rig16.json")


def rig(kind, num_cams, width, height, scale=1.0):
    if kind == "golden":
        r = json.load(open(GOLDEN_RIG))
    elif kind == "RECTILINEAR":
        r = synth.ring_rig(num_cams, width, height, kind="RECTILINEAR", hfov_deg=100.0)
    else:
        r = synth.ring_rig(num_cams, width, height, kind=kind)
    return capi.rescaled_descs(capi.rig_descs(r), scale)


def images(descs, seed=0, pad=0):
    """One float B, G, R, A image per camera of round(resolution) (+ pad) pixels, values in [0, 1) with real alpha."""
    rng = np.random.default_rng(seed)
    out = []
    for d in descs:
        w, h = int(round(d.resolution[0])) + pad, int(round(d.resolution[1])) + pad
        out.append(rng.random((h, w, 4), dtype=np.float32))
    return out


def slice_disparities(n, min_depth_m=1, max_depth_m=10):
    """GenerateCameraOverlaps' slices: float(probeDisparity(d, n, 1.0f / min, 1.0f / max)) (ImageUtil.cpp:100-107)."""
    lo = float(np.float32(1.0) / np.float32(min_depth_m))
    hi = float(np.float32(1.0) / np.float32(max_depth_m))
    return np.array([(d / (n - 1)) * lo + (1 - d / (n - 1)) * hi for d in range(n)], np.float64).astype(np.float32)


def equirect_depths(n, depth_min=1.0, depth_max=10.0):
    """GenerateEquirect's depths for i = n - 1 .. 0 (fp32)."""
    f32 = np.float32
    dmin, dmax = f32(1.0) / f32(depth_max), f32(1.0) / f32(depth_min)
    out = []
    for i in range(n - 1, -1, -1):
        frac = f32(i) / f32(n - 1) if n > 1 else f32(0)
        disp = dmin if n == 1 else f32(frac * dmin) + f32(f32(1) - frac) * dmax
        out.append(f32(1.0) / f32(disp))
    return np.array(out, np.float32)


def diff_count(a, b):
    """Values that differ: bits, with any two NaNs equal (the GPU's NaN is not x86's default NaN)."""
    a, b = np.asarray(a), np.asarray(b)
    both_nan = np.isnan(a) & np.isnan(b)
    return int(((a.view(np.uint32) != b.view(np.uint32)) & ~both_nan).sum())


def write_png(path, bgra_u8):
    """A minimal 8-bit RGBA PNG writer (no cv2: GPU tests may not import it); input B, G, R, A."""
    import struct
    import zlib
    h, w = bgra_u8.shape[:2]
    rgba = bgra_u8[..., [2, 1, 0, 3]]
    raw = b"".join(b"\x00" + rgba[y].tobytes() for y in range(h))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def read_png(path):
    """Decoder of 8-bit RGBA, non-interlaced PNGs with filter 0 rows (what io::writePng8 writes): B, G, R, A uint8."""
    import struct
    import zlib
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, w, h = 8, b"", 0, 0
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        t, d = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if t == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", d[:10])
            assert depth == 8 and ctype == 6
        elif t == b"IDAT":
            idat += d
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 4 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 4)[..., [2, 1, 0, 3]].copy()


def to_png8(bgra):
    """The apps' 8-bit conversion of 255.0f * image (pinned to cv2 by tests/golden/sweep_vectors.npz)."""
    v = (np.float32(255.0) * np.asarray(bgra, np.float32)).astype(np.float32)
    ok = np.isfinite(v) & (v > -2147483648.0) & (v < 2147483648.0)
    r = np.where(ok, np.rint(np.where(ok, v, 0)), 0)
    return np.clip(r, 0, 255).astype(np.uint8)


def dataset(tmp, kind, num_cams, width, height, seed=0):
    """A rig JSON and one frame of B, G, R, A PNGs (real alpha) per camera: returns (rig path, color dir, rig dict)."""
    import json
    from facebook360_dep_b200 import synth
    if kind == "RECTILINEAR":
        r = synth.ring_rig(num_cams, width, height, kind="RECTILINEAR", hfov_deg=100.0)
    else:
        r = synth.ring_rig(num_cams, width, height, kind=kind)
    rng = np.random.default_rng(seed)
    for c in r["cameras"]:
        os.makedirs(os.path.join(tmp, "color", c["id"]), exist_ok=True)
        write_png(os.path.join(tmp, "color", c["id"], "000000.png"), rng.integers(0, 256, (height, width, 4), np.uint8))
    json.dump(r, open(os.path.join(tmp, "rig.json"), "w"))
    return os.path.join(tmp, "rig.json"), os.path.join(tmp, "color"), r


def area_scaled(img_u8, scale):
    """The float B, G, R, A image the apps sample: u8 * (1 / 255.f); only scale 1 is restated here."""
    assert scale == 1
    return img_u8.astype(np.float32) * np.float32(1.0 / 255.0)
