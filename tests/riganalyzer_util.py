"""Shared inputs of the RigAnalyzer tests: the checker (the reference's own RigAnalyzer.cpp, oracle/riganalyzer.mk),
rigs of every camera model, PPM parsing and the runs of the app and of the checker's main.  The checker is None when it
has not been built."""
import ctypes as C
import json
import os
import subprocess

import numpy as np

from facebook360_dep_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libriganalyzer_ref.so")
APP = os.path.join(ROOT, "facebook360_dep_b200", "bin", "RigAnalyzer")
GOLDEN_RIG = os.path.join(ROOT, "tests", "golden", "sweep_rig16.json")
FLAGS = json.load(open(os.path.join(ROOT, "tests", "golden", "riganalyzer_flags.json")))
TYPES = ["FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"]


class Ref:
    """ctypes binding of oracle/ref_bridge_riganalyzer.cpp."""

    def __init__(self, path=REF_LIB):
        L = self.lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        L.ref_ra_set_flag.argtypes = [C.c_char_p, C.c_char_p]
        L.ref_ra_main.argtypes = [C.POINTER(C.c_char_p), C.c_int, C.c_char_p, C.c_long]
        L.ref_ra_main.restype = C.c_long
        L.ref_ra_samples.argtypes = [C.c_int, C.c_double, C.c_void_p, C.c_int]
        L.ref_ra_save.argtypes = [C.c_int, C.c_char_p, C.c_char_p, C.c_char_p]
        L.ref_ra_count.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_void_p]

    def set_flags(self, args):
        """Every flag to its default, then the --name=value arguments."""
        values = {k: v[1] for k, v in FLAGS.items()}
        values["overlap_distance"] = "1e4"  # Camera::kNearInfinity
        for a in args:
            k, _, v = a[2:].partition("=")
            values[k] = v if _ else "true"
        for k, v in values.items():
            assert self.lib.ref_ra_set_flag(k.encode(), v.encode()) == 0, k

    def main(self, args):
        """main with the flags of args; returns its stdout as text."""
        self.set_flags(args)
        argv = ["RigAnalyzer"] + list(args)
        arr = (C.c_char_p * len(argv))(*[a.encode() for a in argv])
        buf = C.create_string_buffer(1 << 20)
        n = self.lib.ref_ra_main(arr, len(argv), buf, len(buf))
        assert 0 <= n <= len(buf)
        return buf.raw[:n].decode()

    def samples(self, count, discard_degrees=0.0):
        out = np.zeros((max(count, 1), 3))
        n = self.lib.ref_ra_samples(count, discard_degrees, out.ctypes.data, max(count, 1))
        return out[:n]

    def save(self, kind, rig_path, out_path, cam_id="", args=()):
        """saveRigObj / saveEquirect / saveCamera / saveCrossSection of the rig at rig_path, with the flags of args."""
        self.set_flags(list(args))
        kinds = {"obj": 0, "equirect": 1, "camera": 2, "cross_section": 3}
        assert self.lib.ref_ra_save(kinds[kind], rig_path.encode(), out_path.encode(), cam_id.encode()) == 0

    def count(self, rig_path, points):
        p = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        out = np.zeros(len(p), np.int32)
        self.lib.ref_ra_count(rig_path.encode(), p.ctypes.data, len(p), out.ctypes.data)
        return out


def load_ref():
    return Ref() if os.path.exists(REF_LIB) else None


def read_ppm(path):
    """(header values [w, h, max], int array [h, w]) of a P2 file."""
    tok = open(path).read().split()
    assert tok[0] == "P2"
    w, h, m = int(tok[1]), int(tok[2]), int(tok[3])
    return (w, h, m), np.array(tok[4:], np.int64).reshape(h, w)


def camera_json(kind, res=(200, 150), fov=None, distortion=None, pos=(0, 0, 0.1), fwd=(0, 0, 1), up=(0, 1, 0),
                focal=None, cam_id="cam0"):
    fwd, up = np.array(fwd, float), np.array(up, float)
    right = np.cross(fwd, up)
    f = focal if focal is not None else {"FTHETA": 60.0, "RECTILINEAR": 100.0, "EQUISOLID": 60.0,
                                         "ORTHOGRAPHIC": 90.0}[kind]
    c = {"version": 1, "type": kind, "origin": list(pos), "forward": list(fwd), "up": list(up), "right": list(right),
         "resolution": list(res), "focal": [f, -f], "id": cam_id}
    if fov is not None:
        c["fov"] = fov
    if distortion is not None:
        c["distortion"] = list(distortion)
    return c


def ring_rig(kind, n=4, fov=None, distortion=None, radius=0.1, res=(200, 150)):
    """n cameras of one model on a horizontal ring, facing outwards"""
    cams = []
    for i in range(n):
        a = 2 * np.pi * i / n
        fwd = (np.cos(a), np.sin(a), 0.0)
        cams.append(camera_json(kind, res=res, fov=fov, distortion=distortion,
                                pos=tuple(radius * np.array(fwd)), fwd=fwd, up=(0, 0, 1), cam_id="cam%d" % i))
    return {"cameras": cams}


def write_rig(path, rig):
    with open(path, "w") as f:
        json.dump(rig, f)
    return str(path)


def descs_of(path):
    return capi.rig_descs(json.load(open(path)))


def run_app(args, cwd=None, timeout=900):
    return subprocess.run([APP] + list(args), capture_output=True, text=True, timeout=timeout, cwd=cwd)
