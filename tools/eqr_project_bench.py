"""Times ProjectEquirectsToCameras' projection and both apps on one GPU, and writes one JSON line.

  library : derp_project_equirect_masks on the golden 16-camera rig (tests/golden/sweep_rig16.json) at its full
            3360 x 2160 with one 4096 x 2048 mask per camera, masks and outputs resident on the device, CUDA events
            around the call; with the pixels the device left to the host per call (derp_project_last_host_pixels).
            The masks are a painted region (a band of latitude with a hole) plus a 1-pixel checkerboard in one
            quadrant, so both the proof and the mask reads are exercised.
  app     : ProjectEquirectsToCameras on a dataset of the same shape (--frames frames), wall time per frame split into
            decode / device / encode as the app logs it.
  c2e     : ProjectCamerasToEquirects on the same rig with colour frames, per frame at --eqr_width 1024 and 4096.
Usage: python tools/eqr_project_bench.py [--out profiles/h100_eqr_project_16cam.json] [--frames 2]"""
import argparse
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from facebook360_dep_b200 import capi  # noqa: E402
from tests import eqr_project_util as eu, sweep_util as su  # noqa: E402

BIN = os.path.join(ROOT, "facebook360_dep_b200", "bin")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "not measured"


def mask(w, h, seed):
    yy, xx = np.mgrid[0:h, 0:w]
    m = ((yy > h // 4) & (yy < 3 * h // 4)).astype(np.uint8)
    m[h // 3:h // 2, w // 3:w // 2] = 0
    q = (yy < h // 2) & (xx < w // 2)
    m[q] = ((xx + yy + seed) % 2)[q]
    return m


def timing(stderr):
    m = re.search(r"Timing: decode ([\d.e+-]+) ms, device ([\d.e+-]+) ms, encode ([\d.e+-]+) ms .*wall ([\d.e+-]+) ms",
                  stderr)
    return [float(v) for v in m.groups()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_eqr_project_16cam.json"))
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    name, limit = gpu_info()
    lib = capi.load_cuda().lib
    lib.derp_project_equirect_masks.restype = C.c_int
    lib.derp_project_last_host_pixels.restype = C.c_uint64
    descs = eu.rig("golden")
    n = len(descs)
    W, H = int(descs[0].resolution[0]), int(descs[0].resolution[1])
    masks = [torch.from_numpy(mask(4096, 2048, i)).cuda() for i in range(n)]
    outs = [torch.empty((int(d.resolution[1]), int(d.resolution[0])), dtype=torch.uint8, device="cuda") for d in descs]
    mp = (C.c_void_p * n)(*[m.data_ptr() for m in masks])
    op = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    sizes = np.array([[4096, 2048]] * n, np.int32).reshape(-1)

    def call():
        rc = lib.derp_project_equirect_masks(0, descs, n, C.c_double(1000.0), mp, sizes.ctypes.data, op)
        assert rc == 0, capi.load_cuda().lib.derp_last_error()

    call()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(a.reps):
        call()
    end.record()
    torch.cuda.synchronize()
    lib_ms = start.elapsed_time(end) / a.reps
    host_px = int(lib.derp_project_last_host_pixels())
    pixels = sum(int(d.resolution[0]) * int(d.resolution[1]) for d in descs)

    tmp = tempfile.mkdtemp(prefix="eqr_project_bench_")
    try:
        rig = json.load(open(su.GOLDEN_RIG))
        rig_path = os.path.join(tmp, "rig.json")
        json.dump(rig, open(rig_path, "w"))
        rng = np.random.default_rng(0)
        color = rng.integers(0, 256, (H, W, 4), np.uint8)
        for f in range(a.frames):
            for i, c in enumerate(rig["cameras"]):
                for sub in ("masks", "color"):
                    os.makedirs(os.path.join(tmp, sub, c["id"]), exist_ok=True)
                eu.write_png_gray8(os.path.join(tmp, "masks", c["id"], "%06d.png" % f), mask(4096, 2048, i) * 255)
                p = os.path.join(tmp, "color", c["id"], "%06d.png" % f)
                if f == 0 and i == 0:
                    su.write_png(p, color)
                else:
                    shutil.copy(os.path.join(tmp, "color", rig["cameras"][0]["id"], "000000.png"), p)
        last = "%06d" % (a.frames - 1)
        p = subprocess.run([os.path.join(BIN, "ProjectEquirectsToCameras"), "--rig=" + rig_path,
                            "--eqr_masks=" + os.path.join(tmp, "masks"), "--output=" + os.path.join(tmp, "out"),
                            "--last=" + last], capture_output=True, text=True, timeout=3000)
        assert p.returncode == 0, p.stderr[-2000:]
        dec, dev, enc, wall = timing(p.stderr)
        app = {"frames": a.frames, "wall_ms_per_frame": wall / a.frames, "decode_ms_per_frame": dec / a.frames,
               "device_ms_per_frame": dev / a.frames, "encode_ms_per_frame_summed_over_threads": enc / a.frames}
        c2e = {}
        for ew in (1024, 4096):
            p = subprocess.run([os.path.join(BIN, "ProjectCamerasToEquirects"), "--rig=" + rig_path,
                                "--color=" + os.path.join(tmp, "color"), "--output=" + os.path.join(tmp, "c2e"),
                                "--last=" + last, "--eqr_width=%d" % ew], capture_output=True, text=True, timeout=3000)
            assert p.returncode == 0, p.stderr[-2000:]
            dec, dev, enc, wall = timing(p.stderr)
            c2e[str(ew)] = {"wall_ms_per_frame": wall / a.frames, "decode_ms_per_frame": dec / a.frames,
                            "device_ms_per_frame": dev / a.frames,
                            "encode_ms_per_frame_summed_over_threads": enc / a.frames}
    finally:
        shutil.rmtree(tmp, True)

    res = {"gpu": name, "power_limit": limit, "rig": "golden 16-camera FTHETA, 3360 x 2160",
           "masks": "4096 x 2048 per camera, device-resident", "depth_m": 1000.0,
           "library_ms_per_call": lib_ms, "pixels_per_call": pixels, "host_resolved_pixels_per_call": host_px,
           "host_resolved_share": host_px / pixels, "ProjectEquirectsToCameras": app, "ProjectCamerasToEquirects": c2e}
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
